// Role-warp kernel: one CTA = a tile of 32 environments x 4 warps; warp r advances the links of role r of the
// tree decomposition of tds_team.h (role 0: trunk + one subtree, roles 1..3: one subtree each) for the 32
// environments of the tile, lane = environment.  The step body is tds_team_step.cuh; this file holds the thread
// mapping and the launcher.
//
// Inside a warp every lane executes the same link with the same model constants (uniform index arithmetic, link
// table in constant memory, all 32 lanes active, no divergence between roles), and the four warps of a CTA run on
// the four schedulers of one SM.  The CTA's block of scratch is the shared region [word][environment] plus XTRA
// words, then one private region [word][environment] per role.  Roles communicate through the shared region and
// CTA barriers:
//   load | B | pass 1a (role 0: trunk) | B | pass 1b (all: subtrees), active contact set | B | pass 2a (all) | B |
//   role 0: sums the attachment accumulators, pass 2b, base, pass 3a | B | pass 3b, own-block factorisation,
//   partial Schur complements (all) | B | role 0: trunk factorisation | B | Y rows of own contacts (all) |
//   PGS in the reference's row order, one barrier whenever the owner of the next row changes | B |
//   role 0: z_trunk | B | z_own, integrate | B | write back.
#include <cuda_runtime.h>

#include "tds_team_step.cuh"

namespace tdsteam {

// per-role link tables (tds_team.h); uniform index per warp -> constant-cache broadcast
__constant__ TeamLink c_team[TDS_TEAM_T * TDS_TEAM_MAXK];

struct RoleWarps {
  static constexpr bool ROLE_WARPS = true;
  static constexpr int THREADS = 32 * TDS_TEAM_T, MIN_BLOCKS = 1;
  static constexpr int STM = 32;                        // environments per CTA
  static constexpr int XTRA = 12;                       // words appended to the shared region: active masks (2 per role), done flag
  static constexpr bool MAX_CARVEOUT = false;
  static TDS_D int role() { return __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0); }   // warp index, known uniform to the compiler
  static TDS_D int team() { return threadIdx.x & 31; }
  static TDS_D int tile() { return blockIdx.x; }
  static TDS_D const TeamLink* table(const TeamLink*, int role) { return c_team + role * TDS_TEAM_MAXK; }
  template <typename T> static TDS_D T ld(const T& x) { return x; }
  static TDS_D void sync() { __syncthreads(); }
  static __host__ __device__ size_t tile_bytes(const TeamModel& TM) {
    return ((size_t)(TM.t_total + XTRA) + (size_t)TDS_TEAM_T * TM.l_total) * 32 * 4;
  }
  static TDS_D char* role_base(const TeamModel& TM, char* tb, int r) {
    return tb + ((size_t)(TM.t_total + XTRA) + (size_t)r * TM.l_total) * 32 * 4;
  }
  static TDS_D size_t clock_row(int tile, int role) { return (size_t)tile * TDS_TEAM_T + role; }
};

}  // namespace tdsteam

#ifndef TDS_TEAM_KERNEL_ONLY   // launcher: not part of the host-compiled kernel source (tests/cpp/team_host.cpp)
// The link table lives in constant memory: one table resident per device.  `token` identifies the table of the
// calling simulator; a different token re-uploads (after draining the device, since kernels of the previous owner
// may still be reading the symbol).  Not allowed while the stream is being captured into a CUDA graph.
static unsigned long long g_table_token[64] = {0};

// Owner of the table resident on a device (0: none yet).  A CUDA graph that holds a launch of this kernel replays WITHOUT
// passing through tds_launch_stepr: whoever replays one must check that its simulator still owns the table (the library's
// own graph of tds_b200_env_step_host does, tds_capi.cu; user captures of tds_b200_env_step_device: see INTEGRATION.md).
extern "C" unsigned long long tds_stepr_table_owner(int dev) { return (dev >= 0 && dev < 64) ? g_table_token[dev] : 0ull; }

extern "C" int tds_launch_stepr(const TeamModel* TM, const TeamLink* tl_host, unsigned long long token, const DevModel* M,
                                const SimParams* P, const EnvParams* E, const StepIO* io, int mode, int use_pd,
                                int precision, char* gscratch, int use_smem, cudaStream_t stream) {
  using namespace tdsteam;
  int dev = 0;
  cudaError_t err = cudaGetDevice(&dev);
  if (err != cudaSuccess) return (int)err;
  if (dev < 0 || dev >= 64) return (int)cudaErrorInvalidDevice;
  if (g_table_token[dev] != token) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (stream && cudaStreamIsCapturing(stream, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone)
      return (int)cudaErrorStreamCaptureUnsupported;
    err = cudaDeviceSynchronize();
    if (err == cudaSuccess) err = cudaMemcpyToSymbol(c_team, tl_host, sizeof(TeamLink) * TDS_TEAM_T * TDS_TEAM_MAXK);
    if (err != cudaSuccess) return (int)err;
    g_table_token[dev] = token;
  }
  return launch_team_step<RoleWarps>(TM, nullptr, M, P, E, io, mode, use_pd, precision, gscratch, use_smem, stream);
}

// bytes of shared memory (or global scratch) one tile of 32 environments needs
extern "C" size_t tds_stepr_tile_bytes(const TeamModel* TM) { return tdsteam::RoleWarps::tile_bytes(*TM); }
#endif  // TDS_TEAM_KERNEL_ONLY
