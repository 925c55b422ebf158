// Lane-team kernel: one environment is advanced by a team of TDS_TEAM_T = 4 adjacent lanes, lane % 4 = role
// (8 environments per warp, one warp per CTA).  The step body is tds_team_step.cuh; this file holds the thread
// mapping and the launcher.
//
// Each warp works on its own block of scratch: the team region [word][team] (stride 8) followed by the lane region
// [word][lane] (stride 32).  The link table is read from global memory through the non-coherent path, the four
// lanes of a team meet at __syncwarp and combine partial results with xor shuffles.  The library selects this
// kernel when a role-warp tile does not fit in shared memory (tds_capi.cu).
#include <cuda_runtime.h>

#include "tds_team_step.cuh"

namespace tdsteam {

struct LaneTeam {
  static constexpr bool ROLE_WARPS = false;
  static constexpr int THREADS = 32, MIN_BLOCKS = 4;
  static constexpr int STM = 32 / TDS_TEAM_T;           // environments per warp
  static constexpr bool MAX_CARVEOUT = true;            // several one-warp CTAs must be co-resident per SM
  static TDS_D int role() { return (threadIdx.x & 31) % TDS_TEAM_T; }
  static TDS_D int team() { return (threadIdx.x & 31) / TDS_TEAM_T; }
  static TDS_D int tile() { return (blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
  static TDS_D const TeamLink* table(const TeamLink* tl, int role) { return tl + (size_t)role * TDS_TEAM_MAXK; }
  template <typename T> static TDS_D T ld(const T& x) { return __ldg(&x); }
  static TDS_D void sync() { __syncwarp(); }
  static __host__ __device__ size_t tile_bytes(const TeamModel& TM) { return ((size_t)TM.t_total * STM + (size_t)TM.l_total * 32) * 4; }
  static TDS_D char* role_base(const TeamModel& TM, char* tb, int) { return tb + (size_t)TM.t_total * STM * 4; }
  static TDS_D size_t clock_row(int tile, int) { return (size_t)tile; }
};

}  // namespace tdsteam

#ifndef TDS_TEAM_KERNEL_ONLY   // launcher: not part of the host-compiled kernel source (tests/cpp/team_host.cpp)
extern "C" int tds_launch_stept(const TeamModel* TM, const TeamLink* tl_dev, const DevModel* M, const SimParams* P,
                                const EnvParams* E, const StepIO* io, int mode, int use_pd, int precision,
                                char* gscratch, int use_smem, cudaStream_t stream) {
  return tdsteam::launch_team_step<tdsteam::LaneTeam>(TM, tl_dev, M, P, E, io, mode, use_pd, precision, gscratch,
                                                      use_smem, stream);
}

// bytes of shared memory (or global scratch) one warp of 8 environments needs
extern "C" size_t tds_stept_tile_bytes(const TeamModel* TM) { return tdsteam::LaneTeam::tile_bytes(*TM); }
#endif  // TDS_TEAM_KERNEL_ONLY
