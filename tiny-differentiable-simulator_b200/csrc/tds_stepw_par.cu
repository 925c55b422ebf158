// Launchers of the world-frame kernel's instances with per-environment physical parameters (tds_stepw.cu, template flag PAR;
// DESIGN.md section 7.9).  A translation unit of their own: nvcc's inlining of the kernel's shared device functions depends on
// how many instances call them, so keeping these instances out of tds_stepw.cu leaves the code of the instances there unchanged.
#include <cuda_runtime.h>

#define TDS_STEPW_KERNEL_ONLY 1
#include "tds_stepw.cu"

namespace tdsw {
template <typename RA, typename RC, typename RS, bool SM>
cudaError_t launch_par(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, int mode, int use_pd, char* gscratch,
                       int blocks, int threads, size_t smem, cudaStream_t stream, const ParMap& pm) {
  cudaError_t err = cudaSuccess;
  auto k = tds_stepw_kernel<RA, RC, RS, float, SM, true>;
  static size_t smem_set_dev[64] = {0}; int dev_ = 0; cudaGetDevice(&dev_); size_t& smem_set = smem_set_dev[dev_ & 63];
  if (smem > 48 * 1024 && smem > smem_set) {
    err = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err == cudaSuccess) smem_set = smem;
  }
  if (err == cudaSuccess) {
    k<<<blocks, threads, smem, stream>>>(*M, *P, *E, *io, mode, use_pd, gscratch, pm);
    err = cudaGetLastError();
  }
  return err;
}
}  // namespace tdsw

// tds_launch_stepw with the installed parameters pm
extern "C" int tds_launch_stepw_par(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
                                    int mode, int use_pd, int precision, char* gscratch, int use_smem, int warps_per_block,
                                    cudaStream_t stream) {
  using namespace tdsw;
  const int threads = 32 * warps_per_block;
  const int blocks = (io->n + threads - 1) / threads;
  const size_t smem = use_smem ? (size_t)warps_per_block * M->x_total * 32 * 4 : 0;
  cudaError_t err;
#define TDSW_PAR(RA, RC, RS) (use_smem ? launch_par<RA, RC, RS, true>(M, P, E, io, mode, use_pd, gscratch, blocks, threads, smem, stream, *pm) \
                                       : launch_par<RA, RC, RS, false>(M, P, E, io, mode, use_pd, gscratch, blocks, threads, smem, stream, *pm))
  if (precision == 0) err = TDSW_PAR(float, double, float);
  else if (precision == 1) err = TDSW_PAR(double, double, double);
  else err = TDSW_PAR(float, float, float);
#undef TDSW_PAR
  return (int)err;
}

// tds_launch_stepw_jacobian with the installed parameters: directions n_in + s (n_in = the Jacobian's input columns) are the
// parameters s, written to column s of io->jac; directions below n_in are the inputs, as without parameters.
extern "C" int tds_launch_stepw_jacobian_par(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
                                             int mode, int use_pd, int n_dirs, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  typedef tds::Dual<double> D;
  const dim3 grid((io->n + 31) / 32, n_dirs);
  tds_stepw_kernel<D, D, D, D, false, true><<<grid, 32, 0, stream>>>(*M, *P, *E, *io, mode, use_pd, gscratch, *pm);
  return (int)cudaGetLastError();
}

// tds_launch_stepw_vjp with the installed parameters: they are the tape's leaves after the inputs, pm->grad receives their
// cotangents; io->g_in and pm->grad may be null.
extern "C" int tds_launch_stepw_vjp_par(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
                                        int mode, int use_pd, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  typedef tds::Tape<double> T;
  tds_stepw_kernel<T, T, T, T, false, true><<<(io->n + 31) / 32, 32, 0, stream>>>(*M, *P, *E, *io, mode, use_pd, gscratch, *pm);
  return (int)cudaGetLastError();
}
