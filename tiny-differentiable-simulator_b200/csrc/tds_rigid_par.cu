// Launchers of the rigid-body kernel's instances with per-world physical parameters (tds_rigid.cu, template flag PAR; DESIGN.md
// section 7.11).  A translation unit of their own: nvcc's inlining of the kernel's shared device functions (sphere_sphere,
// plane_sphere) depends on how many instances call them, so keeping these instances out of tds_rigid.cu leaves the code of the
// instances there unchanged.
#include <cuda_runtime.h>

#define TDS_RIGID_KERNEL_ONLY 1
#include "tds_rigid.cu"

namespace {
const int kThreads = 128;
inline dim3 blocks(int n) { return dim3((n + kThreads - 1) / kThreads); }

// dst[s * ns + i] += src[s * ns + i], s < k, i < n: a chunk's per-step parameter cotangents into the rollout's sum
__global__ void rigid_accumulate_kernel(double* __restrict__ dst, const double* __restrict__ src, int k, int n, int ns) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int s = 0; s < k; ++s) dst[(size_t)s * ns + i] += src[(size_t)s * ns + i];
}
}  // namespace

// `steps` steps of n worlds by the fp64 instance with the parameters pm
extern "C" int tds_launch_rigid_step_par(const RigidWorld* W, const RigidParMap* pm, const double* s_in, double* s_out, const double* force,
                                         int steps, int n, int ns, cudaStream_t stream) {
  tdsrb::tds_rigid_step_kernel<double, double, false, true><<<blocks(n), kThreads, 0, stream>>>(*W, s_in, s_out, force, steps, n, ns, nullptr, 0,
                                                                                               tdsrb::RigidVjpIO{}, *pm);
  return (int)cudaGetLastError();
}

// the dual instance over directions dir0 .. dir0 + n_dirs - 1: below 16 n_bodies the state | force inputs (jac [13 nb * 16 nb][ns]),
// from 16 n_bodies on the installed parameters (jac [13 nb * k][ns])
extern "C" int tds_launch_rigid_jacobian_par(const RigidWorld* W, const RigidParMap* pm, const double* s_in, double* s_out, const double* force,
                                             int steps, int n, int ns, double* jac, int dir0, int n_dirs, cudaStream_t stream) {
  const dim3 grid(blocks(n).x, n_dirs);
  tdsrb::tds_rigid_step_kernel<tds::Dual<double>, double, false, true><<<grid, kThreads, 0, stream>>>(*W, s_in, s_out, force, steps, n, ns, jac,
                                                                                                     dir0, tdsrb::RigidVjpIO{}, *pm);
  return (int)cudaGetLastError();
}

// the tangent-seeded dual instance: one lane per (world, tangent), the parameters' tangents in pm->t_par
extern "C" int tds_launch_rigid_jvp_par(const RigidWorld* W, const RigidParMap* pm, const double* s_in, double* s_out, const double* force,
                                        int steps, int n, int ns, const tdsrb::RigidJvpIO* v, cudaStream_t stream) {
  const dim3 grid(blocks(n).x, v->m);
  tdsrb::tds_rigid_step_kernel<tds::Dual<double>, double, true, true><<<grid, kThreads, 0, stream>>>(*W, s_in, s_out, force, steps, n, ns, nullptr,
                                                                                                    0, *v, *pm);
  return (int)cudaGetLastError();
}

// one step of n worlds by the taping instance (values only when v->g_out is null); the parameters' cotangents go to pm->grad
extern "C" int tds_launch_rigid_vjp_par(const RigidWorld* W, const RigidParMap* pm, const double* s_in, double* s_out, const double* force,
                                        int n, int ns, const tdsrb::RigidVjpIO* v, cudaStream_t stream) {
  tdsrb::tds_rigid_step_kernel<tds::Tape<double>, double, false, true><<<blocks(n), kThreads, 0, stream>>>(*W, s_in, s_out, force, 1, n, ns,
                                                                                                          nullptr, 0, *v, *pm);
  return (int)cudaGetLastError();
}

extern "C" int tds_launch_rigid_accumulate(double* dst, const double* src, int k, int n, int ns, cudaStream_t stream) {
  rigid_accumulate_kernel<<<blocks(n), kThreads, 0, stream>>>(dst, src, k, n, ns);
  return (int)cudaGetLastError();
}
