// Launchers of the world-frame kernel's inverse-mass-matrix instances (tds_stepw.cu, template flags MASS and MINV; DESIGN.md section 7.20):
// M^-1(q) by the blocked Cholesky factor of the CRBA matrix the mass matrix returns, in fp64 and as tangent-seeded dual numbers, with and
// without installed physical parameters.  A translation unit of their own for the reason tds_stepw_par.cu gives: the instances in the
// other units keep their code.  Also the batched contraction of the operational-space inverse inertia J M^-1 J^T from the point Jacobians
// of the MOT instances and M^-1.  The vector-Jacobian product reuses the mass matrix's two helper kernels (tds_mass.cu).
#include <cuda_runtime.h>

#ifndef TDS_STEPW_KERNEL_ONLY
#define TDS_STEPW_KERNEL_ONLY 1
#endif
#include "tds_stepw.cu"
#include "tds_soa.cuh"

namespace {
constexpr int kMaxQd = 3 * TDS_MAX_LINKS + 6;

// Row a = blockIdx.y of L = J M^-1 J^T [R x R] (R = 6K) of environment e, tangent j = j0 + blockIdx.z: t = J_a M^-1, then L_ab = t . J_b for
// b >= a, written to (a, b) and (b, a).  J [R * nq][ns], Mi [nq * nq][ns] (values) with their tangents dJ [R * nq * m][ns] and
// dMi [nq * nq * m][ns] (Dual instance; dJ may be null: zero), L [R * R][ns] or its tangents [R * R * m][ns].
template <typename T>
__global__ void osim_kernel(const double* J, const double* dJ, const double* Mi, const double* dMi, double* L, int R, int nq, int m, int j0,
                            int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int a = blockIdx.y, j = j0 + (int)blockIdx.z;
  if (e >= n) return;
  T t[kMaxQd];
  for (int c = 0; c < nq; ++c) t[c] = T(0.0);
  for (int r = 0; r < nq; ++r) {
    const T jr = osim_ld<T>(J, dJ, (size_t)a * nq + r, m, j, ns, e);
    for (int c = 0; c < nq; ++c) t[c] = t[c] + jr * osim_ld<T>(Mi, dMi, (size_t)r * nq + c, m, j, ns, e);
  }
  for (int b = a; b < R; ++b) {
    T acc = T(0.0);
    for (int c = 0; c < nq; ++c) acc = acc + t[c] * osim_ld<T>(J, dJ, (size_t)b * nq + c, m, j, ns, e);
    osim_st(L, acc, (size_t)a * R + b, m, j, ns, e);
    if (b > a) osim_st(L, acc, (size_t)b * R + a, m, j, ns, e);
  }
}
}  // namespace

// (TDS_MINV_KERNEL_ONLY: the contraction kernel alone, for the host build of the tests)
#ifndef TDS_MINV_KERNEL_ONLY
// (the MINV lanes run in MODE_NOCONTACT, as the MASS lanes)

// M^-1 [n_qd * n_qd][ns] (io->jac, row-major per environment) from io->q_in.  M must carry the 8-byte layout
// (tds_build_layout_w(..., 8, 8, 8, -1, 8)); gscratch: ceil(n / 32) blocks of x_total * 128 bytes.  pm: the installed parameters, or null.
extern "C" int tds_launch_mass_inverse(const DevModel* M, const StepIO* io, const ParMap* pm, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  SimParams P;
  EnvParams E;
  memset(&P, 0, sizeof(P));
  memset(&E, 0, sizeof(E));
  const dim3 grid((io->n + 31) / 32, 1);
  if (pm)
    tds_stepw_kernel<double, double, double, double, false, true, false, true, false, false, false, false, false, false, false, true>
        <<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0, gscratch, *pm);
  else
    tds_stepw_kernel<double, double, double, double, false, false, false, true, false, false, false, false, false, false, false, true>
        <<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0, gscratch, NoPar{});
  return (int)cudaGetLastError();
}

// Tangents [io->jac_dir0, io->jac_dir0 + n_dirs) of t_q [n_q * m][ns] / t_par [k * m][ns] (either may be null: zero tangent) ->
// columns of dM^-1 = io->jac [n_qd * n_qd * m][ns] (io->jac_n_in = m).  M must carry the 16-byte layout; gscratch: n_dirs * ceil(n / 32)
// blocks of x_total * 128 bytes.
extern "C" int tds_launch_mass_inverse_jvp(const DevModel* M, const StepIO* io, const ParMap* pm, const double* t_q, const double* t_par,
                                           int m, int n_dirs, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  typedef tds::Dual<double> D;
  SimParams P;
  EnvParams E;
  memset(&P, 0, sizeof(P));
  memset(&E, 0, sizeof(E));
  const dim3 grid((io->n + 31) / 32, n_dirs);
  const JvpTan jv{t_q, t_par, m};
  if (pm) {
    ParMapJvp a;
    static_cast<ParMap&>(a) = *pm;
    a.jv = jv;
    tds_stepw_kernel<D, D, D, D, false, true, true, true, false, false, false, false, false, false, false, true>
        <<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0, gscratch, a);
  } else {
    tds_stepw_kernel<D, D, D, D, false, false, true, true, false, false, false, false, false, false, false, true>
        <<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0, gscratch, NoParJvp{jv});
  }
  return (int)cudaGetLastError();
}

// Lambda^-1 = J M^-1 J^T [6K * 6K][ns] of every environment from J [6K * n_qd][ns] (the MOT instances' spatial point Jacobians) and
// Mi [n_qd * n_qd][ns] (above).  With dMi (m tangents), the tangents dLambda^-1 [36 K^2 * m][ns] from those of J (dJ; null: zero) and M^-1.
extern "C" int tds_launch_osim(const double* J, const double* dJ, const double* Mi, const double* dMi, double* L, int K, int n_qd, int m,
                               int n, int ns, cudaStream_t stream) {
  if (n_qd > kMaxQd) return (int)cudaErrorInvalidValue;
  if (!dMi) {
    osim_kernel<double><<<dim3((n + 127) / 128, 6 * K, 1), 128, 0, stream>>>(J, nullptr, Mi, nullptr, L, 6 * K, n_qd, 1, 0, n, ns);
    return (int)cudaGetLastError();
  }
  for (int j0 = 0; j0 < m; j0 += 65535) {   // (gridDim.z)
    const int nz = m - j0 < 65535 ? m - j0 : 65535;
    osim_kernel<tds::Dual<double>><<<dim3((n + 127) / 128, 6 * K, nz), 128, 0, stream>>>(J, dJ, Mi, dMi, L, 6 * K, n_qd, m, j0, n, ns);
    if (const cudaError_t err = cudaGetLastError()) return (int)err;
  }
  return 0;
}
#endif  // TDS_MINV_KERNEL_ONLY
