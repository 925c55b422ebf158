// Launchers of the world-frame kernel's mass-matrix instances (tds_stepw.cu, template flag MASS; DESIGN.md section 7.12): M(q) by
// the CRBA the contact solve factors, in fp64 and as tangent-seeded dual numbers, with and without installed physical parameters.  A
// translation unit of their own for the reason tds_stepw_par.cu gives: the instances in the other units keep their code.  Also the
// two small kernels of the mass matrix's vector-Jacobian product (identity tangents, contraction with the cotangent).
#include <cuda_runtime.h>

#define TDS_STEPW_KERNEL_ONLY 1
#include "tds_stepw.cu"

// (the MASS lanes run in MODE_NOCONTACT: no contact detection, and the mode read of the step is left as it is)

// M [n_qd * n_qd][ns] (io->jac, row-major per environment) from io->q_in.  M must carry the 8-byte layout
// (tds_build_layout_w(..., 8, 8, 8, -1, 8)); gscratch: ceil(n / 32) blocks of x_total * 128 bytes.  pm: the installed parameters, or null.
extern "C" int tds_launch_mass(const DevModel* M, const StepIO* io, const ParMap* pm, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  SimParams P;
  EnvParams E;
  memset(&P, 0, sizeof(P));
  memset(&E, 0, sizeof(E));
  const dim3 grid((io->n + 31) / 32, 1);
  if (pm) tds_stepw_kernel<double, double, double, double, false, true, false, true><<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0, gscratch, *pm);
  else tds_stepw_kernel<double, double, double, double, false, false, false, true><<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0, gscratch, NoPar{});
  return (int)cudaGetLastError();
}

// Tangents [io->jac_dir0, io->jac_dir0 + n_dirs) of t_q [n_q * m][ns] / t_par [k * m][ns] (either may be null: zero tangent) ->
// columns of dM = io->jac [n_qd * n_qd * m][ns] (io->jac_n_in = m).  M must carry the 16-byte layout; gscratch: n_dirs * ceil(n / 32)
// blocks of x_total * 128 bytes.
extern "C" int tds_launch_mass_jvp(const DevModel* M, const StepIO* io, const ParMap* pm, const double* t_q, const double* t_par, int m,
                                   int n_dirs, char* gscratch, cudaStream_t stream) {
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
    tds_stepw_kernel<D, D, D, D, false, true, true, true><<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0, gscratch, a);
  } else {
    tds_stepw_kernel<D, D, D, D, false, false, true, true><<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0, gscratch, NoParJvp{jv});
  }
  return (int)cudaGetLastError();
}

namespace {
// identity tangents of directions [d0, d0 + m) over the inputs q (n_q columns) | installed parameters (k columns):
// t_q [(c m + j) ns + e] = (c == d0 + j), t_par [(s m + j) ns + e] = (n_q + s == d0 + j)
__global__ void mass_eye_kernel(double* t_q, double* t_par, int n_q, int k, int d0, int m, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y;   // input column
  if (e >= ns) return;
  for (int j = 0; j < m; ++j) {
    const double v = c == d0 + j ? 1.0 : 0.0;
    if (c < n_q) t_q[((size_t)c * m + j) * ns + e] = v;
    else t_par[((size_t)(c - n_q) * m + j) * ns + e] = v;
  }
}

// g[d0 + j] = sum_r G[r] dM[r][j] over the nn entries r of M, in the order of r; inputs below n_q go to g_q, the rest to g_par
__global__ void mass_contract_kernel(const double* G, const double* dM, int nn, int m, int d0, int n_q, double* g_q, double* g_par, int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int j = blockIdx.y;
  if (e >= n) return;
  double acc = 0.0;
  for (int r = 0; r < nn; ++r) acc += G[(size_t)r * ns + e] * dM[((size_t)r * m + j) * ns + e];
  const int c = d0 + j;
  if (c < n_q) { if (g_q) g_q[(size_t)c * ns + e] = acc; }
  else if (g_par) g_par[(size_t)(c - n_q) * ns + e] = acc;
}
}  // namespace

extern "C" int tds_launch_mass_eye(double* t_q, double* t_par, int n_q, int k, int d0, int m, int ns, cudaStream_t stream) {
  mass_eye_kernel<<<dim3((ns + 127) / 128, n_q + k), 128, 0, stream>>>(t_q, t_par, n_q, k, d0, m, ns);
  return (int)cudaGetLastError();
}

extern "C" int tds_launch_mass_contract(const double* G, const double* dM, int nn, int m, int d0, int n_q, double* g_q, double* g_par, int n,
                                        int ns, cudaStream_t stream) {
  mass_contract_kernel<<<dim3((n + 127) / 128, m), 128, 0, stream>>>(G, dM, nn, m, d0, n_q, g_q, g_par, n, ns);
  return (int)cudaGetLastError();
}
