// Launchers of the world-frame kernel's regressor instances (tds_stepw.cu, template flags INV and REG; DESIGN.md section 7.19): the
// joint-torque regressor Y(q, qd, qdd) with tau = Y pi and the energy regressors yT(q, qd), yV(q) of the inertial, stiffness and damping
// parameters pi, in fp64 and as tangent-seeded dual numbers.  A translation unit of their own for the reason tds_stepw_par.cu gives: the
// instances in the other units keep their code.  The vector-Jacobian product reuses the mass matrix's two helper kernels (tds_mass.cu).
#include <cuda_runtime.h>

#define TDS_STEPW_KERNEL_ONLY 1
#include "tds_stepw.cu"

// (the REG lanes run in MODE_NOCONTACT without PD, as the INV lanes: no contact detection; P supplies the gravity; installed parameters
// do not enter)

// Y [n_qd * n_pi][ns] (io->jac, entry (r, c) at row r * n_pi + c), yT and yV [n_pi][ns] (out, each may be null) from io->q_in, io->qd_in
// and io->tau_in = qdd (either of the last two may be null: zero).  M must carry the 8-byte layout (tds_build_layout_w(..., 8, 8, 8, -1,
// 8)); gscratch: ceil(n / 32) blocks of x_total * 128 bytes.
extern "C" int tds_launch_regressor(const DevModel* M, const SimParams* P, const StepIO* io, const TdsRegCall* out, char* gscratch,
                                    cudaStream_t stream) {
  using namespace tdsw;
  EnvParams E;
  memset(&E, 0, sizeof(E));
  const dim3 grid((io->n + 31) / 32, 1);
  RegArg<NoPar> a;
  a.yT = out->yT; a.yV = out->yV;
  tds_stepw_kernel<double, double, double, double, false, false, false, false, false, true, false, false, false, false, true>
      <<<grid, 32, 0, stream>>>(*M, *P, E, *io, MODE_NOCONTACT, 0, gscratch, a);
  return (int)cudaGetLastError();
}

// Tangents [io->jac_dir0, io->jac_dir0 + n_dirs) of t_in [(n_q + 2 n_qd) * m][ns] (q | qd | qdd) -> columns of dY = io->jac
// [n_qd * n_pi * m][ns], dyT and dyV [n_pi * m][ns] (out; rows at (r * m + j) * ns + e, io->jac_n_in = m).  M must carry the 16-byte layout;
// gscratch: n_dirs * ceil(n / 32) blocks of x_total * 128 bytes.
extern "C" int tds_launch_regressor_jvp(const DevModel* M, const SimParams* P, const StepIO* io, const TdsRegCall* out, const double* t_in,
                                        int m, int n_dirs, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  typedef tds::Dual<double> D;
  EnvParams E;
  memset(&E, 0, sizeof(E));
  const dim3 grid((io->n + 31) / 32, n_dirs);
  RegArg<NoParJvp> a;
  a.jv = JvpTan{t_in, nullptr, m};
  a.yT = out->yT; a.yV = out->yV;
  tds_stepw_kernel<D, D, D, D, false, false, true, false, false, true, false, false, false, false, true><<<grid, 32, 0, stream>>>(
      *M, *P, E, *io, MODE_NOCONTACT, 0, gscratch, a);
  return (int)cudaGetLastError();
}
