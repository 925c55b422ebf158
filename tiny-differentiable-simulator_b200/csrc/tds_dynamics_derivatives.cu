// Launchers of the world-frame kernel's dynamics-derivative instances (tds_stepw.cu, template flag DER; DESIGN.md section 7.23): d tau / dq
// and d tau / dqd of the inverse dynamics in the velocities' tangent coordinates, in fp64 and as tangent-seeded dual numbers, with and
// without installed physical parameters.  A translation unit of their own for the reason tds_stepw_par.cu gives: the instances in the
// other units keep their code.  The vector-Jacobian product reuses the mass matrix's two helper kernels (tds_mass.cu).
#include <cuda_runtime.h>

#define TDS_STEPW_KERNEL_ONLY 1
#include "tds_stepw.cu"

#include "tds_model.h"

// (the DER lanes run in MODE_NOCONTACT without PD, as INV's: no contact detection; P supplies the gravity)

// d tau / dq (io->jac) and d tau / dqd (io->g_in) [n_qd * n_qd][ns] (either may be null) from io->q_in, io->qd_in and io->tau_in = qdd (either
// of the last two may be null: zero), or qdd in fp64 from io->g_out [n_qd][ns] when that is not null (DESIGN.md section 7.24).  M: the 8-byte layout (tds_build_layout_w(..., 8, 8, 8, -1, 8)); gscratch: ceil(n / 32) blocks of
// tds_der_layout_w(M, 8) * 128 bytes.  pm: the installed parameters, or null.
extern "C" int tds_launch_dynamics_derivatives(const DevModel* M, const SimParams* P, const StepIO* io, const ParMap* pm, char* gscratch,
                                               cudaStream_t stream) {
  using namespace tdsw;
  EnvParams E;
  memset(&E, 0, sizeof(E));
  DevModel* Md = new DevModel(*M);
  Md->x_total = tds_der_layout_w(M, 8);
  const dim3 grid((io->n + 31) / 32, 1);
  if (pm)
    tds_stepw_kernel<double, double, double, double, false, true, false, false, false, false, false, false, false, false, false, false, false,
                     true><<<grid, 32, 0, stream>>>(*Md, *P, E, *io, MODE_NOCONTACT, 0, gscratch, *pm);
  else
    tds_stepw_kernel<double, double, double, double, false, false, false, false, false, false, false, false, false, false, false, false, false,
                     true><<<grid, 32, 0, stream>>>(*Md, *P, E, *io, MODE_NOCONTACT, 0, gscratch, NoPar{});
  delete Md;
  return (int)cudaGetLastError();
}

// Tangents [io->jac_dir0, io->jac_dir0 + n_dirs) of t_in [(n_q + 2 n_qd) * m][ns] (q | qd | qdd, the q tangents in n_q coordinates) and
// t_par [k * m][ns] (either may be null: zero tangent) -> columns of the derivatives' tangents io->jac and io->g_in [n_qd * n_qd * m][ns]
// (io->jac_n_in = m; either may be null).  M: the 16-byte layout; gscratch: n_dirs * ceil(n / 32) blocks of tds_der_layout_w(M, 16) * 128
// bytes.
extern "C" int tds_launch_dynamics_derivatives_jvp(const DevModel* M, const SimParams* P, const StepIO* io, const ParMap* pm, const double* t_in,
                                                   const double* t_par, int m, int n_dirs, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  typedef tds::Dual<double> D;
  EnvParams E;
  memset(&E, 0, sizeof(E));
  DevModel* Md = new DevModel(*M);
  Md->x_total = tds_der_layout_w(M, 16);
  const dim3 grid((io->n + 31) / 32, n_dirs);
  const JvpTan jv{t_in, t_par, m};
  if (pm) {
    ParMapJvp a;
    static_cast<ParMap&>(a) = *pm;
    a.jv = jv;
    tds_stepw_kernel<D, D, D, D, false, true, true, false, false, false, false, false, false, false, false, false, false, true>
        <<<grid, 32, 0, stream>>>(*Md, *P, E, *io, MODE_NOCONTACT, 0, gscratch, a);
  } else {
    tds_stepw_kernel<D, D, D, D, false, false, true, false, false, false, false, false, false, false, false, false, false, true>
        <<<grid, 32, 0, stream>>>(*Md, *P, E, *io, MODE_NOCONTACT, 0, gscratch, NoParJvp{jv});
  }
  delete Md;
  return (int)cudaGetLastError();
}
