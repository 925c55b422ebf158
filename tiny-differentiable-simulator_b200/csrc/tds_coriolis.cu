// Launchers of the world-frame kernel's Coriolis-matrix instances (tds_stepw.cu, template flag COR; DESIGN.md section 7.22): C(q, qd) of
// Echeandia & Wensing in the coordinates of the mass matrix, in fp64 and as tangent-seeded dual numbers, with and without installed
// physical parameters.  A translation unit of their own for the reason tds_stepw_par.cu gives: the instances in the other units keep
// their code.  The vector-Jacobian product reuses the mass matrix's two helper kernels (tds_mass.cu).
#include <cuda_runtime.h>

#define TDS_STEPW_KERNEL_ONLY 1
#include "tds_stepw.cu"

// (the COR lanes run in MODE_NOCONTACT without PD and without gravity: no contact detection)

// C [n_qd * n_qd][ns] (io->jac, row-major per environment) from io->q_in and io->qd_in (null: zero).  M must carry the 8-byte layout
// (tds_build_layout_w(..., 8, 8, 8, -1, 8)); gscratch: ceil(n / 32) blocks of x_total * 128 bytes.  pm: the installed parameters, or null.
extern "C" int tds_launch_coriolis(const DevModel* M, const StepIO* io, const ParMap* pm, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  SimParams P;
  EnvParams E;
  memset(&P, 0, sizeof(P));
  memset(&E, 0, sizeof(E));
  const dim3 grid((io->n + 31) / 32, 1);
  if (pm)
    tds_stepw_kernel<double, double, double, double, false, true, false, false, false, false, false, false, false, false, false, false, true>
        <<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0, gscratch, *pm);
  else
    tds_stepw_kernel<double, double, double, double, false, false, false, false, false, false, false, false, false, false, false, false, true>
        <<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0, gscratch, NoPar{});
  return (int)cudaGetLastError();
}

// Tangents [io->jac_dir0, io->jac_dir0 + n_dirs) of t_in [(n_q + n_qd) * m][ns] (q | qd) and t_par [k * m][ns] (either may be null: zero
// tangent) -> columns of dC = io->jac [n_qd * n_qd * m][ns] (io->jac_n_in = m).  M must carry the 16-byte layout; gscratch: n_dirs *
// ceil(n / 32) blocks of x_total * 128 bytes.
extern "C" int tds_launch_coriolis_jvp(const DevModel* M, const StepIO* io, const ParMap* pm, const double* t_in, const double* t_par, int m,
                                       int n_dirs, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  typedef tds::Dual<double> D;
  SimParams P;
  EnvParams E;
  memset(&P, 0, sizeof(P));
  memset(&E, 0, sizeof(E));
  const dim3 grid((io->n + 31) / 32, n_dirs);
  const JvpTan jv{t_in, t_par, m};
  if (pm) {
    ParMapJvp a;
    static_cast<ParMap&>(a) = *pm;
    a.jv = jv;
    tds_stepw_kernel<D, D, D, D, false, true, true, false, false, false, false, false, false, false, false, false, true>
        <<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0, gscratch, a);
  } else {
    tds_stepw_kernel<D, D, D, D, false, false, true, false, false, false, false, false, false, false, false, false, true>
        <<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0, gscratch, NoParJvp{jv});
  }
  return (int)cudaGetLastError();
}
