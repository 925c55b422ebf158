// Launchers of the world-frame kernel's Jacobian-vector product instances (tds_stepw.cu, template flag JV; DESIGN.md section 7.10):
// the dual-number instance with its lanes seeded by given tangents instead of unit directions, with and without installed physical
// parameters.  A translation unit of their own for the reason tds_stepw_par.cu gives: the instances in tds_stepw.cu and
// tds_stepw_par.cu keep their code.
#include <cuda_runtime.h>

#define TDS_STEPW_KERNEL_ONLY 1
#include "tds_stepw.cu"

// Tangents [io->jac_dir0, io->jac_dir0 + n_dirs) of t_in [cols * m][ns] / t_par [k * m][ns] (either may be null: zero tangent) ->
// columns of io->jac [rows * m][ns] (io->jac_n_in = m).  pm: the installed parameters, or null.  gscratch as for
// tds_launch_stepw_jacobian: n_dirs * ceil(n / 32) blocks of x_total * 128 bytes.
extern "C" int tds_launch_stepw_jvp(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
                                    const double* t_in, const double* t_par, int m, int mode, int use_pd, int n_dirs, char* gscratch,
                                    cudaStream_t stream) {
  using namespace tdsw;
  typedef tds::Dual<double> D;
  const dim3 grid((io->n + 31) / 32, n_dirs);
  const JvpTan jv{t_in, t_par, m};
  if (pm) {
    ParMapJvp a;
    static_cast<ParMap&>(a) = *pm;
    a.jv = jv;
    tds_stepw_kernel<D, D, D, D, false, true, true><<<grid, 32, 0, stream>>>(*M, *P, *E, *io, mode, use_pd, gscratch, a);
  } else {
    tds_stepw_kernel<D, D, D, D, false, false, true><<<grid, 32, 0, stream>>>(*M, *P, *E, *io, mode, use_pd, gscratch, NoParJvp{jv});
  }
  return (int)cudaGetLastError();
}
