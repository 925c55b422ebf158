// Launchers of the world-frame kernel's contact-reporting instances (tds_stepw.cu, template flag CF; DESIGN.md section 7.15): the step
// in MODE_FULL or MODE_WORLD that also writes one record per contact candidate (normal on b, point on b, distance, impulse on b), in the
// three step precisions and as tangent-seeded dual numbers, with and without installed physical parameters.  A translation unit of its
// own for the reason tds_stepw_par.cu gives: the instances in the other units keep their code.  The vector-Jacobian product runs the JVP
// along identity tangents with the mass matrix's two helper kernels (tds_mass.cu).
#include <cuda_runtime.h>

#define TDS_STEPW_KERNEL_ONLY 1
#include "tds_stepw.cu"

// q', qd' (io->q_out, io->qd_out) and the records cf [10 * n_pts][ns] fp32 of one step, one lane per environment, 32 lanes per block on
// the arena in global memory (the arena's place does not change the arithmetic: q' and qd' are those of tds_launch_stepw).  M: the
// precision's layout; gscratch: ceil(n / 32) blocks of x_total * 128 bytes.  pm: the installed parameters, or null.
extern "C" int tds_launch_contacts(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm, float* cf,
                                   int mode, int use_pd, int precision, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  const int blocks = (io->n + 31) / 32;
#define TDSW_CF(RA, RC, RS)                                                                                                          \
  do {                                                                                                                               \
    if (pm) {                                                                                                                        \
      CfArgPar a;                                                                                                                    \
      static_cast<ParMap&>(a) = *pm;                                                                                                 \
      a.cf = cf;                                                                                                                     \
      tds_stepw_kernel<RA, RC, RS, float, false, true, false, false, false, false, true><<<blocks, 32, 0, stream>>>(*M, *P, *E, *io, \
                                                                                                                 mode, use_pd, gscratch, a); \
    } else {                                                                                                                         \
      tds_stepw_kernel<RA, RC, RS, float, false, false, false, false, false, false, true><<<blocks, 32, 0, stream>>>(               \
          *M, *P, *E, *io, mode, use_pd, gscratch, CfArg{cf});                                                                       \
    }                                                                                                                                \
  } while (0)
  if (precision == 0) TDSW_CF(float, double, float);
  else if (precision == 1) TDSW_CF(double, double, double);
  else TDSW_CF(float, float, float);
#undef TDSW_CF
  return (int)cudaGetLastError();
}

// Tangents [io->jac_dir0, io->jac_dir0 + n_dirs) of t_in [cols * m][ns] / t_par [k * m][ns] (either may be null: zero tangent) ->
// columns of io->jac [(n_q + n_qd + 10 n_pts) * m][ns] (q' | qd' | records, io->jac_n_in = m).  M must carry the 16-byte layout;
// gscratch: n_dirs * ceil(n / 32) blocks of x_total * 128 bytes.
extern "C" int tds_launch_contacts_jvp(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
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
    tds_stepw_kernel<D, D, D, D, false, true, true, false, false, false, true><<<grid, 32, 0, stream>>>(*M, *P, *E, *io, mode, use_pd, gscratch, a);
  } else {
    tds_stepw_kernel<D, D, D, D, false, false, true, false, false, false, true><<<grid, 32, 0, stream>>>(*M, *P, *E, *io, mode, use_pd, gscratch,
                                                                                                      NoParJvp{jv});
  }
  return (int)cudaGetLastError();
}
