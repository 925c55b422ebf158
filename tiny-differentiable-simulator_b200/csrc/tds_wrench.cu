// Launchers of the world-frame kernel's external-wrench instances (tds_stepw.cu, template flag EXT; DESIGN.md section 7.18): the step in
// MODE_FD, MODE_NOCONTACT or MODE_FULL with a wrench [n; f] per environment at every point of a point table, in the three step precisions
// and as tangent-seeded dual numbers, with and without installed physical parameters.  A translation unit of its own for the reason
// tds_stepw_par.cu gives: the instances in the other units keep their code.  The vector-Jacobian product runs the JVP along identity
// tangents with the mass matrix's two helper kernels (tds_mass.cu).
#include <cuda_runtime.h>

#define TDS_STEPW_KERNEL_ONLY 1
#include "tds_stepw.cu"

#include "tds_model.h"

// the kernel argument: the instance's argument without EXT (B) and the point table, wrenches and wrench-sum region of layout M
template <typename B> static tdsw::ExtArg<B> ext_arg(const B& b, const TdsExtCall* xc, const DevModel* M, int size_ra, DevModel* Mx) {
  tdsw::ExtArg<B> a;
  memset(&a, 0, sizeof(a));
  static_cast<B&>(a) = b;
  *Mx = *M;
  a.ext.x_ext = tds_ext_layout_w(M, size_ra, &Mx->x_total);
  a.ext.W = xc->W; a.ext.t_W = xc->t_W;
  a.ext.K = xc->K;
  for (int k = 0; k < xc->K; ++k) {
    a.ext.link[k] = xc->link[k];
    if (xc->link[k] >= 0) a.ext.links_with_points |= 1ull << xc->link[k];
    for (int c = 0; c < 3; ++c) a.ext.local[3 * k + c] = xc->local[3 * k + c];
  }
  return a;
}

// q', qd' (io->q_out, io->qd_out; MODE_NOCONTACT, MODE_FULL) or qdd (io->qdd_out; MODE_FD) of one step with the wrenches xc->W, one lane per
// environment, 32 lanes per block on the arena in global memory.  M: the precision's layout; gscratch: ceil(n / 32) blocks of x_total * 128
// bytes with x_total of tds_ext_layout_w(M, size of RA).  pm: the installed parameters, or null.
extern "C" int tds_launch_wrench(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
                                 const TdsExtCall* xc, int mode, int use_pd, int precision, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  const int blocks = (io->n + 31) / 32;
  DevModel* Mx = new DevModel;
#define TDSW_EXT(RA, RC, RS)                                                                                                          \
  do {                                                                                                                                \
    if (pm) {                                                                                                                         \
      const ExtArg<ParMap> a = ext_arg(*pm, xc, M, (int)sizeof(RA), Mx);                                                              \
      tds_stepw_kernel<RA, RC, RS, float, false, true, false, false, false, false, false, false, false, true><<<blocks, 32, 0, stream>>>( \
          *Mx, *P, *E, *io, mode, use_pd, gscratch, a);                                                                               \
    } else {                                                                                                                          \
      const ExtArg<NoPar> a = ext_arg(NoPar{}, xc, M, (int)sizeof(RA), Mx);                                                           \
      tds_stepw_kernel<RA, RC, RS, float, false, false, false, false, false, false, false, false, false, true><<<blocks, 32, 0, stream>>>( \
          *Mx, *P, *E, *io, mode, use_pd, gscratch, a);                                                                               \
    }                                                                                                                                 \
  } while (0)
  if (precision == 0) TDSW_EXT(float, double, float);
  else if (precision == 1) TDSW_EXT(double, double, double);
  else TDSW_EXT(float, float, float);
#undef TDSW_EXT
  delete Mx;
  return (int)cudaGetLastError();
}

// Tangents [io->jac_dir0, io->jac_dir0 + n_dirs) of t_in [cols * m][ns], xc->t_W [6K * m][ns] and t_par [k * m][ns] (each may be null: zero
// tangent) -> columns of io->jac [rows * m][ns] (q' | qd', or qdd in MODE_FD; io->jac_n_in = m).  M must carry the 16-byte layout; gscratch:
// n_dirs * ceil(n / 32) blocks of x_total * 128 bytes with x_total of tds_ext_layout_w(M, 16).
extern "C" int tds_launch_wrench_jvp(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
                                     const TdsExtCall* xc, const double* t_in, const double* t_par, int m, int mode, int use_pd, int n_dirs,
                                     char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  typedef tds::Dual<double> D;
  const dim3 grid((io->n + 31) / 32, n_dirs);
  const JvpTan jv{t_in, t_par, m};
  DevModel* Mx = new DevModel;
  if (pm) {
    ParMapJvp b;
    static_cast<ParMap&>(b) = *pm;
    b.jv = jv;
    const ExtArg<ParMapJvp> a = ext_arg(b, xc, M, (int)sizeof(D), Mx);
    tds_stepw_kernel<D, D, D, D, false, true, true, false, false, false, false, false, false, true><<<grid, 32, 0, stream>>>(
        *Mx, *P, *E, *io, mode, use_pd, gscratch, a);
  } else {
    const ExtArg<NoParJvp> a = ext_arg(NoParJvp{jv}, xc, M, (int)sizeof(D), Mx);
    tds_stepw_kernel<D, D, D, D, false, false, true, false, false, false, false, false, false, true><<<grid, 32, 0, stream>>>(
        *Mx, *P, *E, *io, mode, use_pd, gscratch, a);
  }
  delete Mx;
  return (int)cudaGetLastError();
}
