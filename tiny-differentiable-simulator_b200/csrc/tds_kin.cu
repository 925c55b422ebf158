// Launchers of the world-frame kernel's kinematics instances (tds_stepw.cu, template flag KIN; DESIGN.md section 7.13): link world
// transforms, world positions and linear point Jacobians of a point table from q alone, in fp64 and as tangent-seeded dual numbers.  A
// translation unit of their own for the reason tds_stepw_par.cu gives: the instances in the other units keep their code.  The
// vector-Jacobian product reuses the mass matrix's two helper kernels (tds_mass.cu).
#include <cuda_runtime.h>

#define TDS_STEPW_KERNEL_ONLY 1
#include "tds_stepw.cu"

static tdsw::KinArg kin_arg(const TdsKinCall* kc) {
  tdsw::KinArg a;
  memset(&a, 0, sizeof(a));
  a.xf = kc->xf; a.x = kc->x; a.J = kc->J;
  a.K = kc->K;
  for (int k = 0; k < kc->K; ++k) {
    a.link[k] = kc->link[k];
    for (int c = 0; c < 3; ++c) a.local[3 * k + c] = kc->local[3 * k + c];
  }
  return a;
}

// fp64 outputs from io->q_in (rows at r * ns + e).  M must carry the 8-byte layout (tds_build_layout_w(..., 8, 8, 8, -1, 8)); gscratch:
// ceil(n / 32) blocks of x_total * 128 bytes.
extern "C" int tds_launch_kin(const DevModel* M, const StepIO* io, const TdsKinCall* kc, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  SimParams P;
  EnvParams E;
  memset(&P, 0, sizeof(P));
  memset(&E, 0, sizeof(E));
  const dim3 grid((io->n + 31) / 32, 1);
  tds_stepw_kernel<double, double, double, double, false, false, false, false, true><<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0,
                                                                                                          gscratch, kin_arg(kc));
  return (int)cudaGetLastError();
}

// Tangents [io->jac_dir0, io->jac_dir0 + n_dirs) of t_q [n_q * m][ns] -> columns of the outputs (rows at (r * m + j) * ns + e,
// io->jac_n_in = m).  M must carry the 16-byte layout; gscratch: n_dirs * ceil(n / 32) blocks of x_total * 128 bytes.
extern "C" int tds_launch_kin_jvp(const DevModel* M, const StepIO* io, const TdsKinCall* kc, const double* t_q, int m, int n_dirs,
                                  char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  typedef tds::Dual<double> D;
  SimParams P;
  EnvParams E;
  memset(&P, 0, sizeof(P));
  memset(&E, 0, sizeof(E));
  const dim3 grid((io->n + 31) / 32, n_dirs);
  KinArgJvp a;
  static_cast<KinArg&>(a) = kin_arg(kc);
  a.jv = JvpTan{t_q, nullptr, m};
  tds_stepw_kernel<D, D, D, D, false, false, true, false, true><<<grid, 32, 0, stream>>>(*M, P, E, *io, MODE_NOCONTACT, 0, gscratch, a);
  return (int)cudaGetLastError();
}
