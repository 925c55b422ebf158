// Launchers of the world-frame kernel's point-motion instances (tds_stepw.cu, template flag MOT; DESIGN.md section 7.17): spatial point
// Jacobians, point velocities and point accelerations J qdd + J' qd of a point table from q, qd and qdd, in fp64 and as tangent-seeded
// dual numbers.  A translation unit of their own for the reason tds_stepw_par.cu gives: the instances in the other units keep their code.
// The vector-Jacobian product reuses the mass matrix's two helper kernels (tds_mass.cu).
#include <cuda_runtime.h>

#define TDS_STEPW_KERNEL_ONLY 1
#include "tds_stepw.cu"

// (the MOT lanes run in MODE_NOCONTACT without PD and without gravity: no contact detection; installed parameters do not enter)

template <typename B> static tdsw::MotArg<B> mot_arg(const TdsMotCall* mc) {
  tdsw::MotArg<B> a;
  memset(&a, 0, sizeof(a));
  a.J = mc->J; a.vel = mc->vel; a.acc = mc->acc;
  a.K = mc->K;
  for (int k = 0; k < mc->K; ++k) {
    a.link[k] = mc->link[k];
    for (int c = 0; c < 3; ++c) a.local[3 * k + c] = mc->local[3 * k + c];
  }
  return a;
}

// fp64 outputs from io->q_in, io->qd_in and io->tau_in = qdd (either of the last two may be null: zero), rows at r * ns + e.  M must carry
// the 8-byte layout (tds_build_layout_w(..., 8, 8, 8, -1, 8)); gscratch: ceil(n / 32) blocks of x_total * 128 bytes.
extern "C" int tds_launch_point_motion(const DevModel* M, const StepIO* io, const TdsMotCall* mc, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  SimParams P;
  EnvParams E;
  memset(&P, 0, sizeof(P));
  memset(&E, 0, sizeof(E));
  const dim3 grid((io->n + 31) / 32, 1);
  tds_stepw_kernel<double, double, double, double, false, false, false, false, false, false, false, false, true><<<grid, 32, 0, stream>>>(
      *M, P, E, *io, MODE_NOCONTACT, 0, gscratch, mot_arg<KinArg>(mc));
  return (int)cudaGetLastError();
}

// Tangents [io->jac_dir0, io->jac_dir0 + n_dirs) of t_in [(n_q + 2 n_qd) * m][ns] (q | qd | qdd) -> columns of the outputs (rows at
// (r * m + j) * ns + e, io->jac_n_in = m).  M must carry the 16-byte layout; gscratch: n_dirs * ceil(n / 32) blocks of x_total * 128
// bytes.
extern "C" int tds_launch_point_motion_jvp(const DevModel* M, const StepIO* io, const TdsMotCall* mc, const double* t_in, int m, int n_dirs,
                                           char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  typedef tds::Dual<double> D;
  SimParams P;
  EnvParams E;
  memset(&P, 0, sizeof(P));
  memset(&E, 0, sizeof(E));
  const dim3 grid((io->n + 31) / 32, n_dirs);
  MotArg<KinArgJvp> a = mot_arg<KinArgJvp>(mc);
  a.jv = JvpTan{t_in, nullptr, m};
  tds_stepw_kernel<D, D, D, D, false, false, true, false, false, false, false, false, true><<<grid, 32, 0, stream>>>(*M, P, E, *io,
                                                                                                                   MODE_NOCONTACT, 0, gscratch, a);
  return (int)cudaGetLastError();
}
