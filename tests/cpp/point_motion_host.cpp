// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
//
// The point-motion instances of the product's generic step kernel, tiny-differentiable-simulator_b200/csrc/tds_stepw.cu (template flag
// MOT: fp64 values and the tangent-seeded dual numbers), compiled FOR THE HOST with the same single-lane meanings of the CUDA built-ins as
// tests/cpp/mass_host.cpp, and called lane after lane as tds_launch_point_motion / tds_launch_point_motion_jvp (csrc/tds_point_motion.cu)
// launch them on the GPU.  The vector-Jacobian product is restated as the C-ABI computes it: the JVP along the identity tangents of
// q | qd | qdd, contracted with the cotangent over the concatenated rows J | vel | acc in the order of the rows.  Nothing outside tests/
// builds or loads it.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/point_motion_host.cpp -o tests/cpp/_point_motion_host.so
#include <cuda_runtime.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#define TDS_B200_EXACT_RCP 1
#define TDS_STEPW_KERNEL_ONLY 1
struct EmuDim { unsigned x, y, z; };
static thread_local EmuDim emu_threadIdx, emu_blockIdx, emu_blockDim, emu_gridDim;
#define threadIdx emu_threadIdx
#define blockIdx emu_blockIdx
#define blockDim emu_blockDim
#define gridDim emu_gridDim
#define __any_sync(mask, pred) ((pred) ? 1 : 0)
#define __reduce_max_sync(mask, v) (v)
static inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
#define __syncwarp() ((void)0)
#define clock64() (0LL)
#undef __shared__
#define __shared__
#undef __grid_constant__
#define __grid_constant__
#undef __global__
#define __global__
#undef __launch_bounds__
#define __launch_bounds__(...)
alignas(16) char smem_raw[16];

#include "tds_model.h"
#include "../../tiny-differentiable-simulator_b200/csrc/tds_stepw.cu"

namespace {
template <typename R, bool JV, typename MA>
void run_grid(const DevModel& M, const StepIO& io, int n_dirs, char* scratch, const MA& ma) {
  SimParams P;
  EnvParams E;
  memset(&P, 0, sizeof(P));
  memset(&E, 0, sizeof(E));
  const int warps = (io.n + 31) / 32;
  emu_blockDim = {32, 1, 1};
  emu_gridDim = {(unsigned)warps, (unsigned)n_dirs, 1};
  for (unsigned by = 0; by < (unsigned)n_dirs; ++by)
    for (unsigned bx = 0; bx < (unsigned)warps; ++bx)
      for (unsigned t = 0; t < 32; ++t) {
        if ((int)(bx * 32 + t) >= io.n) continue;
        emu_blockIdx = {bx, by, 0};
        emu_threadIdx = {t, 0, 0};
        tdsw::tds_stepw_kernel<R, R, R, R, false, false, JV, false, false, false, false, false, true>(M, P, E, io, tdsw::MODE_NOCONTACT, 0,
                                                                                                       scratch, ma);
      }
}

struct Setup {
  DevModel D;
  int n, ns, K;
  std::vector<float> sq, sqd, sqdd;
  bool has_qd, has_qdd;
  tdsw::MotArg<tdsw::KinArg> ma;
  size_t r_J, r_v;   // rows of J, of vel (and of acc)
};

// q [n][n_q], qd and qdd [n][n_qd] (null: zero) rounded to fp32 in the device layouts, and the point table
int setup(Setup& S, const double* model, int n_model, int n, const double* q, const double* qd, const double* qdd, int K, const int* links,
          const double* local, int size) {
  int rc = tds_build_dev_model(model, n_model, &S.D);
  if (rc) return rc;
  if (K < 0 || K > TDS_MAX_KIN_POINTS) return -101;
  tds_build_layout_w(&S.D, size, size, size, -1, size);
  S.n = n; S.ns = (n + 31) & ~31; S.K = K;
  S.has_qd = qd != nullptr; S.has_qdd = qdd != nullptr;
  const int n_q = S.D.n_q, nd = S.D.n_qd;
  S.sq.assign((size_t)(n_q > 0 ? n_q : 1) * S.ns, 0.f);
  S.sqd.assign((size_t)(nd > 0 ? nd : 1) * S.ns, 0.f);
  S.sqdd.assign((size_t)(nd > 0 ? nd : 1) * S.ns, 0.f);
  for (int e = 0; e < n; ++e) {
    for (int j = 0; j < n_q; ++j) S.sq[(size_t)j * S.ns + e] = (float)q[(size_t)e * n_q + j];
    if (qd) for (int j = 0; j < nd; ++j) S.sqd[(size_t)j * S.ns + e] = (float)qd[(size_t)e * nd + j];
    if (qdd) for (int j = 0; j < nd; ++j) S.sqdd[(size_t)j * S.ns + e] = (float)qdd[(size_t)e * nd + j];
  }
  memset(&S.ma, 0, sizeof(S.ma));
  S.ma.K = K;
  for (int k = 0; k < K; ++k) {
    if (links[k] < -1 || links[k] >= S.D.n_links) return -102;
    S.ma.link[k] = links[k];
    for (int c = 0; c < 3; ++c) S.ma.local[3 * k + c] = local[3 * k + c];
  }
  S.r_J = (size_t)6 * K * nd; S.r_v = (size_t)6 * K;
  return 0;
}

StepIO io_of(const Setup& S, int m) {
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = S.sq.data(); io.qd_in = S.has_qd ? S.sqd.data() : nullptr; io.tau_in = S.has_qdd ? S.sqdd.data() : nullptr;
  io.n = S.n; io.n_stride = S.ns; io.jac_n_in = m; io.jac_dir0 = 0;
  return io;
}

// outputs [rows * m][ns] (concatenated J | vel | acc) along tin [(n_q + 2 n_qd) * m][ns] (device layouts)
void jvp_soa(Setup& S, int m, const double* tin, double* out) {
  const StepIO io = io_of(S, m);
  std::vector<char> scratch((size_t)m * ((S.n + 31) / 32) * S.D.x_total * 32 * 4 + 64);
  tdsw::MotArg<tdsw::KinArgJvp> a;
  memset(&a, 0, sizeof(a));
  static_cast<tdsw::KinArg&>(a) = static_cast<const tdsw::KinArg&>(S.ma);
  a.J = out; a.vel = out + S.r_J * m * S.ns; a.acc = a.vel + S.r_v * m * S.ns;
  a.jv = tdsw::JvpTan{tin, nullptr, m};
  run_grid<tds::Dual<double>, true>(S.D, io, m, scratch.data(), a);
}

void to_aos(const Setup& S, const double* soa, size_t rows, double* dst) {
  for (int e = 0; e < S.n; ++e)
    for (size_t r = 0; r < rows; ++r) dst[(size_t)e * rows + r] = soa[r * S.ns + e];
}
}  // namespace

extern "C" {

// J [n][6K * n_qd], vel [n][6K], acc [n][6K] (each may be null) at q [n][n_q], qd and qdd [n][n_qd] (null: zero; all rounded to fp32)
// for the point table links [K], local [3K].  Returns 0, or < 0.
int tdsemu_point_motion(const double* model, int n_model, int n, const double* q, const double* qd, const double* qdd, int K, const int* links,
                        const double* local, double* J, double* vel, double* acc) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, qd, qdd, K, links, local, 8);
  if (rc) { delete S; return rc; }
  const int ns = S->ns;
  std::vector<double> oJ(S->r_J * ns + 1, 0.0), ov(S->r_v * ns + 1, 0.0), oa(S->r_v * ns + 1, 0.0);
  S->ma.J = J ? oJ.data() : nullptr; S->ma.vel = vel ? ov.data() : nullptr; S->ma.acc = acc ? oa.data() : nullptr;
  const StepIO io = io_of(*S, 1);
  std::vector<char> scratch((size_t)((n + 31) / 32) * S->D.x_total * 32 * 4 + 64);
  run_grid<double, false>(S->D, io, 1, scratch.data(), S->ma);
  if (J) to_aos(*S, oJ.data(), S->r_J, J);
  if (vel) to_aos(*S, ov.data(), S->r_v, vel);
  if (acc) to_aos(*S, oa.data(), S->r_v, acc);
  delete S;
  return 0;
}

// d(J | vel | acc) [n][rows][m] along t_in [n][n_q + 2 n_qd][m] (q | qd | qdd).  Other arguments as tdsemu_point_motion.
int tdsemu_point_motion_jvp(const double* model, int n_model, int n, const double* q, const double* qd, const double* qdd, int K,
                            const int* links, const double* local, int m, const double* t_in, double* out) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, qd, qdd, K, links, local, 16);
  if (rc) { delete S; return rc; }
  const int n_in = S->D.n_q + 2 * S->D.n_qd, ns = S->ns;
  const size_t rows = S->r_J + 2 * S->r_v;
  std::vector<double> ti((size_t)n_in * m * ns, 0.0), o(rows * m * ns + 1, 0.0);
  for (int e = 0; e < n; ++e)
    for (int c = 0; c < n_in * m; ++c) ti[(size_t)c * ns + e] = t_in[(size_t)e * n_in * m + c];
  jvp_soa(*S, m, ti.data(), o.data());
  to_aos(*S, o.data(), rows * m, out);
  delete S;
  return 0;
}

// g [n][n_q + 2 n_qd] = sum_r G[r] d(J | vel | acc)[r] / d(q | qd | qdd) for the cotangent G [n][rows] over the concatenated rows, as
// tds_b200_point_motion_vjp_* computes it (identity tangents, contraction in the order of r).
int tdsemu_point_motion_vjp(const double* model, int n_model, int n, const double* q, const double* qd, const double* qdd, int K,
                            const int* links, const double* local, const double* G, double* g) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, qd, qdd, K, links, local, 16);
  if (rc) { delete S; return rc; }
  const int m = S->D.n_q + 2 * S->D.n_qd, ns = S->ns;
  const size_t rows = S->r_J + 2 * S->r_v;
  std::vector<double> ti((size_t)m * m * ns, 0.0), o(rows * m * ns + 1, 0.0);
  for (int e = 0; e < ns; ++e)
    for (int c = 0; c < m; ++c) ti[((size_t)c * m + c) * ns + e] = 1.0;
  jvp_soa(*S, m, ti.data(), o.data());
  for (int e = 0; e < n; ++e)
    for (int j = 0; j < m; ++j) {
      double acc = 0.0;
      for (size_t r = 0; r < rows; ++r) acc += G[(size_t)e * rows + r] * o[(r * m + j) * ns + e];
      g[(size_t)e * m + j] = acc;
    }
  delete S;
  return 0;
}

}  // extern "C"
