// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
//
// The regressor instances of the product's generic step kernel, tiny-differentiable-simulator_b200/csrc/tds_stepw.cu (template flags INV
// and REG: fp64 values and the tangent-seeded dual numbers), compiled FOR THE HOST with the same single-lane meanings of the CUDA built-ins
// as tests/cpp/mass_host.cpp, and called lane after lane as tds_launch_regressor / tds_launch_regressor_jvp (csrc/tds_regressor.cu) launch
// them on the GPU.  The vector-Jacobian product is restated as the C-ABI computes it: the JVP along the identity tangents of q | qd | qdd,
// contracted with the cotangent over the concatenated rows Y | yT | yV in the order of the rows.  Nothing outside tests/ builds or loads it.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/regressor_host.cpp -o tests/cpp/_regressor_host.so
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
template <typename R, bool JV, typename RA>
void run_grid(const DevModel& M, const SimParams& P, const StepIO& io, int n_dirs, char* scratch, const RA& ra) {
  EnvParams E;
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
        tdsw::tds_stepw_kernel<R, R, R, R, false, false, JV, false, false, true, false, false, false, false, true>(M, P, E, io,
                                                                                                                   tdsw::MODE_NOCONTACT, 0,
                                                                                                                   scratch, ra);
      }
}

struct Setup {
  DevModel D;
  SimParams P;
  int n, ns;
  std::vector<float> sq, sqd, sqdd;
  bool has_qd, has_qdd;
  size_t r_Y, r_pi;   // rows of Y, of yT (and of yV)
};

// q [n][n_q], qd and qdd [n][n_qd] (null: zero) rounded to fp32 in the device layouts
int setup(Setup& S, const double* model, int n_model, int n, const double* q, const double* qd, const double* qdd, const double* gravity,
          int size) {
  int rc = tds_build_dev_model(model, n_model, &S.D);
  if (rc) return rc;
  tds_build_layout_w(&S.D, size, size, size, -1, size);
  memset(&S.P, 0, sizeof(S.P));
  for (int c = 0; c < 3; ++c) S.P.gravity[c] = gravity[c];
  S.n = n; S.ns = (n + 31) & ~31;
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
  S.r_pi = (size_t)12 * S.D.n_links + 10;
  S.r_Y = (size_t)nd * S.r_pi;
  return 0;
}

StepIO io_of(const Setup& S, int m, double* jac) {
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = S.sq.data(); io.qd_in = S.has_qd ? S.sqd.data() : nullptr; io.tau_in = S.has_qdd ? S.sqdd.data() : nullptr;
  io.jac = jac; io.n = S.n; io.n_stride = S.ns; io.jac_n_in = m; io.jac_dir0 = 0;
  return io;
}

// outputs [rows * m][ns] (concatenated Y | yT | yV) along tin [(n_q + 2 n_qd) * m][ns] (device layouts)
void jvp_soa(Setup& S, int m, const double* tin, double* out) {
  const StepIO io = io_of(S, m, out);
  std::vector<char> scratch((size_t)m * ((S.n + 31) / 32) * S.D.x_total * 32 * 4 + 64);
  tdsw::RegArg<tdsw::NoParJvp> a;
  memset(&a, 0, sizeof(a));
  a.jv = tdsw::JvpTan{tin, nullptr, m};
  a.yT = out + S.r_Y * m * S.ns; a.yV = a.yT + S.r_pi * m * S.ns;
  run_grid<tds::Dual<double>, true>(S.D, S.P, io, m, scratch.data(), a);
}

void to_aos(const Setup& S, const double* soa, size_t rows, double* dst) {
  for (int e = 0; e < S.n; ++e)
    for (size_t r = 0; r < rows; ++r) dst[(size_t)e * rows + r] = soa[r * S.ns + e];
}
}  // namespace

extern "C" {

// Y [n][n_qd * n_pi], yT [n][n_pi], yV [n][n_pi] (each may be null) at q [n][n_q], qd and qdd [n][n_qd] (null: zero; all rounded to fp32)
// under gravity[3].  The device buffers start filled with `fill`, so that an entry the kernel leaves unwritten shows.  Returns 0, or < 0.
int tdsemu_regressor(const double* model, int n_model, int n, const double* q, const double* qd, const double* qdd, const double* gravity,
                     double fill, double* Y, double* yT, double* yV) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, qd, qdd, gravity, 8);
  if (rc) { delete S; return rc; }
  const int ns = S->ns;
  std::vector<double> oY(S->r_Y * ns + 1, fill), oT(S->r_pi * ns + 1, fill), oV(S->r_pi * ns + 1, fill);
  tdsw::RegArg<tdsw::NoPar> a;
  a.yT = yT ? oT.data() : nullptr; a.yV = yV ? oV.data() : nullptr;
  const StepIO io = io_of(*S, 1, Y ? oY.data() : nullptr);
  std::vector<char> scratch((size_t)((n + 31) / 32) * S->D.x_total * 32 * 4 + 64);
  run_grid<double, false>(S->D, S->P, io, 1, scratch.data(), a);
  if (Y) to_aos(*S, oY.data(), S->r_Y, Y);
  if (yT) to_aos(*S, oT.data(), S->r_pi, yT);
  if (yV) to_aos(*S, oV.data(), S->r_pi, yV);
  delete S;
  return 0;
}

// d(Y | yT | yV) [n][rows][m] along t_in [n][n_q + 2 n_qd][m] (q | qd | qdd).  Other arguments as tdsemu_regressor.
int tdsemu_regressor_jvp(const double* model, int n_model, int n, const double* q, const double* qd, const double* qdd, const double* gravity,
                         int m, const double* t_in, double* out) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, qd, qdd, gravity, 16);
  if (rc) { delete S; return rc; }
  const int n_in = S->D.n_q + 2 * S->D.n_qd, ns = S->ns;
  const size_t rows = S->r_Y + 2 * S->r_pi;
  std::vector<double> ti((size_t)n_in * m * ns, 0.0), o(rows * m * ns + 1, 0.0);
  for (int e = 0; e < n; ++e)
    for (int c = 0; c < n_in * m; ++c) ti[(size_t)c * ns + e] = t_in[(size_t)e * n_in * m + c];
  jvp_soa(*S, m, ti.data(), o.data());
  to_aos(*S, o.data(), rows * m, out);
  delete S;
  return 0;
}

// g [n][n_q + 2 n_qd] = sum_r G[r] d(Y | yT | yV)[r] / d(q | qd | qdd) for the cotangent G [n][rows] over the concatenated rows, as
// tds_b200_regressor_vjp_* computes it (identity tangents, contraction in the order of r).
int tdsemu_regressor_vjp(const double* model, int n_model, int n, const double* q, const double* qd, const double* qdd, const double* gravity,
                         const double* G, double* g) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, qd, qdd, gravity, 16);
  if (rc) { delete S; return rc; }
  const int m = S->D.n_q + 2 * S->D.n_qd, ns = S->ns;
  const size_t rows = S->r_Y + 2 * S->r_pi;
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
