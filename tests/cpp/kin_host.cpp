// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
//
// The kinematics instances of the product's generic step kernel, tiny-differentiable-simulator_b200/csrc/tds_stepw.cu (template flag
// KIN: fp64 forward and the tangent-seeded dual numbers), compiled FOR THE HOST with the same single-lane meanings of the CUDA built-ins
// as tests/cpp/mass_host.cpp, and called lane after lane as tds_launch_kin / tds_launch_kin_jvp (csrc/tds_kin.cu) launch them on the
// GPU.  The vector-Jacobian product is restated as the C-ABI computes it: the JVP along the identity tangents of q, contracted with the
// cotangent over the concatenated rows xf | x | J in the order of the rows.  Nothing outside tests/ builds or loads it.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/kin_host.cpp -o tests/cpp/_kin_host.so
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
template <typename R, bool JV, typename KA>
void run_grid(const DevModel& M, const StepIO& io, int n_dirs, char* scratch, const KA& ka) {
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
        tdsw::tds_stepw_kernel<R, R, R, R, false, false, JV, false, true>(M, P, E, io, tdsw::MODE_NOCONTACT, 0, scratch, ka);
      }
}

struct Setup {
  DevModel D;
  int n, ns, K;
  std::vector<float> sq;
  tdsw::KinArg ka;
  size_t r_xf, r_x, r_J;   // rows of the three outputs
};

int setup(Setup& S, const double* model, int n_model, int n, const double* q, int K, const int* links, const double* local, int size) {
  int rc = tds_build_dev_model(model, n_model, &S.D);
  if (rc) return rc;
  if (K < 0 || K > TDS_MAX_KIN_POINTS) return -101;
  tds_build_layout_w(&S.D, size, size, size, -1, size);
  S.n = n; S.ns = (n + 31) & ~31; S.K = K;
  const int n_q = S.D.n_q;
  S.sq.assign((size_t)(n_q > 0 ? n_q : 1) * S.ns, 0.f);
  for (int e = 0; e < n; ++e)
    for (int j = 0; j < n_q; ++j) S.sq[(size_t)j * S.ns + e] = (float)q[(size_t)e * n_q + j];
  memset(&S.ka, 0, sizeof(S.ka));
  S.ka.K = K;
  for (int k = 0; k < K; ++k) {
    if (links[k] < -1 || links[k] >= S.D.n_links) return -102;
    S.ka.link[k] = links[k];
    for (int c = 0; c < 3; ++c) S.ka.local[3 * k + c] = local[3 * k + c];
  }
  S.r_xf = (size_t)S.D.n_links * 12; S.r_x = (size_t)3 * K; S.r_J = (size_t)3 * K * S.D.n_qd;
  return 0;
}

// outputs [rows * m][ns] (concatenated xf | x | J) along tq [n_q * m][ns] (device layouts)
void jvp_soa(Setup& S, int m, const double* tq, double* out) {
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = S.sq.data(); io.n = S.n; io.n_stride = S.ns;
  io.jac_n_in = m; io.jac_dir0 = 0;
  std::vector<char> scratch((size_t)m * ((S.n + 31) / 32) * S.D.x_total * 32 * 4 + 64);
  tdsw::KinArgJvp a;
  static_cast<tdsw::KinArg&>(a) = S.ka;
  a.xf = out; a.x = out + S.r_xf * m * S.ns; a.J = a.x + S.r_x * m * S.ns;
  a.jv = tdsw::JvpTan{tq, nullptr, m};
  run_grid<tds::Dual<double>, true>(S.D, io, m, scratch.data(), a);
}

void to_aos(const Setup& S, const double* soa, size_t rows, double* dst) {
  for (int e = 0; e < S.n; ++e)
    for (size_t r = 0; r < rows; ++r) dst[(size_t)e * rows + r] = soa[r * S.ns + e];
}
}  // namespace

extern "C" {

// xf [n][n_links * 12], x [n][3K], J [n][3K * n_qd] (each may be null) at q [n][n_q] (rounded to fp32) for the point table links [K],
// local [3K].  Returns 0, or < 0.
int tdsemu_kin(const double* model, int n_model, int n, const double* q, int K, const int* links, const double* local, double* xf,
               double* x, double* J) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, K, links, local, 8);
  if (rc) { delete S; return rc; }
  const int ns = S->ns;
  std::vector<double> oxf(S->r_xf * ns + 1, 0.0), ox(S->r_x * ns + 1, 0.0), oJ(S->r_J * ns + 1, 0.0);
  S->ka.xf = xf ? oxf.data() : nullptr; S->ka.x = x ? ox.data() : nullptr; S->ka.J = J ? oJ.data() : nullptr;
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = S->sq.data(); io.n = n; io.n_stride = ns; io.jac_n_in = 1;
  std::vector<char> scratch((size_t)((n + 31) / 32) * S->D.x_total * 32 * 4 + 64);
  run_grid<double, false>(S->D, io, 1, scratch.data(), S->ka);
  if (xf) to_aos(*S, oxf.data(), S->r_xf, xf);
  if (x) to_aos(*S, ox.data(), S->r_x, x);
  if (J) to_aos(*S, oJ.data(), S->r_J, J);
  delete S;
  return 0;
}

// d(xf | x | J) [n][rows][m] along t_q [n][n_q][m].  Other arguments as tdsemu_kin.
int tdsemu_kin_jvp(const double* model, int n_model, int n, const double* q, int K, const int* links, const double* local, int m,
                   const double* t_q, double* out) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, K, links, local, 16);
  if (rc) { delete S; return rc; }
  const int n_q = S->D.n_q, ns = S->ns;
  const size_t rows = S->r_xf + S->r_x + S->r_J;
  std::vector<double> tq((size_t)(n_q > 0 ? n_q : 1) * m * ns, 0.0), o(rows * m * ns + 1, 0.0);
  for (int e = 0; e < n; ++e)
    for (int c = 0; c < n_q * m; ++c) tq[(size_t)c * ns + e] = t_q[(size_t)e * n_q * m + c];
  jvp_soa(*S, m, tq.data(), o.data());
  to_aos(*S, o.data(), rows * m, out);
  delete S;
  return 0;
}

// g_q [n][n_q] = sum_r G[r] d(xf | x | J)[r] / dq for the cotangent G [n][rows] over the concatenated rows, as
// tds_b200_kinematics_vjp_* computes it (identity tangents, contraction in the order of r).
int tdsemu_kin_vjp(const double* model, int n_model, int n, const double* q, int K, const int* links, const double* local, const double* G,
                   double* g_q) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, K, links, local, 16);
  if (rc) { delete S; return rc; }
  const int n_q = S->D.n_q, ns = S->ns, m = n_q;
  const size_t rows = S->r_xf + S->r_x + S->r_J;
  std::vector<double> tq((size_t)(n_q > 0 ? n_q : 1) * (m > 0 ? m : 1) * ns, 0.0), o(rows * (m > 0 ? m : 1) * ns + 1, 0.0);
  for (int e = 0; e < ns; ++e)
    for (int c = 0; c < n_q; ++c) tq[((size_t)c * m + c) * ns + e] = 1.0;
  if (m > 0) jvp_soa(*S, m, tq.data(), o.data());
  for (int e = 0; e < n; ++e)
    for (int j = 0; j < m; ++j) {
      double acc = 0.0;
      for (size_t r = 0; r < rows; ++r) acc += G[(size_t)e * rows + r] * o[(r * m + j) * ns + e];
      g_q[(size_t)e * n_q + j] = acc;
    }
  delete S;
  return 0;
}

}  // extern "C"
