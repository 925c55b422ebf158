// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
//
// The Coriolis-matrix instances of the product's generic step kernel, tiny-differentiable-simulator_b200/csrc/tds_stepw.cu (template flag
// COR: fp64 forward and the tangent-seeded dual numbers, with and without installed physical parameters), compiled FOR THE HOST with
// the same single-lane meanings of the CUDA built-ins as tests/cpp/mass_host.cpp, and called lane after lane as tds_launch_coriolis /
// tds_launch_coriolis_jvp (csrc/tds_coriolis.cu) launch them on the GPU.  The vector-Jacobian product is restated as the C-ABI computes
// it: the JVP along the identity tangents of q | qd | installed parameters, contracted with the cotangent in the order of the entries.
// Nothing outside tests/ builds or loads it.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/coriolis_host.cpp -o tests/cpp/_coriolis_host.so
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
template <typename R, bool PAR, bool JV, typename PA>
void run_grid(const DevModel& M, const StepIO& io, int n_dirs, char* scratch, const PA& pa) {
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
        tdsw::tds_stepw_kernel<R, R, R, R, false, PAR, JV, false, false, false, false, false, false, false, false, false, true>(
            M, P, E, io, tdsw::MODE_NOCONTACT, 0, scratch, pa);
      }
}

struct Setup {
  DevModel D;
  ParMap pm;
  int n, ns, k;
  bool has_qd;
  std::vector<float> sq, sqd;
  std::vector<double> par;
};

// qd may be null (zero)
int setup(Setup& S, const double* model, int n_model, int n, const double* q, const double* qd, int k, const int* ids, const double* values,
          int size) {
  int rc = tds_build_dev_model(model, n_model, &S.D);
  if (rc) return rc;
  const char* err = nullptr;
  if (tds_build_par_map(&S.D, k, ids, &S.pm, &err)) return -100;
  tds_build_layout_w(&S.D, size, size, size, -1, size);
  S.n = n; S.ns = (n + 31) & ~31; S.k = k; S.has_qd = qd != nullptr;
  const int n_q = S.D.n_q, nd = S.D.n_qd;
  S.sq.assign((size_t)(n_q > 0 ? n_q : 1) * S.ns, 0.f);
  S.sqd.assign((size_t)(nd > 0 ? nd : 1) * S.ns, 0.f);
  S.par.assign((size_t)(k > 0 ? k : 1) * S.ns, 0.0);
  for (int e = 0; e < n; ++e) {
    for (int j = 0; j < n_q; ++j) S.sq[(size_t)j * S.ns + e] = (float)q[(size_t)e * n_q + j];
    if (qd) for (int j = 0; j < nd; ++j) S.sqd[(size_t)j * S.ns + e] = (float)qd[(size_t)e * nd + j];
    for (int j = 0; j < k; ++j) S.par[(size_t)j * S.ns + e] = values[(size_t)e * k + j];
  }
  S.pm.values = S.par.data(); S.pm.grad = nullptr;
  return 0;
}

// dC [(nn * m)][ns] along the tangents ti [(n_q + n_qd) * m][ns] (q | qd), tp [k * m][ns] (device layouts)
void jvp_soa(const Setup& S, int m, const double* ti, const double* tp, double* dC) {
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = S.sq.data(); io.qd_in = S.has_qd ? S.sqd.data() : nullptr; io.n = S.n; io.n_stride = S.ns;
  io.jac = dC; io.jac_n_in = m; io.jac_dir0 = 0;
  std::vector<char> scratch((size_t)m * ((S.n + 31) / 32) * S.D.x_total * 32 * 4 + 64);
  const tdsw::JvpTan jv{ti, tp, m};
  if (S.k > 0) {
    tdsw::ParMapJvp a;
    static_cast<ParMap&>(a) = S.pm;
    a.jv = jv;
    run_grid<tds::Dual<double>, true, true>(S.D, io, m, scratch.data(), a);
  } else {
    run_grid<tds::Dual<double>, false, true>(S.D, io, m, scratch.data(), tdsw::NoParJvp{jv});
  }
}
}  // namespace

extern "C" {

// C [n][n_qd][n_qd] of every environment at q [n][n_q] and qd [n][n_qd] (rounded to fp32; qd null: zero), with k installed parameters
// ids[k] at values [n][k] (k = 0: the instance without parameters).  Returns 0, or < 0 (-100: rejected ids).
int tdsemu_coriolis(const double* model, int n_model, int n, const double* q, const double* qd, int k, const int* ids, const double* values,
                    double* C) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, qd, k, ids, values, 8);
  if (rc) { delete S; return rc; }
  const int nd = S->D.n_qd, nn = nd * nd, ns = S->ns;
  std::vector<double> out((size_t)(nn > 0 ? nn : 1) * ns, -1.0);   // (every entry is written)
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = S->sq.data(); io.qd_in = qd ? S->sqd.data() : nullptr; io.n = n; io.n_stride = ns; io.jac = out.data(); io.jac_n_in = 1;
  std::vector<char> scratch((size_t)((n + 31) / 32) * S->D.x_total * 32 * 4 + 64);
  if (k > 0) run_grid<double, true, false>(S->D, io, 1, scratch.data(), S->pm);
  else run_grid<double, false, false>(S->D, io, 1, scratch.data(), tdsw::NoPar{});
  for (int e = 0; e < n; ++e)
    for (int r = 0; r < nn; ++r) C[(size_t)e * nn + r] = out[(size_t)r * ns + e];
  delete S;
  return 0;
}

// dC [n][n_qd][n_qd][m] along t_q [n][n_q][m], t_qd [n][n_qd][m] and t_par [n][k][m] (each may be null).  Other arguments as
// tdsemu_coriolis.
int tdsemu_coriolis_jvp(const double* model, int n_model, int n, const double* q, const double* qd, int k, const int* ids, const double* values,
                        int m, const double* t_q, const double* t_qd, const double* t_par, double* dC) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, qd, k, ids, values, 16);
  if (rc) { delete S; return rc; }
  const int n_q = S->D.n_q, nd = S->D.n_qd, nn = nd * nd, ns = S->ns;
  std::vector<double> ti((size_t)(n_q + nd) * m * ns, 0.0), tp((size_t)(k > 0 ? k : 1) * m * ns, 0.0), out((size_t)nn * m * ns, -1.0);
  for (int e = 0; e < n; ++e) {
    if (t_q) for (int c = 0; c < n_q * m; ++c) ti[(size_t)c * ns + e] = t_q[(size_t)e * n_q * m + c];
    if (t_qd) for (int c = 0; c < nd * m; ++c) ti[((size_t)n_q * m + c) * ns + e] = t_qd[(size_t)e * nd * m + c];
    if (t_par) for (int c = 0; c < k * m; ++c) tp[(size_t)c * ns + e] = t_par[(size_t)e * k * m + c];
  }
  jvp_soa(*S, m, (t_q || t_qd) ? ti.data() : nullptr, t_par ? tp.data() : nullptr, out.data());
  for (int e = 0; e < n; ++e)
    for (int c = 0; c < nn * m; ++c) dC[(size_t)e * nn * m + c] = out[(size_t)c * ns + e];
  delete S;
  return 0;
}

// g [n][n_q + n_qd + k] = sum_r G[r] dC[r] / d(q | qd | installed parameters) for the cotangent G [n][n_qd][n_qd], as
// tds_b200_coriolis_vjp_* computes it (identity tangents, contraction in the order of r).
int tdsemu_coriolis_vjp(const double* model, int n_model, int n, const double* q, const double* qd, int k, const int* ids, const double* values,
                        const double* G, double* g) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, qd, k, ids, values, 16);
  if (rc) { delete S; return rc; }
  const int n_in = S->D.n_q + S->D.n_qd, nn = S->D.n_qd * S->D.n_qd, ns = S->ns, m = n_in + k;
  std::vector<double> ti((size_t)n_in * m * ns, 0.0), tp((size_t)(k > 0 ? k : 1) * m * ns, 0.0), out((size_t)nn * m * ns, 0.0);
  for (int e = 0; e < ns; ++e) {
    for (int c = 0; c < n_in; ++c) ti[((size_t)c * m + c) * ns + e] = 1.0;
    for (int s = 0; s < k; ++s) tp[((size_t)s * m + n_in + s) * ns + e] = 1.0;
  }
  jvp_soa(*S, m, ti.data(), k > 0 ? tp.data() : nullptr, out.data());
  for (int e = 0; e < n; ++e)
    for (int j = 0; j < m; ++j) {
      double acc = 0.0;
      for (int r = 0; r < nn; ++r) acc += G[(size_t)e * nn + r] * out[((size_t)r * m + j) * ns + e];
      g[(size_t)e * m + j] = acc;
    }
  delete S;
  return 0;
}

}  // extern "C"
