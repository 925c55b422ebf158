// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
//
// The external-wrench instances of the product's generic step kernel, tiny-differentiable-simulator_b200/csrc/tds_stepw.cu (template flag
// EXT: the three step precisions and the tangent-seeded dual numbers, with and without installed physical parameters), compiled FOR THE
// HOST with the same single-lane meanings of the CUDA built-ins as tests/cpp/stepw_host.cpp, and called lane after lane as
// tds_launch_wrench / tds_launch_wrench_jvp (csrc/tds_wrench.cu) launch them on the GPU, on the same grown layout (tds_ext_layout_w).
// Nothing outside tests/ builds or loads it.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/wrench_host.cpp -o tests/cpp/_wrench_host.so
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
template <typename RA, typename RC, typename RS, typename RQ, bool PAR, bool JV, typename PA>
void run_grid(const DevModel& M, const SimParams& P, const EnvParams& E, const StepIO& io, int mode, int use_pd, int n_dirs, char* scratch,
              const PA& pa) {
  const int warps = (io.n + 31) / 32;
  emu_blockDim = {32, 1, 1};
  emu_gridDim = {(unsigned)warps, (unsigned)n_dirs, 1};
  for (unsigned by = 0; by < (unsigned)n_dirs; ++by)
    for (unsigned bx = 0; bx < (unsigned)warps; ++bx)
      for (unsigned t = 0; t < 32; ++t) {
        if ((int)(bx * 32 + t) >= io.n) continue;
        emu_blockIdx = {bx, by, 0};
        emu_threadIdx = {t, 0, 0};
        tdsw::tds_stepw_kernel<RA, RC, RS, RQ, false, PAR, JV, false, false, false, false, false, false, true>(M, P, E, io, mode, use_pd,
                                                                                                               scratch, pa);
      }
}

// the kernel argument, as ext_arg of csrc/tds_wrench.cu builds it
template <typename B> tdsw::ExtArg<B> ext_arg(const B& b, int K, const int* links, const double* local, const float* W, const double* t_W,
                                              int x_ext) {
  tdsw::ExtArg<B> a;
  memset(&a, 0, sizeof(a));
  static_cast<B&>(a) = b;
  a.ext.x_ext = x_ext;
  a.ext.W = W; a.ext.t_W = t_W;
  a.ext.K = K;
  for (int k = 0; k < K; ++k) {
    a.ext.link[k] = links[k];
    if (links[k] >= 0) a.ext.links_with_points |= 1ull << links[k];
    for (int c = 0; c < 3; ++c) a.ext.local[3 * k + c] = local[3 * k + c];
  }
  return a;
}

template <typename RA, typename RC, typename RS>
void run_value(const DevModel& M, const SimParams& P, const EnvParams& E, const StepIO& io, int mode, int use_pd, char* scratch,
               const ParMap* pm, int K, const int* links, const double* local, const float* W, int x_ext) {
  if (pm) run_grid<RA, RC, RS, float, true, false>(M, P, E, io, mode, use_pd, 1, scratch, ext_arg(*pm, K, links, local, W, nullptr, x_ext));
  else run_grid<RA, RC, RS, float, false, false>(M, P, E, io, mode, use_pd, 1, scratch, ext_arg(tdsw::NoPar{}, K, links, local, W, nullptr, x_ext));
}
}  // namespace

extern "C" {

// params, env, precision, q, qd, tau: as tdsemu_stepw (tests/cpp/stepw_host.cpp); k installed parameters ids[k] at values [n][k] (k = 0:
// the instances without parameters); the point table K, links [K], local [3K] and the wrenches W [n][K][6] (rounded to fp32).  m = 0: the
// value instance of the precision -> q_out [n][n_q], qd_out [n][n_qd] (MODE_NOCONTACT, MODE_FULL) or qdd_out [n][n_qd] (MODE_FD), fp32
// values widened.  m > 0: the dual-number JVP instance along t_in [n][cols][m], t_W [n][K][6][m] and t_par [n][k][m] (each may be null) ->
// t_out [n][rows][m].  Returns 0, or < 0 (-100: rejected ids).
int tdsemu_wrench(const double* model, int n_model, const double* params, const double* env, int precision, int mode, int use_pd, int n,
                  const double* q, const double* qd, const double* tau, int k, const int* ids, const double* values, int K, const int* links,
                  const double* local, const double* W, double* q_out, double* qd_out, double* qdd_out, int m, const double* t_in,
                  const double* t_W, const double* t_par, double* t_out) {
  if (K < 0 || K > TDS_MAX_KIN_POINTS) return -1;
  DevModel* D = new DevModel;
  int rc = tds_build_dev_model(model, n_model, D);
  if (rc) { delete D; return rc; }
  const int sizes[3][3] = {{4, 8, 4}, {8, 8, 8}, {4, 4, 4}};
  if (m > 0) tds_build_layout_w(D, 16, 16, 16, -1, 16);
  else tds_build_layout_w(D, sizes[precision][0], sizes[precision][1], sizes[precision][2], -1);
  int x_total;
  const int x_ext = tds_ext_layout_w(D, m > 0 ? 16 : sizes[precision][0], &x_total);
  D->x_total = x_total;
  ParMap pm;
  const char* err = nullptr;
  if (tds_build_par_map(D, k, ids, &pm, &err)) { delete D; return -100; }
  SimParams P;
  memset(&P, 0, sizeof(P));
  P.dt = params[0]; P.inv_dt = 1.0 / params[0];
  for (int c = 0; c < 3; ++c) P.gravity[c] = params[1 + c];
  P.friction = params[4]; P.restitution = params[5]; P.erp = params[6]; P.cfm = params[7];
  P.pgs_iterations = (int)params[8]; P.keep_all_points = (int)params[9];
  P.contact_model = (int)params[10]; P.spring_k = params[11]; P.damper_d = params[12]; P.exponent_n = params[13];
  P.v_transition = params[14]; P.hard_contact_condition = (int)params[15];
  EnvParams E;
  memset(&E, 0, sizeof(E));
  if (env) {   // tds_b200_set_env (tds_capi.cu): action k drives the k-th non-fixed link at or after start_link
    E.n_act = (int)env[0]; E.start_link = (int)env[1];
    E.kp = (float)env[2]; E.kd = (float)env[3]; E.max_force = (float)env[4]; E.action_limit = (float)env[5];
    int a = 0;
    for (int i = D->floating ? 0 : E.start_link; i < D->n_links && a < E.n_act; ++i) {
      if (D->flags[i] & TDS_LF_FIXED) continue;
      E.act_link[a] = i; E.initial_poses[a] = (float)env[6 + a]; ++a;
    }
  }
  const int ns = (n + 31) & ~31, n_q = D->n_q, n_qd = D->n_qd;
  const int n_tau = n_qd - (D->floating ? 6 : 0), n_in = use_pd ? E.n_act : n_tau;
  const int cols = n_q + n_qd + (use_pd ? E.n_act + 3 : n_tau), rows = mode == 0 ? n_qd : n_q + n_qd;
  std::vector<float> sq((size_t)(n_q > 0 ? n_q : 1) * ns), sqd((size_t)(n_qd > 0 ? n_qd : 1) * ns), st((size_t)(n_in > 0 ? n_in : 1) * ns, 0.f);
  std::vector<float> oq(sq.size()), oqd(sqd.size()), oqdd(sqd.size()), sw((size_t)(6 * K + 1) * ns, 0.f);
  std::vector<double> par((size_t)(k > 0 ? k : 1) * ns, 0.0);
  for (int e = 0; e < n; ++e) {
    for (int j = 0; j < n_q; ++j) sq[(size_t)j * ns + e] = (float)q[(size_t)e * n_q + j];
    for (int j = 0; j < n_qd; ++j) sqd[(size_t)j * ns + e] = (float)qd[(size_t)e * n_qd + j];
    if (tau) for (int j = 0; j < n_in; ++j) st[(size_t)j * ns + e] = (float)tau[(size_t)e * n_in + j];
    for (int j = 0; j < k; ++j) par[(size_t)j * ns + e] = values[(size_t)e * k + j];
    for (int r = 0; r < 6 * K; ++r) sw[(size_t)r * ns + e] = (float)W[(size_t)e * 6 * K + r];
  }
  pm.values = par.data(); pm.grad = nullptr;
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = sq.data(); io.qd_in = sqd.data(); io.tau_in = (tau || use_pd) ? st.data() : nullptr;
  io.q_out = oq.data(); io.qd_out = oqd.data(); io.qdd_out = oqdd.data();
  io.n = n; io.n_stride = ns;
  const int n_dirs = m > 0 ? m : 1;
  std::vector<char> scratch((size_t)n_dirs * ((n + 31) / 32) * D->x_total * 32 * 4 + 64);
  if (m == 0) {
    const ParMap* pp = k > 0 ? &pm : nullptr;
    if (precision == 0) run_value<float, double, float>(*D, P, E, io, mode, use_pd, scratch.data(), pp, K, links, local, sw.data(), x_ext);
    else if (precision == 1) run_value<double, double, double>(*D, P, E, io, mode, use_pd, scratch.data(), pp, K, links, local, sw.data(), x_ext);
    else run_value<float, float, float>(*D, P, E, io, mode, use_pd, scratch.data(), pp, K, links, local, sw.data(), x_ext);
    for (int e = 0; e < n; ++e) {
      for (int j = 0; j < n_q; ++j) q_out[(size_t)e * n_q + j] = oq[(size_t)j * ns + e];
      for (int j = 0; j < n_qd; ++j) qd_out[(size_t)e * n_qd + j] = oqd[(size_t)j * ns + e];
      for (int j = 0; j < n_qd; ++j) qdd_out[(size_t)e * n_qd + j] = oqdd[(size_t)j * ns + e];
    }
  } else {
    std::vector<double> ti((size_t)cols * m * ns, 0.0), tw((size_t)(6 * K + 1) * m * ns, 0.0), tp((size_t)(k > 0 ? k : 1) * m * ns, 0.0),
        out((size_t)rows * m * ns, 0.0);
    for (int e = 0; e < n; ++e) {
      if (t_in) for (int c = 0; c < cols * m; ++c) ti[(size_t)c * ns + e] = t_in[(size_t)e * cols * m + c];
      if (t_W) for (int c = 0; c < 6 * K * m; ++c) tw[(size_t)c * ns + e] = t_W[(size_t)e * 6 * K * m + c];
      if (t_par) for (int c = 0; c < k * m; ++c) tp[(size_t)c * ns + e] = t_par[(size_t)e * k * m + c];
    }
    io.jac = out.data(); io.jac_n_in = m; io.jac_dir0 = 0;
    const tdsw::JvpTan jv{t_in ? ti.data() : nullptr, t_par ? tp.data() : nullptr, m};
    const double* twp = t_W ? tw.data() : nullptr;
    typedef tds::Dual<double> DD;
    if (k > 0) {
      tdsw::ParMapJvp a;
      static_cast<ParMap&>(a) = pm;
      a.jv = jv;
      run_grid<DD, DD, DD, DD, true, true>(*D, P, E, io, mode, use_pd, m, scratch.data(), ext_arg(a, K, links, local, sw.data(), twp, x_ext));
    } else {
      run_grid<DD, DD, DD, DD, false, true>(*D, P, E, io, mode, use_pd, m, scratch.data(),
                                            ext_arg(tdsw::NoParJvp{jv}, K, links, local, sw.data(), twp, x_ext));
    }
    for (int e = 0; e < n; ++e)
      for (int c = 0; c < rows * m; ++c) t_out[(size_t)e * rows * m + c] = out[(size_t)c * ns + e];
  }
  delete D;
  return 0;
}

}  // extern "C"
