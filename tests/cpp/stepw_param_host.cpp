// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
//
// The instances of the product's generic step kernel, tiny-differentiable-simulator_b200/csrc/tds_stepw.cu, that read per-environment
// physical parameters (template flag PAR), compiled FOR THE HOST with the same single-lane meanings of the CUDA built-ins as
// tests/cpp/stepw_host.cpp, and called lane after lane as tds_launch_stepw{,_jacobian,_vjp} launch them on the GPU with a ParMap.
// The CPU test-suite checks them against the instances without parameters (tests/cpp/stepw_host.cpp, stepw_vjp_host.cpp) on
// edited flat models, against central differences and against the C oracle.  Nothing outside tests/ builds or loads it.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/stepw_param_host.cpp -o tests/cpp/_stepw_param_host.so
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
// params / env arrays -> SimParams / EnvParams (as tds_b200_set_params / set_env / set_contact_model)
void set_params_env(const DevModel& Dm, const double* params, const double* env, SimParams& P, EnvParams& E) {
  memset(&P, 0, sizeof(P));
  memset(&E, 0, sizeof(E));
  P.dt = params[0]; P.inv_dt = 1.0 / params[0];
  for (int k = 0; k < 3; ++k) P.gravity[k] = params[1 + k];
  P.friction = params[4]; P.restitution = params[5]; P.erp = params[6]; P.cfm = params[7];
  P.pgs_iterations = (int)params[8]; P.keep_all_points = (int)params[9];
  P.contact_model = (int)params[10]; P.spring_k = params[11]; P.damper_d = params[12]; P.exponent_n = params[13];
  P.v_transition = params[14]; P.hard_contact_condition = (int)params[15];
  if (env) {
    E.n_act = (int)env[0]; E.start_link = (int)env[1];
    E.kp = (float)env[2]; E.kd = (float)env[3]; E.max_force = (float)env[4]; E.action_limit = (float)env[5];
    int k = 0;
    for (int i = Dm.floating ? 0 : E.start_link; i < Dm.n_links && k < E.n_act; ++i) {
      if (Dm.flags[i] & TDS_LF_FIXED) continue;
      E.act_link[k] = i; E.initial_poses[k] = (float)env[6 + k]; ++k;
    }
  }
}

template <typename RA, typename RC, typename RS, typename RQ>
void run_grid(const DevModel& M, const SimParams& P, const EnvParams& E, const StepIO& io, int mode, int use_pd, int n_dirs, char* scratch,
              const ParMap& pm) {
  const int warps = (io.n + 31) / 32;
  emu_blockDim = {32, 1, 1};
  emu_gridDim = {(unsigned)warps, (unsigned)n_dirs, 1};
  for (unsigned by = 0; by < (unsigned)n_dirs; ++by)
    for (unsigned bx = 0; bx < (unsigned)warps; ++bx)
      for (unsigned t = 0; t < 32; ++t) {
        if ((int)(bx * 32 + t) >= io.n) continue;
        emu_blockIdx = {bx, by, 0};
        emu_threadIdx = {t, 0, 0};
        tdsw::tds_stepw_kernel<RA, RC, RS, RQ, false, true>(M, P, E, io, mode, use_pd, scratch, pm);
      }
}
}  // namespace

extern "C" {

int tdsemu_param_count(const double* model, int n_model) {
  DevModel* D = new DevModel;
  int rc = tds_build_dev_model(model, n_model, D);
  if (!rc) rc = tds_param_count(D);
  delete D;
  return rc;
}

// One step of every environment with k installed parameters ids[k], values [n][k], through the PAR instances:
//   what 0: forward, precision 0 mixed / 1 fp64 / 2 fp32 -> q_out, qd_out, qdd_out [n][dim]
//   what 1: dual numbers, directions = the k parameters -> jac [n][rows][k]
//   what 2: dual numbers, directions = the inputs (as tdsemu_stepw's Jacobian) -> jac [n][rows][cols]
//   what 3: taping scalar: g_out [n][rows] -> g_in [n][cols], g_par [n][k]; tape_cap: starting capacity (regrown on overflow);
//           stats [n + 2]: recorded nodes per lane, final capacity, reruns
// Other arguments as tdsemu_stepw (tests/cpp/stepw_host.cpp).  Returns rows * 1000 + cols, or < 0 (-100: rejected ids).
int tdsemu_stepw_par(const double* model, int n_model, const double* params, const double* env, int what, int precision, int mode,
                     int use_pd, int n, const double* q, const double* qd, const double* tau, int k, const int* ids, const double* values,
                     double* q_out, double* qd_out, double* qdd_out, double* jac, const double* g_out, double* g_in, double* g_par,
                     int tape_cap, double* stats) {
  DevModel* D = new DevModel;
  int rc = tds_build_dev_model(model, n_model, D);
  if (rc) { delete D; return rc; }
  ParMap pm;
  const char* err = nullptr;
  if (tds_build_par_map(D, k, ids, &pm, &err)) { delete D; return -100; }   // (values / grad pointers are set below)
  const int sizes[3][3] = {{4, 8, 4}, {8, 8, 8}, {4, 4, 4}};
  if (what == 0) tds_build_layout_w(D, sizes[precision][0], sizes[precision][1], sizes[precision][2], -1);
  else tds_build_layout_w(D, 16, 16, 16, -1, 16);
  SimParams P;
  EnvParams E;
  set_params_env(*D, params, env, P, E);
  const int ns = (n + 31) & ~31, n_q = D->n_q, n_qd = D->n_qd;
  const int n_tau = n_qd - (D->floating ? 6 : 0), n_in = use_pd ? E.n_act : n_tau;
  std::vector<float> sq((size_t)(n_q > 0 ? n_q : 1) * ns), sqd((size_t)(n_qd > 0 ? n_qd : 1) * ns), st((size_t)(n_in > 0 ? n_in : 1) * ns, 0.f);
  std::vector<float> oq(sq.size()), oqd(sqd.size()), oqdd(sqd.size());
  std::vector<double> par((size_t)(k > 0 ? k : 1) * ns, 0.0);
  for (int e = 0; e < n; ++e) {
    for (int j = 0; j < n_q; ++j) sq[(size_t)j * ns + e] = (float)q[(size_t)e * n_q + j];
    for (int j = 0; j < n_qd; ++j) sqd[(size_t)j * ns + e] = (float)qd[(size_t)e * n_qd + j];
    if (tau) for (int j = 0; j < n_in; ++j) st[(size_t)j * ns + e] = (float)tau[(size_t)e * n_in + j];
    for (int j = 0; j < k; ++j) par[(size_t)j * ns + e] = values[(size_t)e * k + j];
  }
  const int rows = mode == 0 ? n_qd : n_q + n_qd, cols = n_q + n_qd + (use_pd ? E.n_act + 3 : n_tau);
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = sq.data(); io.qd_in = sqd.data(); io.tau_in = (tau || use_pd) ? st.data() : nullptr;
  io.q_out = oq.data(); io.qd_out = oqd.data(); io.qdd_out = oqdd.data();
  io.n = n; io.n_stride = ns;
  pm.values = par.data();
  typedef tds::Dual<double> DD;
  typedef tds::Tape<double> TT;
  if (what == 0) {
    std::vector<char> scratch((size_t)((n + 31) / 32) * D->x_total * 32 * 4 + 64);
    if (precision == 0) run_grid<float, double, float, float>(*D, P, E, io, mode, use_pd, 1, scratch.data(), pm);
    else if (precision == 1) run_grid<double, double, double, float>(*D, P, E, io, mode, use_pd, 1, scratch.data(), pm);
    else run_grid<float, float, float, float>(*D, P, E, io, mode, use_pd, 1, scratch.data(), pm);
    for (int e = 0; e < n; ++e) {
      if (q_out) for (int j = 0; j < n_q; ++j) q_out[(size_t)e * n_q + j] = oq[(size_t)j * ns + e];
      if (qd_out) for (int j = 0; j < n_qd; ++j) qd_out[(size_t)e * n_qd + j] = oqd[(size_t)j * ns + e];
      if (qdd_out) for (int j = 0; j < n_qd; ++j) qdd_out[(size_t)e * n_qd + j] = oqdd[(size_t)j * ns + e];
    }
  } else if (what == 1 || what == 2) {
    const int n_dirs = what == 1 ? k : cols;
    std::vector<double> jbuf((size_t)rows * (n_dirs > 0 ? n_dirs : 1) * ns, 0.0);
    io.jac = jbuf.data(); io.jac_n_in = n_dirs; io.jac_dir0 = what == 1 ? cols : 0;
    std::vector<char> scratch((size_t)(n_dirs > 0 ? n_dirs : 1) * ((n + 31) / 32) * D->x_total * 32 * 4 + 64);
    if (n_dirs > 0) run_grid<DD, DD, DD, DD>(*D, P, E, io, mode, use_pd, n_dirs, scratch.data(), pm);
    for (int e = 0; e < n; ++e)
      for (int j = 0; j < rows * n_dirs; ++j) jac[(size_t)e * rows * n_dirs + j] = jbuf[(size_t)j * ns + e];
  } else {
    std::vector<double> go((size_t)rows * ns, 0.0), gi((size_t)cols * ns, 0.0), gp((size_t)(k > 0 ? k : 1) * ns, 0.0);
    for (int e = 0; e < n; ++e) for (int j = 0; j < rows; ++j) go[(size_t)j * ns + e] = g_out[(size_t)e * rows + j];
    io.g_out = go.data(); io.g_in = g_in ? gi.data() : nullptr; pm.grad = gp.data();
    const int warps = (n + 31) / 32;
    std::vector<char> scratch((size_t)warps * D->x_total * 32 * 4 + 64);
    std::vector<tds::TapeNode> tape;
    std::vector<double> adj, len(n, 0.0);
    int overflow = 0, reruns = -1;
    do {
      if (overflow) tape_cap *= 2;
      overflow = 0; ++reruns;
      tape.assign((size_t)warps * tape_cap * 32, tds::TapeNode{});
      adj.assign((size_t)warps * tape_cap * 32, 0.0);
      io.tape = tape.data(); io.tape_adj = adj.data(); io.tape_cap = tape_cap; io.tape_overflow = &overflow;
      emu_blockDim = {32, 1, 1};
      emu_gridDim = {(unsigned)warps, 1, 1};
      for (unsigned bx = 0; bx < (unsigned)warps; ++bx)
        for (unsigned t = 0; t < 32; ++t) {
          if ((int)(bx * 32 + t) >= n) continue;
          emu_blockIdx = {bx, 0, 0};
          emu_threadIdx = {t, 0, 0};
          tdsw::tds_stepw_kernel<TT, TT, TT, TT, false, true>(*D, P, E, io, mode, use_pd, scratch.data(), pm);
          len[bx * 32 + t] = tds::tape_length();
        }
    } while (overflow);
    for (int e = 0; e < n; ++e) {
      if (g_in) for (int j = 0; j < cols; ++j) g_in[(size_t)e * cols + j] = gi[(size_t)j * ns + e];
      for (int j = 0; j < k; ++j) g_par[(size_t)e * k + j] = gp[(size_t)j * ns + e];
    }
    if (stats) {
      for (int e = 0; e < n; ++e) stats[e] = len[e];
      stats[n] = tape_cap; stats[n + 1] = reruns;
    }
  }
  delete D;
  return rows * 1000 + cols;
}

}  // extern "C"
