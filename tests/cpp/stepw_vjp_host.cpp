// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
//
// The reverse-mode (taping) instance of the product's generic step kernel, tiny-differentiable-simulator_b200/csrc/tds_stepw.cu,
// compiled FOR THE HOST with the same single-lane meanings of the CUDA built-ins as tests/cpp/stepw_host.cpp, and called lane after
// lane as tds_launch_stepw_vjp launches it on the GPU.  The CPU test-suite checks its vector-Jacobian products against the
// dual-number instance of the same source (tests/cpp/stepw_host.cpp) and against the C oracle.  Nothing outside tests/ builds or
// loads it.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/stepw_vjp_host.cpp -o tests/cpp/_stepw_vjp_host.so
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

// params / env arrays of the entry points below -> SimParams / EnvParams (as tds_b200_set_params / set_env / set_contact_model)
static void set_params_env(const DevModel& Dm, const double* params, const double* env, SimParams& P, EnvParams& E) {
  const DevModel* D = &Dm;
  memset(&P, 0, sizeof(P));
  memset(&E, 0, sizeof(E));
  P.dt = params[0]; P.inv_dt = 1.0 / params[0];
  for (int k = 0; k < 3; ++k) P.gravity[k] = params[1 + k];
  P.friction = params[4]; P.restitution = params[5]; P.erp = params[6]; P.cfm = params[7];
  P.pgs_iterations = (int)params[8]; P.keep_all_points = (int)params[9];
  P.contact_model = (int)params[10]; P.spring_k = params[11]; P.damper_d = params[12]; P.exponent_n = params[13];
  P.v_transition = params[14]; P.hard_contact_condition = (int)params[15];
  if (env) {   // tds_b200_set_env (tds_capi.cu): action k drives the k-th non-fixed link at or after start_link
    E.n_act = (int)env[0]; E.start_link = (int)env[1];
    E.kp = (float)env[2]; E.kd = (float)env[3]; E.max_force = (float)env[4]; E.action_limit = (float)env[5];
    int k = 0;
    for (int i = D->floating ? 0 : E.start_link; i < D->n_links && k < E.n_act; ++i) {
      if (D->flags[i] & TDS_LF_FIXED) continue;
      E.act_link[k] = i; E.initial_poses[k] = (float)env[6 + k]; ++k;
    }
  }
}

extern "C" {

// Vector-Jacobian product by the taping instance (Tape<double>, one lane per environment, as tds_launch_stepw_vjp launches it):
// g_out [n][rows] -> g_in [n][cols] (rows / columns as for the Jacobian of tdsemu_stepw, tests/cpp/stepw_host.cpp).  tape_cap: starting capacity in nodes per lane
// (test argument: a tape that overflows is rerun with twice the capacity, as the C-ABI does).  stats (or null): [n][1] recorded
// nodes per lane, then the final capacity and the number of reruns.  Returns rows * 1000 + cols.
int tdsemu_stepw_vjp(const double* model, int n_model, const double* params, const double* env, int mode, int use_pd, int n,
                     const double* q, const double* qd, const double* tau, const double* g_out, double* g_in, int tape_cap,
                     double* stats) {
  DevModel* D = new DevModel;
  int rc = tds_build_dev_model(model, n_model, D);
  if (rc) { delete D; return rc; }
  tds_build_layout_w(D, 16, 16, 16, -1, 16);
  SimParams P;
  EnvParams E;
  set_params_env(*D, params, env, P, E);
  const int ns = (n + 31) & ~31, n_q = D->n_q, n_qd = D->n_qd;
  const int n_tau = n_qd - (D->floating ? 6 : 0), n_in = use_pd ? E.n_act : n_tau;
  std::vector<float> sq((size_t)(n_q > 0 ? n_q : 1) * ns), sqd((size_t)(n_qd > 0 ? n_qd : 1) * ns), st((size_t)(n_in > 0 ? n_in : 1) * ns, 0.f);
  for (int e = 0; e < n; ++e) {
    for (int k = 0; k < n_q; ++k) sq[(size_t)k * ns + e] = (float)q[(size_t)e * n_q + k];
    for (int k = 0; k < n_qd; ++k) sqd[(size_t)k * ns + e] = (float)qd[(size_t)e * n_qd + k];
    if (tau) for (int k = 0; k < n_in; ++k) st[(size_t)k * ns + e] = (float)tau[(size_t)e * n_in + k];
  }
  const int rows = mode == 0 ? n_qd : n_q + n_qd, cols = n_q + n_qd + (use_pd ? E.n_act + 3 : n_tau);
  std::vector<double> go((size_t)rows * ns, 0.0), gi((size_t)cols * ns, 0.0);
  for (int e = 0; e < n; ++e) for (int k = 0; k < rows; ++k) go[(size_t)k * ns + e] = g_out[(size_t)e * rows + k];
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = sq.data(); io.qd_in = sqd.data(); io.tau_in = (tau || use_pd) ? st.data() : nullptr;
  io.n = n; io.n_stride = ns;
  io.g_out = go.data(); io.g_in = gi.data();
  const int warps = (n + 31) / 32;
  std::vector<char> scratch((size_t)warps * D->x_total * 32 * 4 + 64);
  std::vector<tds::TapeNode> tape;
  std::vector<double> adj;
  std::vector<double> len(n, 0.0);
  int overflow = 0, reruns = -1;
  typedef tds::Tape<double> TT;
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
        tdsw::tds_stepw_kernel<TT, TT, TT, TT, false>(*D, P, E, io, mode, use_pd, scratch.data());
        len[bx * 32 + t] = tds::tape_length();
      }
  } while (overflow);
  for (int e = 0; e < n; ++e) for (int k = 0; k < cols; ++k) g_in[(size_t)e * cols + k] = gi[(size_t)k * ns + e];
  if (stats) {
    for (int e = 0; e < n; ++e) stats[e] = len[e];
    stats[n] = tape_cap; stats[n + 1] = reruns;
  }
  delete D;
  return rows * 1000 + cols;
}

}  // extern "C"
