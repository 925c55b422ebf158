// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
// The instances of the rigid-body world kernel with per-world physical parameters (tiny-differentiable-simulator_b200/csrc/tds_rigid.cu,
// template flag PAR) compiled FOR THE HOST and called world after world (and direction / tangent after direction), like
// tests/cpp/rigid_host.cpp, rigid_jvp_host.cpp and rigid_vjp_host.cpp do for the instances without parameters.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/rigid_param_host.cpp -o tests/cpp/_rigid_param_host.so
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <vector>

#define TDS_B200_EXACT_RCP 1
#define TDS_RIGID_KERNEL_ONLY 1
namespace emu { struct Dim { unsigned x, y, z; }; static Dim tIdx, bIdx, bDim; }
#define threadIdx emu::tIdx
#define blockIdx emu::bIdx
#define blockDim emu::bDim
#undef __global__
#define __global__
#undef __grid_constant__
#define __grid_constant__
#undef __launch_bounds__
#define __launch_bounds__(...)

#include "../../tiny-differentiable-simulator_b200/csrc/tds_rigid.cu"

namespace {
// the world of desc / params (dt, g[3], friction, restitution, erp, iterations) and the map of the ids with SoA values [k][ns]
struct Setup {
  RigidWorld W;
  RigidParMap pm;
  int n, ns, rows, k;
  std::vector<double> s, f, vals;
};

int setup(Setup& S, const double* desc, int nb, const double* params, int n, const double* state, const double* force, int k, const int* ids,
          const double* values) {
  { const int rcw = tds_rigid_world_from_desc(desc, nb, &S.W); if (rcw) return rcw; }
  S.W.dt = params[0]; for (int c = 0; c < 3; ++c) S.W.gravity[c] = params[1 + c];
  S.W.friction = params[4]; S.W.restitution = params[5]; S.W.erp = params[6]; S.W.num_solver_iterations = (int)params[7];
  if (tds_rigid_par_map(S.W, k, ids, &S.pm)) return -100;
  S.n = n; S.ns = (n + 31) & ~31; S.rows = 13 * nb; S.k = k;
  S.s.assign((size_t)S.rows * S.ns, 0.0); S.f.assign((size_t)3 * nb * S.ns, 0.0); S.vals.assign((size_t)(k > 0 ? k : 1) * S.ns, 0.0);
  for (int e = 0; e < n; ++e) {
    for (int r = 0; r < S.rows; ++r) S.s[(size_t)r * S.ns + e] = state[(size_t)e * S.rows + r];
    if (force) for (int r = 0; r < 3 * nb; ++r) S.f[(size_t)r * S.ns + e] = force[(size_t)e * 3 * nb + r];
    for (int j = 0; j < k; ++j) S.vals[(size_t)j * S.ns + e] = values[(size_t)e * k + j];
  }
  S.pm.values = S.vals.data();
  return 0;
}
}  // namespace

extern "C" {
// the checks of tds_b200_rigid_set_physical_params_host: 0, -2 (ids; reason to err) or -3 (values [n][k])
int tdsemu_rigid_par_check(const double* desc, int nb, int k, const int* ids, int n, const double* values, char* err, int err_len) {
  RigidWorld W;
  if (tds_rigid_world_from_desc(desc, nb, &W)) return -1;
  RigidParMap pm;
  if (const char* r = tds_rigid_par_map(W, k, ids, &pm)) { snprintf(err, err_len, "%s", r); return -2; }
  for (int e = 0; e < n; ++e)
    for (int s = 0; s < k; ++s)
      if (!tds_rigid_par_value_ok(ids[s], values[(size_t)e * k + s])) { snprintf(err, err_len, "value"); return -3; }
  return 0;
}

// `steps` steps with the parameters ids = values [n][k]: state_out [n][nb][13] by the fp64 PAR instance; jac_in [n][13 nb][16 nb] (or
// null) and jac_par [n][13 nb][k] (or null) by the dual PAR instance.  force null: zero force for the dual instance, none for fp64.
int tdsemu_rigid_par(const double* desc, int nb, const double* params, int n, const double* state, const double* force, int steps, int k,
                     const int* ids, const double* values, double* state_out, double* jac_in, double* jac_par) {
  Setup S;
  if (const int rc = setup(S, desc, nb, params, n, state, force, k, ids, values)) return rc;
  const int ns = S.ns, rows = S.rows, cols = 16 * nb;
  std::vector<double> o((size_t)rows * ns, 0.0), Ji, Jp;
  emu::bDim = {1, 1, 1};
  emu::tIdx = {0, 0, 0};
  for (int e = 0; e < n; ++e) {
    emu::bIdx = {(unsigned)e, 0, 0};
    tdsrb::tds_rigid_step_kernel<double, double, false, true>(S.W, S.s.data(), o.data(), force ? S.f.data() : nullptr, steps, n, ns, nullptr, 0,
                                                             tdsrb::RigidVjpIO{}, S.pm);
  }
  std::vector<double> o2((size_t)rows * ns, 0.0);
  if (jac_in) {
    Ji.assign((size_t)rows * cols * ns, 0.0);
    for (int e = 0; e < n; ++e)
      for (int d = 0; d < cols; ++d) {
        emu::bIdx = {(unsigned)e, (unsigned)d, 0};
        tdsrb::tds_rigid_step_kernel<tds::Dual<double>, double, false, true>(S.W, S.s.data(), o2.data(), S.f.data(), steps, n, ns, Ji.data(), 0,
                                                                            tdsrb::RigidVjpIO{}, S.pm);
      }
  }
  if (jac_par && k > 0) {
    Jp.assign((size_t)rows * k * ns, 0.0);
    for (int e = 0; e < n; ++e)
      for (int d = 0; d < k; ++d) {
        emu::bIdx = {(unsigned)e, (unsigned)d, 0};
        tdsrb::tds_rigid_step_kernel<tds::Dual<double>, double, false, true>(S.W, S.s.data(), o2.data(), S.f.data(), steps, n, ns, Jp.data(),
                                                                            16 * nb, tdsrb::RigidVjpIO{}, S.pm);
      }
  }
  for (int e = 0; e < n; ++e) {
    if (state_out) for (int r = 0; r < rows; ++r) state_out[(size_t)e * rows + r] = o[(size_t)r * ns + e];
    if (jac_in) for (int r = 0; r < rows * cols; ++r) jac_in[(size_t)e * rows * cols + r] = Ji[(size_t)r * ns + e];
    if (jac_par && k > 0) for (int r = 0; r < rows * k; ++r) jac_par[(size_t)e * rows * k + r] = Jp[(size_t)r * ns + e];
  }
  return 0;
}

// Jacobian-vector products of `steps` steps by the tangent-seeded dual PAR instance: t_state [n][nb][13][m], t_force [n][nb][3][m],
// t_par [n][k][m] (each may be null) -> state_out [n][nb][13] (or null), t_out [n][nb][13][m]
int tdsemu_rigid_par_jvp(const double* desc, int nb, const double* params, int n, const double* state, const double* force, int steps, int k,
                         const int* ids, const double* values, int m, const double* t_state, const double* t_force, const double* t_par,
                         double* state_out, double* t_out) {
  Setup S;
  if (const int rc = setup(S, desc, nb, params, n, state, force, k, ids, values)) return rc;
  const int ns = S.ns, rows = S.rows;
  std::vector<double> o((size_t)rows * ns, 0.0), ts((size_t)rows * m * ns, 0.0), tf((size_t)3 * nb * m * ns, 0.0),
      tp((size_t)(k > 0 ? k : 1) * m * ns, 0.0), to((size_t)rows * m * ns, 0.0);
  for (int e = 0; e < n; ++e) {
    if (t_state) for (int r = 0; r < rows * m; ++r) ts[(size_t)r * ns + e] = t_state[(size_t)e * rows * m + r];
    if (t_force) for (int r = 0; r < 3 * nb * m; ++r) tf[(size_t)r * ns + e] = t_force[(size_t)e * 3 * nb * m + r];
    if (t_par) for (int r = 0; r < k * m; ++r) tp[(size_t)r * ns + e] = t_par[(size_t)e * k * m + r];
  }
  const tdsrb::RigidJvpIO v{t_state ? ts.data() : nullptr, t_force ? tf.data() : nullptr, to.data(), m};
  S.pm.t_par = t_par ? tp.data() : nullptr;
  emu::bDim = {1, 1, 1};
  emu::tIdx = {0, 0, 0};
  for (int e = 0; e < n; ++e)
    for (int j = 0; j < m; ++j) {
      emu::bIdx = {(unsigned)e, (unsigned)j, 0};
      tdsrb::tds_rigid_step_kernel<tds::Dual<double>, double, true, true>(S.W, S.s.data(), o.data(), S.f.data(), steps, n, ns, nullptr, 0, v, S.pm);
    }
  for (int e = 0; e < n; ++e) {
    if (state_out) for (int r = 0; r < rows; ++r) state_out[(size_t)e * rows + r] = o[(size_t)r * ns + e];
    for (int r = 0; r < rows * m; ++r) t_out[(size_t)e * rows * m + r] = to[(size_t)r * ns + e];
  }
  return 0;
}

// Vector-Jacobian product of `steps` steps by the taping PAR instance, checkpointed and chunked as tds_b200_rigid_vjp_params_device does
// it: the forward keeps the states (values only), then one recorded step per step runs backwards over chunks of `chunk` worlds; a chunk
// whose tape overflowed is rerun with twice the capacity, and its parameter cotangents (written to a staging buffer) are added to g_par
// only once the chunk ran clear.  g_state_out / g_state [n][13 nb], g_force [n][3 nb], g_par [n][k] (summed over the steps).
// stats (or null): [0] the longest tape of a step, [1] final capacity, [2] reruns.
int tdsemu_rigid_par_vjp(const double* desc, int nb, const double* params, int n, const double* state, const double* force, int steps, int k,
                         const int* ids, const double* values, const double* g_state_out, double* g_state, double* g_force, double* g_par,
                         int tape_cap, int chunk, double* stats) {
  Setup S;
  if (const int rc = setup(S, desc, nb, params, n, state, force, k, ids, values)) return rc;
  const int ns = S.ns, rows = S.rows;
  const size_t st = (size_t)rows * ns;
  std::vector<double> ck(st * (steps > 0 ? steps : 1), 0.0), g(st, 0.0), gn(st, 0.0), gf((size_t)3 * nb * ns, 0.0);
  std::vector<double> gp((size_t)(k > 0 ? k : 1) * ns, 0.0), stage((size_t)(k > 0 ? k : 1) * ns, 0.0);
  std::copy(S.s.begin(), S.s.end(), ck.begin());
  for (int e = 0; e < n; ++e) for (int r = 0; r < rows; ++r) g[(size_t)r * ns + e] = g_state_out[(size_t)e * rows + r];
  emu::bDim = {1, 1, 1};
  emu::tIdx = {0, 0, 0};
  const double* fp = force ? S.f.data() : nullptr;
  for (int s = 0; s + 1 < steps; ++s)
    for (int e = 0; e < n; ++e) {
      emu::bIdx = {(unsigned)e, 0, 0};
      tdsrb::tds_rigid_step_kernel<tds::Tape<double>, double, false, true>(S.W, ck.data() + s * st, ck.data() + (s + 1) * st, s == 0 ? fp : nullptr,
                                                                          1, n, ns, nullptr, 0, tdsrb::RigidVjpIO{}, S.pm);
    }
  std::vector<tds::TapeNode> tape;
  std::vector<double> adj;
  int overflow = 0, reruns = 0, longest = 0;
  for (int s = steps - 1; s >= 0; --s) {
    for (int e0 = 0; e0 < n;) {
      const int c = chunk < n - e0 ? chunk : n - e0;
      tape.assign((size_t)ns * tape_cap, tds::TapeNode{});
      adj.assign((size_t)ns * tape_cap, 0.0);
      tdsrb::RigidVjpIO v{g.data(), gn.data(), s == 0 ? gf.data() : nullptr, tape.data(), adj.data(), tape_cap, &overflow};
      RigidParMap pm = S.pm;
      pm.grad = stage.data();
      overflow = 0;
      for (int e = e0; e < e0 + c; ++e) {
        emu::bIdx = {(unsigned)e, 0, 0};
        tdsrb::tds_rigid_step_kernel<tds::Tape<double>, double, false, true>(S.W, ck.data() + s * st, nullptr, s == 0 ? fp : nullptr, 1, n, ns,
                                                                            nullptr, 0, v, pm);
        if (tds::tape_length() > longest) longest = tds::tape_length();
      }
      if (overflow) { tape_cap *= 2; ++reruns; continue; }
      for (int j = 0; j < k; ++j) for (int e = e0; e < e0 + c; ++e) gp[(size_t)j * ns + e] += stage[(size_t)j * ns + e];
      e0 += c;
    }
    g.swap(gn);
  }
  for (int e = 0; e < n; ++e) {
    for (int r = 0; r < rows; ++r) g_state[(size_t)e * rows + r] = g[(size_t)r * ns + e];
    if (g_force) for (int r = 0; r < 3 * nb; ++r) g_force[(size_t)e * 3 * nb + r] = gf[(size_t)r * ns + e];
    for (int j = 0; j < k; ++j) g_par[(size_t)e * k + j] = gp[(size_t)j * ns + e];
  }
  if (stats) { stats[0] = longest; stats[1] = tape_cap; stats[2] = reruns; }
  return 0;
}
}  // extern "C"
