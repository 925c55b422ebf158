// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
// The reverse-mode (taping) instance of the rigid-body world kernel (tiny-differentiable-simulator_b200/csrc/tds_rigid.cu) compiled FOR
// THE HOST and called world after world, like tests/cpp/rigid_host.cpp does for the double and dual-number instances.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/rigid_vjp_host.cpp -o tests/cpp/_rigid_vjp_host.so
#include <cuda_runtime.h>
#include <math.h>
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

extern "C" {
// Vector-Jacobian product of `steps` steps by the taping instance, checkpointed as tds_b200_rigid_vjp_device does it: the forward
// runs one step at a time (values only) and keeps the states, then one recorded step per world and step runs backwards, chaining
// the state cotangent.  g_state_out / g_state [n][13 nb], g_force [n][3 nb].  tape_cap: starting capacity in nodes per lane
// (doubled and the step rerun on overflow).  stats (or null): [0] the longest tape of a step, [1] final capacity, [2] reruns.
int tdsemu_rigid_vjp(const double* desc, int nb, const double* params, int n, const double* state, const double* force, int steps,
                     const double* g_state_out, double* g_state, double* g_force, int tape_cap, double* stats) {
  RigidWorld W;
  { const int rcw = tds_rigid_world_from_desc(desc, nb, &W); if (rcw) return rcw; }
  W.dt = params[0]; for (int k = 0; k < 3; ++k) W.gravity[k] = params[1 + k];
  W.friction = params[4]; W.restitution = params[5]; W.erp = params[6]; W.num_solver_iterations = (int)params[7];
  const int ns = (n + 31) & ~31, rows = 13 * nb;
  const size_t st = (size_t)rows * ns;
  std::vector<double> ck(st * (steps > 0 ? steps : 1), 0.0), f((size_t)3 * nb * ns, 0.0), g(st, 0.0), gn(st, 0.0), gf((size_t)3 * nb * ns, 0.0);
  for (int e = 0; e < n; ++e) {
    for (int k = 0; k < rows; ++k) { ck[(size_t)k * ns + e] = state[(size_t)e * rows + k]; g[(size_t)k * ns + e] = g_state_out[(size_t)e * rows + k]; }
    if (force) for (int k = 0; k < 3 * nb; ++k) f[(size_t)k * ns + e] = force[(size_t)e * 3 * nb + k];
  }
  emu::bDim = {1, 1, 1};
  emu::tIdx = {0, 0, 0};
  const double* fp = force ? f.data() : nullptr;
  for (int s = 0; s + 1 < steps; ++s)
    for (int e = 0; e < n; ++e) {
      emu::bIdx = {(unsigned)e, 0, 0};
      tdsrb::tds_rigid_step_kernel<tds::Tape<double>, double>(W, ck.data() + s * st, ck.data() + (s + 1) * st, s == 0 ? fp : nullptr, 1, n, ns,
                                                              nullptr, 0, tdsrb::RigidVjpIO{});
    }
  std::vector<tds::TapeNode> tape;
  std::vector<double> adj;
  int overflow = 0, reruns = 0, longest = 0;
  for (int s = steps - 1; s >= 0; --s) {
    for (;;) {
      tape.assign((size_t)ns * tape_cap, tds::TapeNode{});
      adj.assign((size_t)ns * tape_cap, 0.0);
      tdsrb::RigidVjpIO v{g.data(), gn.data(), s == 0 ? gf.data() : nullptr, tape.data(), adj.data(), tape_cap, &overflow};
      overflow = 0;
      for (int e = 0; e < n; ++e) {
        emu::bIdx = {(unsigned)e, 0, 0};
        tdsrb::tds_rigid_step_kernel<tds::Tape<double>, double>(W, ck.data() + s * st, nullptr, s == 0 ? fp : nullptr, 1, n, ns, nullptr, 0, v);
        if (tds::tape_length() > longest) longest = tds::tape_length();
      }
      if (!overflow) break;
      tape_cap *= 2; ++reruns;
    }
    g.swap(gn);
  }
  for (int e = 0; e < n; ++e) {
    for (int k = 0; k < rows; ++k) g_state[(size_t)e * rows + k] = g[(size_t)k * ns + e];
    if (g_force) for (int k = 0; k < 3 * nb; ++k) g_force[(size_t)e * 3 * nb + k] = gf[(size_t)k * ns + e];
  }
  if (stats) { stats[0] = longest; stats[1] = tape_cap; stats[2] = reruns; }
  return 0;
}
}  // extern "C"
