// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
// The Jacobian-vector product instance of the rigid-body world kernel (tiny-differentiable-simulator_b200/csrc/tds_rigid.cu, template
// flag JV) compiled FOR THE HOST and called world after world and tangent after tangent, like tests/cpp/rigid_host.cpp does for the
// dual-number Jacobian.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/rigid_jvp_host.cpp -o tests/cpp/_rigid_jvp_host.so
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
// desc [n_bodies][6]; params: dt, g[3], friction, restitution, erp, iterations; state [n][n_bodies][13]; force [n][n_bodies][3] or null
// (zero force, passed to the kernel as rigid_host.cpp does for the Jacobian); t_state [n][n_bodies][13][m], t_force [n][n_bodies][3][m]
// (either may be null) -> state_out [n][n_bodies][13] (or null), t_out [n][n_bodies][13][m]
int tdsemu_rigid_jvp(const double* desc, int nb, const double* params, int n, const double* state, const double* force, int steps, int m,
                     const double* t_state, const double* t_force, double* state_out, double* t_out) {
  RigidWorld W;
  { const int rcw = tds_rigid_world_from_desc(desc, nb, &W); if (rcw) return rcw; }
  W.dt = params[0]; for (int k = 0; k < 3; ++k) W.gravity[k] = params[1 + k];
  W.friction = params[4]; W.restitution = params[5]; W.erp = params[6]; W.num_solver_iterations = (int)params[7];
  const int ns = (n + 31) & ~31, rows = 13 * nb;
  std::vector<double> s((size_t)rows * ns, 0.0), o((size_t)rows * ns, 0.0), f((size_t)3 * nb * ns, 0.0);
  std::vector<double> ts((size_t)rows * m * ns, 0.0), tf((size_t)3 * nb * m * ns, 0.0), to((size_t)rows * m * ns, 0.0);
  for (int e = 0; e < n; ++e) {
    for (int k = 0; k < rows; ++k) s[(size_t)k * ns + e] = state[(size_t)e * rows + k];
    if (force) for (int k = 0; k < 3 * nb; ++k) f[(size_t)k * ns + e] = force[(size_t)e * 3 * nb + k];
    if (t_state) for (int k = 0; k < rows * m; ++k) ts[(size_t)k * ns + e] = t_state[(size_t)e * rows * m + k];
    if (t_force) for (int k = 0; k < 3 * nb * m; ++k) tf[(size_t)k * ns + e] = t_force[(size_t)e * 3 * nb * m + k];
  }
  const tdsrb::RigidJvpIO v{t_state ? ts.data() : nullptr, t_force ? tf.data() : nullptr, to.data(), m};
  emu::bDim = {1, 1, 1};
  emu::tIdx = {0, 0, 0};
  for (int e = 0; e < n; ++e)
    for (int j = 0; j < m; ++j) {
      emu::bIdx = {(unsigned)e, (unsigned)j, 0};
      tdsrb::tds_rigid_step_kernel<tds::Dual<double>, double, true>(W, s.data(), o.data(), f.data(), steps, n, ns, nullptr, 0, v);
    }
  for (int e = 0; e < n; ++e) {
    if (state_out) for (int k = 0; k < rows; ++k) state_out[(size_t)e * rows + k] = o[(size_t)k * ns + e];
    for (int k = 0; k < rows * m; ++k) t_out[(size_t)e * rows * m + k] = to[(size_t)k * ns + e];
  }
  return 0;
}
}  // extern "C"
