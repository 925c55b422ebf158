// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
//
// The dynamics-derivative instances of the product's generic step kernel, tiny-differentiable-simulator_b200/csrc/tds_stepw.cu (template
// flag DER: fp64 forward and the tangent-seeded dual numbers, with and without installed physical parameters), compiled FOR THE HOST with
// the same single-lane meanings of the CUDA built-ins as tests/cpp/mass_host.cpp, on the grown layout (tds_der_layout_w), and called lane
// after lane as tds_launch_dynamics_derivatives / tds_launch_dynamics_derivatives_jvp (csrc/tds_dynamics_derivatives.cu) launch them on
// the GPU.  Nothing outside tests/ builds or loads it.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/dynamics_derivatives_host.cpp -o tests/cpp/_dynamics_derivatives_host.so
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
void run_grid(const DevModel& M, const StepIO& io, int n_dirs, char* scratch, const PA& pa, const double* gravity) {
  SimParams P;
  EnvParams E;
  memset(&P, 0, sizeof(P));
  memset(&E, 0, sizeof(E));
  for (int c = 0; c < 3; ++c) P.gravity[c] = gravity[c];
  const int warps = (io.n + 31) / 32;
  emu_blockDim = {32, 1, 1};
  emu_gridDim = {(unsigned)warps, (unsigned)n_dirs, 1};
  for (unsigned by = 0; by < (unsigned)n_dirs; ++by)
    for (unsigned bx = 0; bx < (unsigned)warps; ++bx)
      for (unsigned t = 0; t < 32; ++t) {
        if ((int)(bx * 32 + t) >= io.n) continue;
        emu_blockIdx = {bx, by, 0};
        emu_threadIdx = {t, 0, 0};
        tdsw::tds_stepw_kernel<R, R, R, R, false, PAR, JV, false, false, false, false, false, false, false, false, false, false, true>(
            M, P, E, io, tdsw::MODE_NOCONTACT, 0, scratch, pa);
      }
}

struct Setup {
  DevModel D;
  ParMap pm;
  int n, ns, k;
  bool has_qd, has_qdd;
  std::vector<float> sq, sqd, sqdd;
  std::vector<double> par;
};

// qd, qdd may be null (zero); D gets the grown layout of scalar size `size`
int setup(Setup& S, const double* model, int n_model, int n, const double* q, const double* qd, const double* qdd, int k, const int* ids,
          const double* values, int size) {
  int rc = tds_build_dev_model(model, n_model, &S.D);
  if (rc) return rc;
  const char* err = nullptr;
  if (tds_build_par_map(&S.D, k, ids, &S.pm, &err)) return -100;
  tds_build_layout_w(&S.D, size, size, size, -1, size);
  S.D.x_total = tds_der_layout_w(&S.D, size);
  S.n = n; S.ns = (n + 31) & ~31; S.k = k; S.has_qd = qd != nullptr; S.has_qdd = qdd != nullptr;
  const int n_q = S.D.n_q, nd = S.D.n_qd;
  S.sq.assign((size_t)(n_q > 0 ? n_q : 1) * S.ns, 0.f);
  S.sqd.assign((size_t)(nd > 0 ? nd : 1) * S.ns, 0.f);
  S.sqdd.assign((size_t)(nd > 0 ? nd : 1) * S.ns, 0.f);
  S.par.assign((size_t)(k > 0 ? k : 1) * S.ns, 0.0);
  for (int e = 0; e < n; ++e) {
    for (int j = 0; j < n_q; ++j) S.sq[(size_t)j * S.ns + e] = (float)q[(size_t)e * n_q + j];
    if (qd) for (int j = 0; j < nd; ++j) S.sqd[(size_t)j * S.ns + e] = (float)qd[(size_t)e * nd + j];
    if (qdd) for (int j = 0; j < nd; ++j) S.sqdd[(size_t)j * S.ns + e] = (float)qdd[(size_t)e * nd + j];
    for (int j = 0; j < k; ++j) S.par[(size_t)j * S.ns + e] = values[(size_t)e * k + j];
  }
  S.pm.values = S.par.data(); S.pm.grad = nullptr;
  return 0;
}

StepIO io_of(const Setup& S) {
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = S.sq.data(); io.qd_in = S.has_qd ? S.sqd.data() : nullptr; io.tau_in = S.has_qdd ? S.sqdd.data() : nullptr;
  io.n = S.n; io.n_stride = S.ns;
  return io;
}
}  // namespace

extern "C" {

// d tau / dq and d tau / dqd [n][n_qd][n_qd] of every environment at q [n][n_q], qd and qdd [n][n_qd] (rounded to fp32; qd, qdd null:
// zero) under the gravity g [3], with k installed parameters ids[k] at values [n][k] (k = 0: the instance without parameters).  Either
// output may be null.  Returns 0, or < 0 (-100: rejected ids).
int tdsemu_dynamics_derivatives(const double* model, int n_model, int n, const double* q, const double* qd, const double* qdd, const double* g,
                                int k, const int* ids, const double* values, double* dq, double* dqd) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, qd, qdd, k, ids, values, 8);
  if (rc) { delete S; return rc; }
  const int nd = S->D.n_qd, nn = nd * nd, ns = S->ns;
  std::vector<double> o0((size_t)(nn > 0 ? nn : 1) * ns, -1.0), o1((size_t)(nn > 0 ? nn : 1) * ns, -1.0);   // (every entry is written)
  StepIO io = io_of(*S);
  io.jac = dq ? o0.data() : nullptr; io.g_in = dqd ? o1.data() : nullptr; io.jac_n_in = 1;
  std::vector<char> scratch((size_t)((n + 31) / 32) * S->D.x_total * 32 * 4 + 64);
  if (k > 0) run_grid<double, true, false>(S->D, io, 1, scratch.data(), S->pm, g);
  else run_grid<double, false, false>(S->D, io, 1, scratch.data(), tdsw::NoPar{}, g);
  for (int e = 0; e < n; ++e)
    for (int r = 0; r < nn; ++r) {
      if (dq) dq[(size_t)e * nn + r] = o0[(size_t)r * ns + e];
      if (dqd) dqd[(size_t)e * nn + r] = o1[(size_t)r * ns + e];
    }
  delete S;
  return 0;
}

// tangents of d tau / dq and d tau / dqd [n][n_qd][n_qd][m] along t_q [n][n_q][m], t_qd and t_qdd [n][n_qd][m] and t_par [n][k][m] (each may
// be null).  Other arguments as tdsemu_dynamics_derivatives.
int tdsemu_dynamics_derivatives_jvp(const double* model, int n_model, int n, const double* q, const double* qd, const double* qdd,
                                    const double* g, int k, const int* ids, const double* values, int m, const double* t_q, const double* t_qd,
                                    const double* t_qdd, const double* t_par, double* ddq, double* ddqd) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, qd, qdd, k, ids, values, 16);
  if (rc) { delete S; return rc; }
  const int n_q = S->D.n_q, nd = S->D.n_qd, nn = nd * nd, ns = S->ns;
  std::vector<double> ti((size_t)(n_q + 2 * nd) * m * ns, 0.0), tp((size_t)(k > 0 ? k : 1) * m * ns, 0.0);
  std::vector<double> o0((size_t)nn * m * ns + 1, -1.0), o1((size_t)nn * m * ns + 1, -1.0);
  for (int e = 0; e < n; ++e) {
    if (t_q) for (int c = 0; c < n_q * m; ++c) ti[(size_t)c * ns + e] = t_q[(size_t)e * n_q * m + c];
    if (t_qd) for (int c = 0; c < nd * m; ++c) ti[((size_t)n_q * m + c) * ns + e] = t_qd[(size_t)e * nd * m + c];
    if (t_qdd) for (int c = 0; c < nd * m; ++c) ti[((size_t)(n_q + nd) * m + c) * ns + e] = t_qdd[(size_t)e * nd * m + c];
    if (t_par) for (int c = 0; c < k * m; ++c) tp[(size_t)c * ns + e] = t_par[(size_t)e * k * m + c];
  }
  StepIO io = io_of(*S);
  io.jac = o0.data(); io.g_in = o1.data(); io.jac_n_in = m; io.jac_dir0 = 0;
  std::vector<char> scratch((size_t)m * ((n + 31) / 32) * S->D.x_total * 32 * 4 + 64);
  const tdsw::JvpTan jv{(t_q || t_qd || t_qdd) ? ti.data() : nullptr, t_par ? tp.data() : nullptr, m};
  if (k > 0) {
    tdsw::ParMapJvp a;
    static_cast<ParMap&>(a) = S->pm;
    a.jv = jv;
    run_grid<tds::Dual<double>, true, true>(S->D, io, m, scratch.data(), a, g);
  } else {
    run_grid<tds::Dual<double>, false, true>(S->D, io, m, scratch.data(), tdsw::NoParJvp{jv}, g);
  }
  for (int e = 0; e < n; ++e)
    for (int c = 0; c < nn * m; ++c) {
      ddq[(size_t)e * nn * m + c] = o0[(size_t)c * ns + e];
      ddqd[(size_t)e * nn * m + c] = o1[(size_t)c * ns + e];
    }
  delete S;
  return 0;
}

}  // extern "C"
