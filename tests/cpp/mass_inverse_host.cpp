// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
//
// The inverse-mass-matrix instances of the product's generic step kernel, tiny-differentiable-simulator_b200/csrc/tds_stepw.cu (template
// flags MASS and MINV: fp64 forward and the tangent-seeded dual numbers, with and without installed physical parameters), and the
// contraction kernel of J M^-1 J^T (csrc/tds_mass_inverse.cu, double and dual), compiled FOR THE HOST with the same single-lane meanings
// of the CUDA built-ins as tests/cpp/mass_host.cpp, and called lane after lane as tds_launch_mass_inverse / tds_launch_mass_inverse_jvp /
// tds_launch_osim launch them on the GPU.  Nothing outside tests/ builds or loads it.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/mass_inverse_host.cpp -o tests/cpp/_mass_inverse_host.so
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
#define TDS_MINV_KERNEL_ONLY 1
#include "../../tiny-differentiable-simulator_b200/csrc/tds_mass_inverse.cu"

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
        tdsw::tds_stepw_kernel<R, R, R, R, false, PAR, JV, true, false, false, false, false, false, false, false, true>(M, P, E, io,
                                                                                                                       tdsw::MODE_NOCONTACT, 0,
                                                                                                                       scratch, pa);
      }
}

struct Setup {
  DevModel D;
  ParMap pm;
  int n, ns, k;
  std::vector<float> sq;
  std::vector<double> par;
};

int setup(Setup& S, const double* model, int n_model, int n, const double* q, int k, const int* ids, const double* values, int size) {
  int rc = tds_build_dev_model(model, n_model, &S.D);
  if (rc) return rc;
  const char* err = nullptr;
  if (tds_build_par_map(&S.D, k, ids, &S.pm, &err)) return -100;
  tds_build_layout_w(&S.D, size, size, size, -1, size);
  S.n = n; S.ns = (n + 31) & ~31; S.k = k;
  const int n_q = S.D.n_q;
  S.sq.assign((size_t)(n_q > 0 ? n_q : 1) * S.ns, 0.f);
  S.par.assign((size_t)(k > 0 ? k : 1) * S.ns, 0.0);
  for (int e = 0; e < n; ++e) {
    for (int j = 0; j < n_q; ++j) S.sq[(size_t)j * S.ns + e] = (float)q[(size_t)e * n_q + j];
    for (int j = 0; j < k; ++j) S.par[(size_t)j * S.ns + e] = values[(size_t)e * k + j];
  }
  S.pm.values = S.par.data(); S.pm.grad = nullptr;
  return 0;
}

// dM [(nn * m)][ns] along the tangents tq [n_q * m][ns], tp [k * m][ns] (device layouts)
void jvp_soa(const Setup& S, int m, const double* tq, const double* tp, double* dM) {
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = S.sq.data(); io.n = S.n; io.n_stride = S.ns;
  io.jac = dM; io.jac_n_in = m; io.jac_dir0 = 0;
  std::vector<char> scratch((size_t)m * ((S.n + 31) / 32) * S.D.x_total * 32 * 4 + 64);
  const tdsw::JvpTan jv{tq, tp, m};
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

// M^-1 [n][n_qd][n_qd] of every environment at q [n][n_q] (rounded to fp32), with k installed parameters ids[k] at values [n][k] (k = 0: the
// instance without parameters).  Returns 0, or < 0 (-100: rejected ids).
int tdsemu_mass_inverse(const double* model, int n_model, int n, const double* q, int k, const int* ids, const double* values, double* M) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, k, ids, values, 8);
  if (rc) { delete S; return rc; }
  const int nd = S->D.n_qd, nn = nd * nd, ns = S->ns;
  std::vector<double> out((size_t)(nn > 0 ? nn : 1) * ns, 0.0);
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = S->sq.data(); io.n = n; io.n_stride = ns; io.jac = out.data(); io.jac_n_in = 1;
  std::vector<char> scratch((size_t)((n + 31) / 32) * S->D.x_total * 32 * 4 + 64);
  if (k > 0) run_grid<double, true, false>(S->D, io, 1, scratch.data(), S->pm);
  else run_grid<double, false, false>(S->D, io, 1, scratch.data(), tdsw::NoPar{});
  for (int e = 0; e < n; ++e)
    for (int r = 0; r < nn; ++r) M[(size_t)e * nn + r] = out[(size_t)r * ns + e];
  delete S;
  return 0;
}

// dM^-1 [n][n_qd][n_qd][m] along t_q [n][n_q][m] (or null) and t_par [n][k][m] (or null).  Other arguments as tdsemu_mass_inverse.
int tdsemu_mass_inverse_jvp(const double* model, int n_model, int n, const double* q, int k, const int* ids, const double* values, int m,
                    const double* t_q, const double* t_par, double* dM) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, k, ids, values, 16);
  if (rc) { delete S; return rc; }
  const int n_q = S->D.n_q, nn = S->D.n_qd * S->D.n_qd, ns = S->ns;
  std::vector<double> tq((size_t)(n_q > 0 ? n_q : 1) * m * ns, 0.0), tp((size_t)(k > 0 ? k : 1) * m * ns, 0.0), out((size_t)nn * m * ns, 0.0);
  for (int e = 0; e < n; ++e) {
    if (t_q) for (int c = 0; c < n_q * m; ++c) tq[(size_t)c * ns + e] = t_q[(size_t)e * n_q * m + c];
    if (t_par) for (int c = 0; c < k * m; ++c) tp[(size_t)c * ns + e] = t_par[(size_t)e * k * m + c];
  }
  jvp_soa(*S, m, t_q ? tq.data() : nullptr, t_par ? tp.data() : nullptr, out.data());
  for (int e = 0; e < n; ++e)
    for (int c = 0; c < nn * m; ++c) dM[(size_t)e * nn * m + c] = out[(size_t)c * ns + e];
  delete S;
  return 0;
}

// L = J Mi J^T [n][R][R] (R = 6K) from J [n][R][n_qd] and Mi [n][n_qd][n_qd] by the contraction kernel; with m >= 1 its tangents
// [n][R * R][m] from dJ [n][R * n_qd][m] (or null) and dMi [n][n_qd * n_qd][m], as tds_launch_osim runs them.
int tdsemu_osim(int n, int K, int n_qd, const double* J, const double* Mi, int m, const double* dJ, const double* dMi, double* L) {
  const int ns = (n + 31) & ~31, R = 6 * K;
  const size_t nJ = (size_t)R * n_qd, nn = (size_t)n_qd * n_qd, nL = (size_t)R * R;
  const int mm = m > 0 ? m : 1;
  std::vector<double> sJ(nJ * ns + 1, 0.0), sM(nn * ns + 1, 0.0), sdJ(nJ * mm * ns + 1, 0.0), sdM(nn * mm * ns + 1, 0.0), o(nL * mm * ns + 1, 0.0);
  for (int e = 0; e < n; ++e) {
    for (size_t r = 0; r < nJ; ++r) sJ[r * ns + e] = J[(size_t)e * nJ + r];
    for (size_t r = 0; r < nn; ++r) sM[r * ns + e] = Mi[(size_t)e * nn + r];
    if (m > 0) {
      if (dJ) for (size_t r = 0; r < nJ * m; ++r) sdJ[r * ns + e] = dJ[(size_t)e * nJ * m + r];
      for (size_t r = 0; r < nn * m; ++r) sdM[r * ns + e] = dMi[(size_t)e * nn * m + r];
    }
  }
  emu_blockDim = {128, 1, 1};
  for (int j = 0; j < mm; ++j)
    for (int a = 0; a < R; ++a)
      for (int e = 0; e < n; ++e) {
        emu_blockIdx = {(unsigned)(e / 128), (unsigned)a, (unsigned)j};
        emu_threadIdx = {(unsigned)(e % 128), 0, 0};
        if (m > 0) osim_kernel<tds::Dual<double>>(sJ.data(), dJ ? sdJ.data() : nullptr, sM.data(), sdM.data(), o.data(), R, n_qd, m, 0, n, ns);
        else osim_kernel<double>(sJ.data(), nullptr, sM.data(), nullptr, o.data(), R, n_qd, 1, 0, n, ns);
      }
  for (int e = 0; e < n; ++e)
    for (size_t r = 0; r < nL * mm; ++r) L[(size_t)e * nL * mm + r] = o[r * ns + e];
  return 0;
}

}  // extern "C"
