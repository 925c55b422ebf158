// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
//
// The kernels of the point-constrained forward dynamics, tiny-differentiable-simulator_b200/csrc/tds_constrained.cu (the constraint rows
// and the solve, double and dual), compiled FOR THE HOST with single-lane meanings of the CUDA built-ins, and called lane after lane as
// tds_launch_cdyn launches them on the GPU.  The inputs (h, M^-1, J and the drift, and their tangents) come from the host builds of the
// inverse-dynamics, inverse-mass-matrix and point-motion instances (tests/emu_invdyn.py, emu_mass_inverse.py, emu_point_motion.py), as
// the C-ABI takes them from their device launches.  Nothing outside tests/ builds or loads it.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/constrained_dynamics_host.cpp -o ...
#include <cuda_runtime.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#define TDS_B200_EXACT_RCP 1
struct EmuDim { unsigned x, y, z; };
static thread_local EmuDim emu_threadIdx, emu_blockIdx, emu_blockDim, emu_gridDim;
#define threadIdx emu_threadIdx
#define blockIdx emu_blockIdx
#define blockDim emu_blockDim
#define gridDim emu_gridDim
#undef __global__
#define __global__

#define TDS_CDYN_KERNEL_ONLY 1
#include "../../tiny-differentiable-simulator_b200/csrc/tds_constrained.cu"

namespace {
// host [n][rows] -> device layout [rows][ns]
std::vector<double> soa(const double* x, int n, size_t rows, int ns) {
  std::vector<double> o(rows * ns + 1, 0.0);
  if (x)
    for (int e = 0; e < n; ++e)
      for (size_t r = 0; r < rows; ++r) o[r * ns + e] = x[(size_t)e * rows + r];
  return o;
}
void aos(double* y, const std::vector<double>& o, int n, size_t rows, int ns) {
  if (y)
    for (int e = 0; e < n; ++e)
      for (size_t r = 0; r < rows; ++r) y[(size_t)e * rows + r] = o[r * ns + e];
}
}  // namespace

extern "C" {

// qdd [n][n_qd] and f [n][R] (R = dims K) from tau [n][n_qd] (fp32-exact values; null: zero), h [n][n_qd], Mi [n][n_qd][n_qd], J [n][6K][n_qd]
// and acc [n][6K] by the value instances; with m >= 1 instead their tangents t_qdd [n][n_qd][m] and t_f [n][R][m] by the dual instances
// from the tangents dtau, dh [n][n_qd][m], dMi [n][n_qd^2][m], dJ [n][6K n_qd][m], dacc [n][6K][m] (each may be null: zero).
int tdsemu_cdyn(int n, int K, int dims, int nd, double eps, const double* tau, const double* h, const double* Mi, const double* J,
                const double* acc, int m, const double* dtau, const double* dh, const double* dMi, const double* dJ, const double* dacc,
                double* qdd, double* f, double* t_qdd, double* t_f) {
  const int ns = (n + 31) & ~31, R = dims * K, mm = m > 0 ? m : 1;
  const size_t nn = (size_t)nd * nd, nJ = (size_t)6 * K * nd, scr = (size_t)R * nd + (size_t)R * R + R;
  std::vector<float> stau((size_t)nd * ns + 1, 0.f);
  if (tau)
    for (int e = 0; e < n; ++e)
      for (int r = 0; r < nd; ++r) stau[(size_t)r * ns + e] = (float)tau[(size_t)e * nd + r];
  std::vector<double> sh = soa(h, n, nd, ns), sM = soa(Mi, n, nn, ns), sJ = soa(J, n, nJ, ns), sa = soa(acc, n, 6 * K, ns);
  std::vector<double> sdt = soa(dtau, n, (size_t)nd * mm, ns), sdh = soa(dh, n, (size_t)nd * mm, ns), sdM = soa(dMi, n, nn * mm, ns),
                      sdJ = soa(dJ, n, nJ * mm, ns), sda = soa(dacc, n, (size_t)6 * K * mm, ns);
  std::vector<double> v(scr * mm * ns + 1, 0.0), d(scr * mm * ns + 1, 0.0), oq((size_t)nd * mm * ns + 1, 0.0), of((size_t)R * mm * ns + 1, 0.0);
  TdsCdynCall c;
  memset(&c, 0, sizeof(c));
  c.K = K; c.dims = dims; c.n_qd = nd; c.m = mm; c.j0 = 0; c.m_out = mm; c.eps = eps;
  c.tau = tau ? stau.data() : nullptr; c.h = sh.data(); c.Mi = sM.data(); c.J = sJ.data(); c.acc = sa.data();
  if (m > 0) {
    c.dtau = dtau ? sdt.data() : nullptr; c.dh = dh ? sdh.data() : nullptr; c.dMi = dMi ? sdM.data() : nullptr;
    c.dJ = dJ ? sdJ.data() : nullptr; c.dacc = dacc ? sda.data() : nullptr;
  }
  c.Y = v.data(); c.A = c.Y + (size_t)R * nd * mm * ns; c.b = c.A + (size_t)R * R * mm * ns;
  c.dY = d.data(); c.dA = c.dY + (size_t)R * nd * mm * ns; c.db = c.dA + (size_t)R * R * mm * ns;
  c.qdd = oq.data(); c.f = R ? of.data() : nullptr;
  emu_blockDim = {128, 1, 1};
  for (int j = 0; j < mm; ++j)
    for (int e = 0; e < n; ++e) {
      emu_threadIdx = {(unsigned)(e % 128), 0, 0};
      for (int a = 0; a < R; ++a) {
        emu_blockIdx = {(unsigned)(e / 128), (unsigned)a, (unsigned)j};
        if (m > 0) cd_rows_kernel<tds::Dual<double>>(c, n, ns);
        else cd_rows_kernel<double>(c, n, ns);
      }
      emu_blockIdx = {(unsigned)(e / 128), (unsigned)j, 0};
      if (m > 0) cd_solve_kernel<tds::Dual<double>>(c, n, ns);
      else cd_solve_kernel<double>(c, n, ns);
    }
  aos(m > 0 ? t_qdd : qdd, oq, n, (size_t)nd * mm, ns);
  aos(m > 0 ? t_f : f, of, n, (size_t)R * mm, ns);
  return 0;
}

}  // extern "C"
