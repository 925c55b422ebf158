// Kernels of the point-constrained forward dynamics (DESIGN.md section 7.21): from h = ID(q, qd, 0), M^-1, the point-motion J and drift
// J' qd of the existing value and dual-number launches, the dense per-environment solve of
//   M qdd - J_c^T f = tau - h,   J_c qdd = -d_c - eps f
// as f = -(J_c M^-1 J_c^T + eps I)^-1 (J_c M^-1 (tau - h) + d_c), qdd = M^-1 (tau - h + J_c^T f).  Two kernels, each on double and on
// the tangent-seeded Dual<double>: the constraint rows (one thread per environment, row and tangent) and the solve (one thread per
// environment and tangent).  The dual instances differentiate the Cholesky factorisation itself.
#include <cuda_runtime.h>
#include <math.h>

#include "tds_types.h"
#include "tds_soa.cuh"

namespace {
constexpr int kCdMaxQd = 3 * TDS_MAX_LINKS + 6;

// entry r of a scratch quantity: the value at [r][ns] (T = double; m = 1, j = 0), or the (value, tangent) pair of tangent j at [r * m + j]
template <typename T> __device__ __forceinline__ T cd_ld(const double* v, const double* d, size_t r, int m, int j, int ns, int e);
template <> __device__ __forceinline__ double cd_ld<double>(const double* v, const double*, size_t r, int m, int j, int ns, int e) {
  return v[(r * m + j) * ns + e];
}
template <> __device__ __forceinline__ tds::Dual<double> cd_ld<tds::Dual<double>>(const double* v, const double* d, size_t r, int m, int j,
                                                                                    int ns, int e) {
  const size_t i = (r * m + j) * ns + e;
  return tds::Dual<double>(v[i], d[i]);
}
__device__ __forceinline__ void cd_st(double* v, double*, double x, size_t r, int m, int j, int ns, int e) { v[(r * m + j) * ns + e] = x; }
__device__ __forceinline__ void cd_st(double* v, double* d, const tds::Dual<double>& x, size_t r, int m, int j, int ns, int e) {
  const size_t i = (r * m + j) * ns + e;
  v[i] = x.v;
  d[i] = x.d;
}

// tau_c - h_c: tau fp32 (null: zero) with its tangent (null: zero), h fp64
template <typename T> __device__ __forceinline__ T cd_rhs(const TdsCdynCall& c, int r, int j, int ns, int e);
template <> __device__ __forceinline__ double cd_rhs<double>(const TdsCdynCall& c, int r, int, int ns, int e) {
  return (c.tau ? (double)c.tau[(size_t)r * ns + e] : 0.0) - c.h[(size_t)r * ns + e];
}
template <> __device__ __forceinline__ tds::Dual<double> cd_rhs<tds::Dual<double>>(const TdsCdynCall& c, int r, int j, int ns, int e) {
  const tds::Dual<double> tau(c.tau ? (double)c.tau[(size_t)r * ns + e] : 0.0, c.dtau ? c.dtau[((size_t)r * c.m + j) * ns + e] : 0.0);
  return tau - osim_ld<tds::Dual<double>>(c.h, c.dh, r, c.m, j, ns, e);
}

template <typename T> __device__ __forceinline__ T cd_nan();
template <> __device__ __forceinline__ double cd_nan<double>() { return NAN; }
template <> __device__ __forceinline__ tds::Dual<double> cd_nan<tds::Dual<double>>() { return tds::Dual<double>(NAN, NAN); }

// row of J (6 rows per point) of constrained row a: all six rows of a point (dims 6) or its linear rows 3..5 (dims 3)
__device__ __forceinline__ size_t cd_jrow(int a, int dims) { return (size_t)(a / dims) * 6 + (6 - dims) + a % dims; }

// Constraint row a = blockIdx.y of environment e, tangent j = blockIdx.z: y = J_a M^-1 in a per-thread row, then Y_a = y,
// A_ab = y . J_b for b >= a (written to (a, b) and (b, a)) and b_a = y . (tau - h) + d_a.
template <typename T>
__global__ void cd_rows_kernel(const TdsCdynCall c, int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int a = blockIdx.y, j = blockIdx.z, nd = c.n_qd, R = c.dims * c.K;
  const int sm = tds::is_dual<T>::value ? c.m : 1;   // (tangents of the scratch pairs)
  if (e >= n) return;
  const size_t ja = cd_jrow(a, c.dims);
  T y[kCdMaxQd];
  for (int k = 0; k < nd; ++k) y[k] = T(0.0);
  for (int r = 0; r < nd; ++r) {
    const T jr = osim_ld<T>(c.J, c.dJ, ja * nd + r, c.m, j, ns, e);
    for (int k = 0; k < nd; ++k) y[k] = y[k] + jr * osim_ld<T>(c.Mi, c.dMi, (size_t)r * nd + k, c.m, j, ns, e);
  }
  T s = T(0.0);
  for (int k = 0; k < nd; ++k) {
    cd_st(c.Y, c.dY, y[k], (size_t)a * nd + k, sm, j, ns, e);
    s = s + y[k] * cd_rhs<T>(c, k, j, ns, e);
  }
  cd_st(c.b, c.db, s + osim_ld<T>(c.acc, c.dacc, ja, c.m, j, ns, e), a, sm, j, ns, e);
  for (int b = a; b < R; ++b) {
    const size_t jb = cd_jrow(b, c.dims);
    T acc = T(0.0);
    for (int k = 0; k < nd; ++k) acc = acc + y[k] * osim_ld<T>(c.J, c.dJ, jb * nd + k, c.m, j, ns, e);
    cd_st(c.A, c.dA, acc, (size_t)a * R + b, sm, j, ns, e);
    if (b > a) cd_st(c.A, c.dA, acc, (size_t)b * R + a, sm, j, ns, e);
  }
}

// Environment e, tangent j = blockIdx.y: in place in the scratch, A + eps I = L L^T (lower triangle), f = -(L L^T)^-1 b in b, then
// qdd = M^-1 (tau - h) + sum_a Y_a^T f_a.  A pivot <= 0 (or NaN) makes every output of the lane NaN.  K = 0: qdd = M^-1 (tau - h).
template <typename T>
__global__ void cd_solve_kernel(const TdsCdynCall c, int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int j = blockIdx.y, nd = c.n_qd, R = c.dims * c.K;
  const int sm = tds::is_dual<T>::value ? c.m : 1;
  if (e >= n) return;
  bool ok = true;
  for (int k = 0; k < R && ok; ++k) {
    T d = cd_ld<T>(c.A, c.dA, (size_t)k * R + k, sm, j, ns, e) + T(c.eps);
    for (int p = 0; p < k; ++p) {
      const T l = cd_ld<T>(c.A, c.dA, (size_t)k * R + p, sm, j, ns, e);
      d = d - l * l;
    }
    if (!(d > T(0.0))) { ok = false; break; }
    d = tds::sqrt_t(d);
    cd_st(c.A, c.dA, d, (size_t)k * R + k, sm, j, ns, e);
    for (int r = k + 1; r < R; ++r) {
      T x = cd_ld<T>(c.A, c.dA, (size_t)r * R + k, sm, j, ns, e);
      for (int p = 0; p < k; ++p) x = x - cd_ld<T>(c.A, c.dA, (size_t)r * R + p, sm, j, ns, e) * cd_ld<T>(c.A, c.dA, (size_t)k * R + p, sm, j, ns, e);
      cd_st(c.A, c.dA, x / d, (size_t)r * R + k, sm, j, ns, e);
    }
  }
  const int jo = c.j0 + j;
  if (!ok) {
    for (int k = 0; k < nd; ++k) if (c.qdd) osim_st(c.qdd, cd_nan<T>(), k, c.m_out, jo, ns, e);
    for (int a = 0; a < R; ++a) if (c.f) osim_st(c.f, cd_nan<T>(), a, c.m_out, jo, ns, e);
    return;
  }
  for (int k = 0; k < R; ++k) {   // L z = -b
    T x = -cd_ld<T>(c.b, c.db, k, sm, j, ns, e);
    for (int p = 0; p < k; ++p) x = x - cd_ld<T>(c.A, c.dA, (size_t)k * R + p, sm, j, ns, e) * cd_ld<T>(c.b, c.db, p, sm, j, ns, e);
    cd_st(c.b, c.db, x / cd_ld<T>(c.A, c.dA, (size_t)k * R + k, sm, j, ns, e), k, sm, j, ns, e);
  }
  for (int k = R - 1; k >= 0; --k) {   // L^T f = z
    T x = cd_ld<T>(c.b, c.db, k, sm, j, ns, e);
    for (int p = k + 1; p < R; ++p) x = x - cd_ld<T>(c.A, c.dA, (size_t)p * R + k, sm, j, ns, e) * cd_ld<T>(c.b, c.db, p, sm, j, ns, e);
    x = x / cd_ld<T>(c.A, c.dA, (size_t)k * R + k, sm, j, ns, e);
    cd_st(c.b, c.db, x, k, sm, j, ns, e);
    if (c.f) osim_st(c.f, x, k, c.m_out, jo, ns, e);
  }
  if (!c.qdd) return;
  T u[kCdMaxQd];
  for (int k = 0; k < nd; ++k) u[k] = cd_rhs<T>(c, k, j, ns, e);
  for (int k = 0; k < nd; ++k) {
    T x = T(0.0);
    for (int r = 0; r < nd; ++r) x = x + osim_ld<T>(c.Mi, c.dMi, (size_t)k * nd + r, c.m, j, ns, e) * u[r];
    for (int a = 0; a < R; ++a) x = x + cd_ld<T>(c.Y, c.dY, (size_t)a * nd + k, sm, j, ns, e) * cd_ld<T>(c.b, c.db, a, sm, j, ns, e);
    osim_st(c.qdd, x, k, c.m_out, jo, ns, e);
  }
}
}  // namespace

// (TDS_CDYN_KERNEL_ONLY: the kernels alone, for the host build of the tests)
#ifndef TDS_CDYN_KERNEL_ONLY
// The rows and the solve of one call over n environments: the value instances (dual false), or the dual instances over the call's m
// tangents (m <= 65535: gridDim.y, gridDim.z).
extern "C" int tds_launch_cdyn(const TdsCdynCall* c, int dual, int n, int ns, cudaStream_t stream) {
  if (c->n_qd > kCdMaxQd) return (int)cudaErrorInvalidValue;
  const int R = c->dims * c->K, mz = dual ? c->m : 1, bx = (n + 127) / 128;
  if (R > 0) {
    if (dual) cd_rows_kernel<tds::Dual<double>><<<dim3(bx, R, mz), 128, 0, stream>>>(*c, n, ns);
    else cd_rows_kernel<double><<<dim3(bx, R, 1), 128, 0, stream>>>(*c, n, ns);
    if (const cudaError_t err = cudaGetLastError()) return (int)err;
  }
  if (dual) cd_solve_kernel<tds::Dual<double>><<<dim3(bx, mz), 128, 0, stream>>>(*c, n, ns);
  else cd_solve_kernel<double><<<dim3(bx, 1), 128, 0, stream>>>(*c, n, ns);
  return (int)cudaGetLastError();
}
#endif  // TDS_CDYN_KERNEL_ONLY
