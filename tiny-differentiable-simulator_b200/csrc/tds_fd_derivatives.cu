// The product kernel of the forward dynamics' derivatives (DESIGN.md section 7.24): with qdd = M^-1 (tau - h) and A = [d tau / dq |
// d tau / dqd] of the inverse dynamics at that qdd,
//   d qdd / dq = -M^-1 d tau / dq,   d qdd / dqd = -M^-1 d tau / dqd,   d qdd / dtau = M^-1.
// One thread per environment, column c and tangent: column c of A_q and of A_qd in two per-thread arrays, then row k of -M^-1 A's column
// c in both, each entry of M^-1 read once for the two (the identity's columns copy M^-1's).  The environments run fastest, so that the
// [rows][ns] loads coalesce; neither matrix dimension has unit stride in that layout, which is why a batched GEMM does not fit.  On
// double and on the tangent-seeded Dual<double>, whose (value, tangent) loads differentiate -M^-1 A as -dM^-1 A - M^-1 dA.
#include <cuda_runtime.h>

#include "tds_types.h"
#include "tds_soa.cuh"

namespace {
constexpr int kFddMaxQd = 3 * TDS_MAX_LINKS + 6;

// environment e, column b % n_qd of A_q and A_qd (b < n_qd) or of the identity (b >= n_qd), tangent j = blockIdx.z; b = blockIdx.y, or
// blockIdx.y + n_qd when neither dq nor dqd is wanted (the launch then covers the identity's columns alone)
template <typename T>
__global__ void fdd_product_kernel(const TdsFddCall c, int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int nd = c.n_qd, b = (int)blockIdx.y + ((c.dq || c.dqd) ? 0 : nd), col = b % nd, j = blockIdx.z, jo = c.j0 + j;
  if (e >= n) return;
  if (b >= nd) {
    for (int k = 0; k < nd; ++k) {
      const size_t r = (size_t)k * nd + col;
      osim_st(c.dtau, osim_ld<T>(c.Mi, c.dMi, r, c.m, j, ns, e), r, c.m_out, jo, ns, e);
    }
    return;
  }
  T yq[kFddMaxQd], yd[kFddMaxQd];
  for (int r = 0; r < nd; ++r) {
    if (c.dq) yq[r] = osim_ld<T>(c.Aq, c.dAq, (size_t)r * nd + col, c.m, j, ns, e);
    if (c.dqd) yd[r] = osim_ld<T>(c.Aqd, c.dAqd, (size_t)r * nd + col, c.m, j, ns, e);
  }
  for (int k = 0; k < nd; ++k) {
    T xq = T(0.0), xd = T(0.0);
    for (int r = 0; r < nd; ++r) {
      const T mi = osim_ld<T>(c.Mi, c.dMi, (size_t)k * nd + r, c.m, j, ns, e);
      if (c.dq) xq = xq + mi * yq[r];
      if (c.dqd) xd = xd + mi * yd[r];
    }
    if (c.dq) osim_st(c.dq, -xq, (size_t)k * nd + col, c.m_out, jo, ns, e);
    if (c.dqd) osim_st(c.dqd, -xd, (size_t)k * nd + col, c.m_out, jo, ns, e);
  }
}
}  // namespace

// (TDS_FDD_KERNEL_ONLY: the kernel alone, for the host build of the tests)
#ifndef TDS_FDD_KERNEL_ONLY
// The product of one call over n environments: the value instance (dual false), or the dual instance over the call's m tangents
// (m <= 65535: gridDim.z).  Only the wanted columns are launched: those of A when dq or dqd is wanted, the identity's when dtau is.
extern "C" int tds_launch_fdd(const TdsFddCall* c, int dual, int n, int ns, cudaStream_t stream) {
  if (c->n_qd > kFddMaxQd) return (int)cudaErrorInvalidValue;
  const int cols = ((c->dq || c->dqd) ? c->n_qd : 0) + (c->dtau ? c->n_qd : 0);
  if (cols == 0 || n == 0) return 0;
  const dim3 grid((n + 127) / 128, cols, dual ? c->m : 1);
  if (dual) fdd_product_kernel<tds::Dual<double>><<<grid, 128, 0, stream>>>(*c, n, ns);
  else fdd_product_kernel<double><<<grid, 128, 0, stream>>>(*c, n, ns);
  return (int)cudaGetLastError();
}
#endif  // TDS_FDD_KERNEL_ONLY
