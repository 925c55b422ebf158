// Shared device helpers of the world-frame kernels (tds_stepw.cu: one lane per environment,
// tds_team_step.cuh: four roles per environment, on lanes or warps): strided shared-memory accessors,
// accumulator records, 3x3 register blocks for the blocked dense solves.
#pragma once
#include <cuda_runtime.h>

#include "tds_math.cuh"
#include "tds_dual.cuh"
#include "tds_tape.cuh"
#include "tds_types.h"
#include "tds_b200_model.h"

namespace tdsw {
using namespace tds;

struct Arena {
  char* blk;
  int stride;
  int col;
  template <typename T> TDS_D T* ptr(int word) const {
    if (sizeof(T) == 4) return ((T*)blk) + (size_t)word * stride + col;
    if (sizeof(T) == 16) return ((T*)blk) + (size_t)(word >> 2) * stride + col;   // dual numbers (tds_dual.cuh)
    return ((T*)blk) + (size_t)(word >> 1) * stride + col;
  }
};

// MultiBodyConstraintSolver::plane_space (src/mb_constraint_solver.hpp:506-520) for a per-contact normal, as the reference
// evaluates it: k = sqrt(a) (not its reciprocal) and p.z = n.y k in both branches.
template <typename T> TDS_D void plane_space_t(const V3<T>& n, V3<T>& p, V3<T>& q) {
  const T n_sqr = n.z * n.z;
  const bool mz = n_sqr > T(0.5);
  const T a = n.y * n.y + (mz ? n_sqr : n.x * n.x);
  const T k = sqrt_t(a);
  p.x = mz ? T(0) : -n.y * k;
  p.y = mz ? -n.z * k : n.x * k;
  p.z = n.y * k;
  q.x = mz ? a * k : -n.z * p.y;
  q.y = mz ? -n.x * p.z : n.z * p.x;
  q.z = mz ? n.x * p.y : a * k;
}

template <typename T> TDS_D void st3(T* p, int s, const V3<T>& v) { p[0] = v.x; p[s] = v.y; p[2 * s] = v.z; }
template <typename T> TDS_D V3<T> ld3(const T* p, int s) { return v3<T>(p[0], p[s], p[2 * s]); }
template <typename T> TDS_D void st6(T* p, int s, const Sv<T>& v) { st3(p, s, v.top); st3(p + 3 * s, s, v.bot); }
template <typename T> TDS_D Sv<T> ld6(const T* p, int s) { Sv<T> r; r.top = ld3(p, s); r.bot = ld3(p + 3 * s, s); return r; }
template <typename T> TDS_D void st9(T* p, int s, const M3<T>& m) {
  p[0] = m.xx; p[s] = m.xy; p[2 * s] = m.xz; p[3 * s] = m.yx; p[4 * s] = m.yy; p[5 * s] = m.yz; p[6 * s] = m.zx; p[7 * s] = m.zy; p[8 * s] = m.zz;
}
template <typename T> TDS_D M3<T> ld9(const T* p, int s) {
  M3<T> m;
  m.xx = p[0]; m.xy = p[s]; m.xz = p[2 * s]; m.yx = p[3 * s]; m.yy = p[4 * s]; m.yz = p[5 * s]; m.zx = p[6 * s]; m.zy = p[7 * s]; m.zz = p[8 * s];
  return m;
}
template <typename T> TDS_D void st_rbi(T* p, int s, const Rbi<T>& r) {
  p[0] = r.m; p[s] = r.h.x; p[2 * s] = r.h.y; p[3 * s] = r.h.z;
  p[4 * s] = r.I.xx; p[5 * s] = r.I.xy; p[6 * s] = r.I.xz; p[7 * s] = r.I.yy; p[8 * s] = r.I.yz; p[9 * s] = r.I.zz;
}
template <typename T> TDS_D Rbi<T> ld_rbi(const T* p, int s) {
  Rbi<T> r;
  r.m = p[0]; r.h = v3<T>(p[s], p[2 * s], p[3 * s]);
  r.I.xx = p[4 * s]; r.I.xy = p[5 * s]; r.I.xz = p[6 * s]; r.I.yy = p[7 * s]; r.I.yz = p[8 * s]; r.I.zz = p[9 * s];
  return r;
}
template <typename TO, typename TI> TDS_D Rbi<TO> cvt_rbi(const Rbi<TI>& a) {
  Rbi<TO> r;
  r.m = TO(a.m); r.h = cvt<TO>(a.h);
  r.I.xx = TO(a.I.xx); r.I.xy = TO(a.I.xy); r.I.xz = TO(a.I.xz); r.I.yy = TO(a.I.yy); r.I.yz = TO(a.I.yz); r.I.zz = TO(a.I.zz);
  return r;
}
template <typename TO, typename TI> TDS_D Sv<TO> cvt_sv(const Sv<TI>& a) { Sv<TO> r; r.top = cvt<TO>(a.top); r.bot = cvt<TO>(a.bot); return r; }
template <typename T> TDS_D M3<T> transpose(const M3<T>& a) {
  M3<T> r; r.xx = a.xx; r.xy = a.yx; r.xz = a.zx; r.yx = a.xy; r.yy = a.yy; r.yz = a.zy; r.zx = a.xz; r.zy = a.yz; r.zz = a.zz;
  return r;
}
template <typename T> TDS_D V3<T> col_x(const M3<T>& a) { return v3<T>(a.xx, a.yx, a.zx); }
template <typename T> TDS_D V3<T> col_y(const M3<T>& a) { return v3<T>(a.xy, a.yy, a.zy); }
template <typename T> TDS_D V3<T> col_z(const M3<T>& a) { return v3<T>(a.xz, a.yz, a.zz); }
template <typename T> TDS_D void set_cols(M3<T>& a, V3<T> x, V3<T> y, V3<T> z) {
  a.xx = x.x; a.yx = x.y; a.zx = x.z; a.xy = y.x; a.yy = y.y; a.zy = y.z; a.xz = z.x; a.yz = z.y; a.zz = z.z;
}
template <typename T> TDS_D V3<T> axpy(V3<T> a, T s, V3<T> b) { return v3<T>(a.x * s + b.x, a.y * s + b.y, a.z * s + b.z); }

// accumulator slot: Ia 21 + pA 6 (RA), composite Ic 10 (RC) at word offset x_acc_ic_word
template <typename T> TDS_D void acc_add27(T* p, int s, const Abi<T>& a, const Sv<T>& f) {
  p[0] += a.I.xx; p[s] += a.I.xy; p[2 * s] += a.I.xz; p[3 * s] += a.I.yy; p[4 * s] += a.I.yz; p[5 * s] += a.I.zz;
  p[6 * s] += a.H.xx; p[7 * s] += a.H.xy; p[8 * s] += a.H.xz; p[9 * s] += a.H.yx; p[10 * s] += a.H.yy; p[11 * s] += a.H.yz;
  p[12 * s] += a.H.zx; p[13 * s] += a.H.zy; p[14 * s] += a.H.zz;
  p[15 * s] += a.M.xx; p[16 * s] += a.M.xy; p[17 * s] += a.M.xz; p[18 * s] += a.M.yy; p[19 * s] += a.M.yz; p[20 * s] += a.M.zz;
  p[21 * s] += f.top.x; p[22 * s] += f.top.y; p[23 * s] += f.top.z; p[24 * s] += f.bot.x; p[25 * s] += f.bot.y; p[26 * s] += f.bot.z;
}
template <typename T> TDS_D void acc_ld27(const T* p, int s, Abi<T>& a, Sv<T>& f) {
  a.I.xx = p[0]; a.I.xy = p[s]; a.I.xz = p[2 * s]; a.I.yy = p[3 * s]; a.I.yz = p[4 * s]; a.I.zz = p[5 * s];
  a.H.xx = p[6 * s]; a.H.xy = p[7 * s]; a.H.xz = p[8 * s]; a.H.yx = p[9 * s]; a.H.yy = p[10 * s]; a.H.yz = p[11 * s];
  a.H.zx = p[12 * s]; a.H.zy = p[13 * s]; a.H.zz = p[14 * s];
  a.M.xx = p[15 * s]; a.M.xy = p[16 * s]; a.M.xz = p[17 * s]; a.M.yy = p[18 * s]; a.M.yz = p[19 * s]; a.M.zz = p[20 * s];
  f.top = v3<T>(p[21 * s], p[22 * s], p[23 * s]); f.bot = v3<T>(p[24 * s], p[25 * s], p[26 * s]);
}
template <typename T> TDS_D void rbi_acc(T* p, int s, const Rbi<T>& r) {
  p[0] += r.m; p[s] += r.h.x; p[2 * s] += r.h.y; p[3 * s] += r.h.z;
  p[4 * s] += r.I.xx; p[5 * s] += r.I.xy; p[6 * s] += r.I.xz; p[7 * s] += r.I.yy; p[8 * s] += r.I.yz; p[9 * s] += r.I.zz;
}

// ---- 3x3 register blocks on strided shared memory ------------------------------------------------
template <typename T> struct B9 { T a[9]; };
template <typename T> TDS_D B9<T> ldb(const T* p, int s) {
  B9<T> b;
#pragma unroll
  for (int k = 0; k < 9; ++k) b.a[k] = p[k * s];
  return b;
}
template <typename T> TDS_D void stb(T* p, int s, const B9<T>& b) {
#pragma unroll
  for (int k = 0; k < 9; ++k) p[k * s] = b.a[k];
}
// C -= A * B^T
template <typename T> TDS_D void gemm_nt_sub(B9<T>& C, const B9<T>& A, const B9<T>& B) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      C.a[r * 3 + c] -= A.a[r * 3] * B.a[c * 3] + A.a[r * 3 + 1] * B.a[c * 3 + 1] + A.a[r * 3 + 2] * B.a[c * 3 + 2];
}
// C -= A * B
template <typename T> TDS_D void gemm_nn_sub(B9<T>& C, const B9<T>& A, const B9<T>& B) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      C.a[r * 3 + c] -= A.a[r * 3] * B.a[c] + A.a[r * 3 + 1] * B.a[3 + c] + A.a[r * 3 + 2] * B.a[6 + c];
}
// C += A^T * B
template <typename T> TDS_D void gemm_tn_add(B9<T>& C, const B9<T>& A, const B9<T>& B) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      C.a[r * 3 + c] += A.a[r] * B.a[c] + A.a[3 + r] * B.a[3 + c] + A.a[6 + r] * B.a[6 + c];
}
template <typename T> TDS_D B9<T> b9_zero() {
  B9<T> b;
#pragma unroll
  for (int k = 0; k < 9; ++k) b.a[k] = T(0);
  return b;
}
// inverse of the lower Cholesky factor of a diagonal block: i00, i10, i11, i20, i21, i22
template <typename T> struct L6 { T i00, i10, i11, i20, i21, i22; };
template <typename T> TDS_D L6<T> chol3_inv(const B9<T>& A) {
  const T l00 = sqrt_t(A.a[0]);
  const T i00 = T(1) / l00;
  const T l10 = A.a[3] * i00, l20 = A.a[6] * i00;
  const T l11 = sqrt_t(A.a[4] - l10 * l10);
  const T i11 = T(1) / l11;
  const T l21 = (A.a[7] - l20 * l10) * i11;
  const T l22 = sqrt_t(A.a[8] - l20 * l20 - l21 * l21);
  const T i22 = T(1) / l22;
  L6<T> r;
  r.i00 = i00; r.i11 = i11; r.i22 = i22;
  r.i10 = -l10 * i00 * i11;
  r.i21 = -l21 * i11 * i22;
  r.i20 = -(l20 * i00 + l21 * r.i10) * i22;
  return r;
}
template <typename T> TDS_D L6<T> ldl6(const T* p, int s) { L6<T> r; r.i00 = p[0]; r.i10 = p[s]; r.i11 = p[2 * s]; r.i20 = p[3 * s]; r.i21 = p[4 * s]; r.i22 = p[5 * s]; return r; }
template <typename T> TDS_D void stl6(T* p, int s, const L6<T>& r) { p[0] = r.i00; p[s] = r.i10; p[2 * s] = r.i11; p[3 * s] = r.i20; p[4 * s] = r.i21; p[5 * s] = r.i22; }
// the lower-triangular block of an L6
template <typename T> TDS_D B9<T> l6_full(const L6<T>& li) {
  B9<T> b = b9_zero<T>();
  b.a[0] = li.i00; b.a[3] = li.i10; b.a[4] = li.i11; b.a[6] = li.i20; b.a[7] = li.i21; b.a[8] = li.i22;
  return b;
}
// X = A * Li^T   (off-diagonal block of L = A * L_jj^-T)
template <typename T> TDS_D B9<T> mul_linvT(const B9<T>& A, const L6<T>& li) {
  B9<T> X;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    X.a[r * 3] = A.a[r * 3] * li.i00;
    X.a[r * 3 + 1] = A.a[r * 3] * li.i10 + A.a[r * 3 + 1] * li.i11;
    X.a[r * 3 + 2] = A.a[r * 3] * li.i20 + A.a[r * 3 + 1] * li.i21 + A.a[r * 3 + 2] * li.i22;
  }
  return X;
}
// Y = Li * A   (3 right-hand-side columns)
template <typename T> TDS_D B9<T> linv_mul(const L6<T>& li, const B9<T>& A) {
  B9<T> Y;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    Y.a[c] = li.i00 * A.a[c];
    Y.a[3 + c] = li.i10 * A.a[c] + li.i11 * A.a[3 + c];
    Y.a[6 + c] = li.i20 * A.a[c] + li.i21 * A.a[3 + c] + li.i22 * A.a[6 + c];
  }
  return Y;
}

TDS_D int btri(int bi, int bj) { return (bi * (bi + 1) / 2 + bj) * 9; }

template <typename T> TDS_D Rbi<T> model_rbi_of(const double* r) {
  Rbi<T> o;
  o.m = T(r[0]); o.h = v3<T>(T(r[1]), T(r[2]), T(r[3]));
  o.I.xx = T(r[4]); o.I.xy = T(r[5]); o.I.xz = T(r[6]); o.I.yy = T(r[7]); o.I.yz = T(r[8]); o.I.zz = T(r[9]);
  return o;
}

template <typename T> TDS_D Sv<T> link_axis(const DevModel& M, int i, V3<T>& ax) {
  ax = v3<T>(T(M.axis[i][0]), T(M.axis[i][1]), T(M.axis[i][2]));
  Sv<T> z; z.top = v3<T>(T(0), T(0), T(0)); z.bot = z.top;
  return z;
}

enum StepMode { MODE_FD = 0, MODE_NOCONTACT = 1, MODE_FULL = 2,
                MODE_WORLD = 3 };   // World::step alone (contact detection + constraint solve on the given q, qd): world-frame kernel only

}  // namespace tdsw
