// Reverse-mode taping scalar for the step kernels (vector-Jacobian products, DESIGN.md section 7.8).
//
// Tape<double> is {value, node id}: 16 bytes like Dual<double>, so the 16-byte-scalar arena layout of the dual instance
// (tds_build_layout_w(..., 16, 16, 16, -1, 16)) serves it unchanged.  id < 0 marks a constant; every operation with a
// non-constant operand appends one node {id_a, id_b, d result / d a, d result / d b} to the lane's tape.  The function set
// and its semantics are those of tds_dual.cuh: comparisons act on the values, min / max select an operand, sqrt has a zero
// derivative at 0, the exponent of pow is a parameter.  So the derivative is that of the branch taken, exactly as with the
// dual numbers, and g^T J (dual) and the reverse sweep agree up to summation order.
//
// Storage: each lane's nodes live in global memory, interleaved by lane within a warp (node k of lane l at
// warp_base + k * 32 + l), so lanes that run in lockstep store coalesced.  The fp64 adjoints of the reverse sweep use the
// same interleave.  Nodes 0 .. n_in - 1 are the inputs (ad_seed below sets the id, no node is written for them).
// The lane's cursor sits in a per-thread slot of a static shared array: the operators are free functions without a
// context argument.  A lane that would exceed its capacity sets the overflow flag and stops recording; values are still
// computed, and the caller reruns with a larger tape.  Capacity 0: values only (nothing is recorded, no flag is set).
#pragma once
#include <type_traits>

#include "tds_math.cuh"

namespace tds {

struct TapeNode { int a, b; double da, db; };

struct TapeLane {
  TapeNode* node;     // node k of this lane at node[k * 32]
  int n, cap;
  int* overflow;      // set to 1 when a push finds the tape full (null: values-only run)
};

#define TDS_TAPE_MAX_THREADS 128
TDS_D TapeLane& tape_lane() {
  static __shared__ TapeLane lanes[TDS_TAPE_MAX_THREADS];
  return lanes[threadIdx.x];
}

// start recording: n_in input leaves, nodes at node_base (already offset to this lane), capacity cap nodes
TDS_D void tape_begin(TapeNode* node_base, int cap, int* overflow, int n_in) {
  TapeLane& L = tape_lane();
  L.node = node_base; L.cap = cap; L.overflow = overflow; L.n = n_in;
  if (n_in > cap) { if (overflow) *overflow = 1; L.cap = 0; }
}

TDS_D int tape_push(int a, double da, int b, double db) {
  TapeLane& L = tape_lane();
  if (L.n >= L.cap) {
    if (L.cap > 0 && L.overflow) *L.overflow = 1;
    L.cap = 0;
    return -1;
  }
  TapeNode* p = L.node + (size_t)L.n * 32;
  p->a = a; p->b = b; p->da = da; p->db = db;
  return L.n++;
}

TDS_D bool tape_ok() { const TapeLane& L = tape_lane(); return L.cap > 0 && L.n <= L.cap; }
TDS_D int tape_length() { return tape_lane().n; }

template <typename T> struct Tape {
  T v; int id;
  TDS_D Tape() {}
  template <typename U, typename = typename std::enable_if<std::is_arithmetic<U>::value>::type>
  TDS_D Tape(U u) : v(T(u)), id(-1) {}
  TDS_D Tape(T v_, int id_) : v(v_), id(id_) {}
  friend TDS_D Tape operator+(Tape a, Tape b) { return bin(a.v + b.v, a, T(1), b, T(1)); }
  friend TDS_D Tape operator-(Tape a, Tape b) { return bin(a.v - b.v, a, T(1), b, T(-1)); }
  friend TDS_D Tape operator*(Tape a, Tape b) { return bin(a.v * b.v, a, b.v, b, a.v); }
  friend TDS_D Tape operator/(Tape a, Tape b) { const T q = a.v / b.v; return bin(q, a, T(1) / b.v, b, -q / b.v); }
  friend TDS_D Tape operator-(Tape a) { return un(-a.v, a, T(-1)); }
  TDS_D Tape& operator+=(Tape b) { *this = *this + b; return *this; }
  TDS_D Tape& operator-=(Tape b) { *this = *this - b; return *this; }
  TDS_D Tape& operator*=(Tape b) { *this = *this * b; return *this; }
  TDS_D Tape& operator/=(Tape b) { *this = *this / b; return *this; }
  friend TDS_D bool operator<(Tape a, Tape b) { return a.v < b.v; }
  friend TDS_D bool operator>(Tape a, Tape b) { return a.v > b.v; }
  friend TDS_D bool operator<=(Tape a, Tape b) { return a.v <= b.v; }
  friend TDS_D bool operator>=(Tape a, Tape b) { return a.v >= b.v; }
  friend TDS_D bool operator==(Tape a, Tape b) { return a.v == b.v; }
  friend TDS_D bool operator!=(Tape a, Tape b) { return a.v != b.v; }
  // one recorded operation: a result with one or two operands and their partial derivatives
  static TDS_D Tape un(T v, Tape a, T da) { return Tape(v, a.id < 0 ? -1 : tape_push(a.id, (double)da, -1, 0.0)); }
  static TDS_D Tape bin(T v, Tape a, T da, Tape b, T db) {
    if (a.id < 0 && b.id < 0) return Tape(v, -1);
    return Tape(v, tape_push(a.id, (double)da, b.id, (double)db));
  }
};

template <typename T> struct is_tape { static constexpr bool value = false; };
template <typename T> struct is_tape<Tape<T>> { static constexpr bool value = true; };

// input idx of the lane is node idx (the Jacobian's column order)
template <typename T> TDS_D Tape<T> ad_seed(Tape<T> x, int idx, int) { x.id = idx; return x; }

template <typename T> TDS_D double val_of(Tape<T> a) { return (double)a.v; }
template <typename T> TDS_D Tape<T> min_t(Tape<T> a, Tape<T> b) { return a.v < b.v ? a : b; }
template <typename T> TDS_D Tape<T> max_t(Tape<T> a, Tape<T> b) { return a.v > b.v ? a : b; }
template <typename T> TDS_D Tape<T> sqrt_t(Tape<T> a) {
  const T r = sqrt_t(a.v);
  return Tape<T>::un(r, a, r > T(0) ? T(1) / (T(2) * r) : T(0));
}
template <typename T> TDS_D void sincos_t(Tape<T> a, Tape<T>* s, Tape<T>* c) {
  T sv, cv;
  sincos_t(a.v, &sv, &cv);
  *s = Tape<T>::un(sv, a, cv);
  *c = Tape<T>::un(cv, a, -sv);
}
template <typename T> TDS_D Tape<T> pow_t(Tape<T> a, Tape<T> b) {   // exponent: a parameter (no derivative)
  const T p = pow_t(a.v, b.v);
  return Tape<T>::un(p, a, a.v > T(0) ? b.v * p / a.v : T(0));
}
template <typename T> TDS_D Tape<T> atan2_t(Tape<T> y, Tape<T> x) {
  const T r2 = x.v * x.v + y.v * y.v;
  return Tape<T>::bin(atan2_t(y.v, x.v), y, r2 > T(0) ? x.v / r2 : T(0), x, r2 > T(0) ? -y.v / r2 : T(0));
}
template <typename T> TDS_D Tape<T> tanh_t(Tape<T> a) {
  const T t = tanh_t(a.v);
  return Tape<T>::un(t, a, T(1) - t * t);
}

// Reverse sweep of this lane's tape.  adj: the lane's fp64 adjoints (entry k at adj[k * 32], >= tape_length() entries);
// out_id(r): node id of output r (< 0: constant), g_out(r): its cotangent; on return adj[k * 32] holds d(g^T out) / d input k
// for k < n_in.  Returns false (adjoints untouched) when the tape overflowed.
template <typename FId, typename FG>
TDS_D bool tape_reverse(double* adj, int n_rows, FId out_id, FG g_out, int n_in) {
  const TapeLane& L = tape_lane();
  if (!tape_ok()) return false;
  const int len = L.n;
  for (int k = 0; k < len; ++k) adj[(size_t)k * 32] = 0.0;
  for (int r = 0; r < n_rows; ++r) {
    const int id = out_id(r);
    if (id >= 0) adj[(size_t)id * 32] += g_out(r);
  }
  for (int k = len - 1; k >= n_in; --k) {
    const double g = adj[(size_t)k * 32];
    if (g == 0.0) continue;
    const TapeNode nd = L.node[(size_t)k * 32];
    if (nd.a >= 0) adj[(size_t)nd.a * 32] += nd.da * g;
    if (nd.b >= 0) adj[(size_t)nd.b * 32] += nd.db * g;
  }
  return true;
}

}  // namespace tds
