// Forward-mode dual numbers for the differentiable step (SURVEY 8f.4; the role of CppAD's tape + <model>_jacobian in the
// reference, src/utils/cuda/cuda_codegen.hpp:303-426): the world-frame step kernel is instantiated on Dual<double> for all
// of its scalar types, every lane carries one input direction, and the derivative parts of q', qd' (or qdd) are the
// Jacobian column of that direction.  Comparisons act on the values: the derivative is that of the branch taken
// (contact activation, clamps of PD and of the Gauss-Seidel sweep), as with any operator-overloading AD.
#pragma once
#include <type_traits>

#include "tds_math.cuh"

namespace tds {

template <typename T> struct Dual {
  T v, d;
  TDS_D Dual() {}
  template <typename U, typename = typename std::enable_if<std::is_arithmetic<U>::value>::type>
  TDS_D Dual(U u) : v(T(u)), d(T(0)) {}
  TDS_D Dual(T v_, T d_) : v(v_), d(d_) {}
  friend TDS_D Dual operator+(Dual a, Dual b) { return Dual(a.v + b.v, a.d + b.d); }
  friend TDS_D Dual operator-(Dual a, Dual b) { return Dual(a.v - b.v, a.d - b.d); }
  friend TDS_D Dual operator*(Dual a, Dual b) { return Dual(a.v * b.v, a.d * b.v + a.v * b.d); }
  friend TDS_D Dual operator/(Dual a, Dual b) { const T q = a.v / b.v; return Dual(q, (a.d - q * b.d) / b.v); }
  friend TDS_D Dual operator-(Dual a) { return Dual(-a.v, -a.d); }
  TDS_D Dual& operator+=(Dual b) { v += b.v; d += b.d; return *this; }
  TDS_D Dual& operator-=(Dual b) { v -= b.v; d -= b.d; return *this; }
  TDS_D Dual& operator*=(Dual b) { d = d * b.v + v * b.d; v *= b.v; return *this; }
  TDS_D Dual& operator/=(Dual b) { *this = *this / b; return *this; }
  friend TDS_D bool operator<(Dual a, Dual b) { return a.v < b.v; }
  friend TDS_D bool operator>(Dual a, Dual b) { return a.v > b.v; }
  friend TDS_D bool operator<=(Dual a, Dual b) { return a.v <= b.v; }
  friend TDS_D bool operator>=(Dual a, Dual b) { return a.v >= b.v; }
  friend TDS_D bool operator==(Dual a, Dual b) { return a.v == b.v; }
  friend TDS_D bool operator!=(Dual a, Dual b) { return a.v != b.v; }
};

template <typename T> struct is_dual { static constexpr bool value = false; };
template <typename T> struct is_dual<Dual<T>> { static constexpr bool value = true; };

// input idx of a lane whose input direction is dir: the dual instance seeds .d, the plain instances do nothing, the taping
// instance (tds_tape.cuh) makes it leaf idx
template <typename T> TDS_D T ad_seed(T x, int, int) { return x; }
template <typename T> TDS_D Dual<T> ad_seed(Dual<T> x, int idx, int dir) { if (idx == dir) x.d = T(1); return x; }
// the Jacobian-vector product instances: entry idx of tangent j gets the dual part t[(idx * m + j) * ns + e] (t null: zero tangent)
template <typename T> TDS_D Dual<T> jv_seed(Dual<T> x, const double* t, int idx, int m, int j, int ns, int e) {
  x.d = t ? T(t[((size_t)idx * m + j) * ns + e]) : T(0);
  return x;
}

template <typename T> TDS_D double val_of(Dual<T> a) { return (double)a.v; }
template <typename T> TDS_D Dual<T> min_t(Dual<T> a, Dual<T> b) { return a.v < b.v ? a : b; }
template <typename T> TDS_D Dual<T> max_t(Dual<T> a, Dual<T> b) { return a.v > b.v ? a : b; }
template <typename T> TDS_D Dual<T> sqrt_t(Dual<T> a) {
  const T r = sqrt_t(a.v);
  return Dual<T>(r, r > T(0) ? a.d / (T(2) * r) : T(0));
}
template <typename T> TDS_D void sincos_t(Dual<T> a, Dual<T>* s, Dual<T>* c) {
  T sv, cv;
  sincos_t(a.v, &sv, &cv);
  *s = Dual<T>(sv, cv * a.d);
  *c = Dual<T>(cv, -sv * a.d);
}
template <typename T> TDS_D Dual<T> pow_t(Dual<T> a, Dual<T> b) {   // exponent: a parameter (its derivative is not carried)
  const T p = pow_t(a.v, b.v);
  return Dual<T>(p, a.v > T(0) ? b.v * p / a.v * a.d : T(0));
}
template <typename T> TDS_D Dual<T> atan2_t(Dual<T> y, Dual<T> x) {
  const T r2 = x.v * x.v + y.v * y.v;
  return Dual<T>(atan2_t(y.v, x.v), r2 > T(0) ? (x.v * y.d - y.v * x.d) / r2 : T(0));
}
template <typename T> TDS_D Dual<T> tanh_t(Dual<T> a) {
  const T t = tanh_t(a.v);
  return Dual<T>(t, (T(1) - t * t) * a.d);
}

}  // namespace tds
