// Loads and stores of the dynamics queries' fp64 outputs in the device layout [rows][ns] (values) and [rows * m][ns] (tangent j of an
// m-tangent block at row r * m + j), as the contraction kernels that read them take them: a plain double for the value instances, a dual
// number (value, tangent j) for the tangent-seeded instances.  Used by tds_mass_inverse.cu and tds_constrained.cu.
#pragma once
#include <stddef.h>

#include "tds_dual.cuh"

namespace {
// entry r of a [rows][ns] fp64 output: the value (T = double), or the value with the dual part of tangent j from [rows * m][ns]
template <typename T> __device__ __forceinline__ T osim_ld(const double* v, const double* d, size_t r, int m, int j, int ns, int e);
template <> __device__ __forceinline__ double osim_ld<double>(const double* v, const double*, size_t r, int, int, int ns, int e) {
  return v[r * ns + e];
}
template <> __device__ __forceinline__ tds::Dual<double> osim_ld<tds::Dual<double>>(const double* v, const double* d, size_t r, int m, int j,
                                                                                      int ns, int e) {
  return tds::Dual<double>(v[r * ns + e], d ? d[(r * m + j) * ns + e] : 0.0);
}
__device__ __forceinline__ void osim_st(double* o, double x, size_t r, int, int, int ns, int e) { o[r * ns + e] = x; }
__device__ __forceinline__ void osim_st(double* o, const tds::Dual<double>& x, size_t r, int m, int j, int ns, int e) {
  o[(r * m + j) * ns + e] = x.d;
}
}  // namespace
