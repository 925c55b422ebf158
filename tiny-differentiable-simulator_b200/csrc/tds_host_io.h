// Host-buffer staging shared by the C-ABI's *_host entry points (tds_capi.cu, tds_rigid.cu).  Caller arrays are
// environment-major [n][rows]; device arrays are row-major over the padded batch [rows][ns] (ns = n rounded up to 32).
// Every function returns the first CUDA error, so each file keeps its own error reporting.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <initializer_list>
#include <vector>

// Grows the device buffer *p of *have bytes to at least `bytes`; the old contents are not kept.  A caller whose stream may still
// read the old buffer synchronises before the call.
template <typename T>
inline cudaError_t grow_dev(T** p, size_t* have, size_t bytes) {
  if (bytes <= *have) return cudaSuccess;
  cudaFree(*p);
  *p = nullptr; *have = 0;
  const cudaError_t e = cudaMalloc((void**)p, bytes);
  if (e == cudaSuccess) *have = bytes;
  return e;
}

// host [n][rows] -> device [rows][ns]; columns e >= n are zero.  Returns once the host memory may be reused.
template <typename T>
inline cudaError_t put_rows(T* dev, const T* host, size_t rows, int n, int ns, cudaStream_t stream) {
  std::vector<T> t(rows * ns, T(0));
  for (int e = 0; e < n; ++e)
    for (size_t r = 0; r < rows; ++r) t[r * ns + e] = host[(size_t)e * rows + r];
  const cudaError_t err = t.empty() ? cudaSuccess : cudaMemcpyAsync(dev, t.data(), sizeof(T) * t.size(), cudaMemcpyHostToDevice, stream);
  return err != cudaSuccess ? err : cudaStreamSynchronize(stream);   // (t is released on return)
}

// device [rows][ns] -> host [n][rows], after the work queued on `stream`; returns with the data in host memory.  A launch error
// left by that work is returned too.
template <typename T>
inline cudaError_t get_rows(T* host, const T* dev, size_t rows, int n, int ns, cudaStream_t stream) {
  std::vector<T> t(rows * ns);
  cudaError_t err = t.empty() ? cudaSuccess : cudaMemcpyAsync(t.data(), dev, sizeof(T) * t.size(), cudaMemcpyDeviceToHost, stream);
  if (err == cudaSuccess) err = cudaStreamSynchronize(stream);
  if (err == cudaSuccess) err = cudaGetLastError();
  if (err != cudaSuccess) return err;
  for (int e = 0; e < n; ++e)
    for (size_t r = 0; r < rows; ++r) host[(size_t)e * rows + r] = t[r * ns + e];
  return cudaSuccess;
}

// One part of a concatenation: `rows` rows at p, or NULL.  The parts lie in consecutive [rows][ns] blocks of one device array.
template <typename T>
struct RowPart { T* p; size_t rows; };

// host parts [n][rows] -> their blocks of dev; a NULL part's block is zeroed
template <typename T>
inline cudaError_t put_parts(T* dev, std::initializer_list<RowPart<const T>> parts, int n, int ns, cudaStream_t stream) {
  for (const RowPart<const T>& a : parts) {
    const cudaError_t err = a.p ? put_rows(dev, a.p, a.rows, n, ns, stream) : cudaMemsetAsync(dev, 0, sizeof(T) * a.rows * ns, stream);
    if (err != cudaSuccess) return err;
    dev += a.rows * ns;
  }
  return cudaSuccess;
}

// blocks of dev -> host parts [n][rows], as get_rows; a NULL part is skipped
template <typename T>
inline cudaError_t get_parts(std::initializer_list<RowPart<T>> parts, const T* dev, int n, int ns, cudaStream_t stream) {
  for (const RowPart<T>& a : parts) {
    if (a.p)
      if (const cudaError_t err = get_rows(a.p, dev, a.rows, n, ns, stream)) return err;
    dev += a.rows * ns;
  }
  return cudaSuccess;
}

// The same concatenation of device parts [rows][ns], device to device and asynchronous on `stream`: put_parts_d2d copies every
// part into its block (NULL: zeros), get_parts_d2d every block out to its part (NULL: skipped).
template <typename T>
inline cudaError_t put_parts_d2d(T* dev, std::initializer_list<RowPart<const T>> parts, int ns, cudaStream_t stream) {
  for (const RowPart<const T>& a : parts) {
    const size_t bytes = sizeof(T) * a.rows * ns;
    const cudaError_t err = a.p ? cudaMemcpyAsync(dev, a.p, bytes, cudaMemcpyDeviceToDevice, stream) : cudaMemsetAsync(dev, 0, bytes, stream);
    if (err != cudaSuccess) return err;
    dev += a.rows * ns;
  }
  return cudaSuccess;
}

template <typename T>
inline cudaError_t get_parts_d2d(std::initializer_list<RowPart<T>> parts, const T* dev, int ns, cudaStream_t stream) {
  for (const RowPart<T>& a : parts) {
    if (a.p)
      if (const cudaError_t err = cudaMemcpyAsync(a.p, dev, sizeof(T) * a.rows * ns, cudaMemcpyDeviceToDevice, stream)) return err;
    dev += a.rows * ns;
  }
  return cudaSuccess;
}
