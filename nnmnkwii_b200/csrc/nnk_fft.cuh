// nnk_fft.cuh -- complex arithmetic and the per-bin operations of the modulation-spectrum kernels, shared by
// csrc/nnk_modspec.cu (utterance level) and csrc/nnk_ms_segment.cu (segment level).
#pragma once
#include <cfloat>

#include <cuda_runtime.h>

namespace nnk {

template <typename T> struct Cx;
template <> struct Cx<float> { using V = float2; };
template <> struct Cx<double> { using V = double2; };

template <typename V> __device__ __forceinline__ V cx(decltype(V::x) re, decltype(V::x) im) { V v; v.x = re; v.y = im; return v; }
template <typename V> __device__ __forceinline__ V cadd(V a, V b) { return cx<V>(a.x + b.x, a.y + b.y); }
template <typename V> __device__ __forceinline__ V csub(V a, V b) { return cx<V>(a.x - b.x, a.y - b.y); }
template <typename V> __device__ __forceinline__ V cmul(V a, V b) { return cx<V>(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
template <typename V> __device__ __forceinline__ V conj_(V a) { return cx<V>(a.x, -a.y); }
template <typename V> __device__ __forceinline__ V times_i(V a) { return cx<V>(-a.y, a.x); }
template <typename V> __device__ __forceinline__ V scale(V a, decltype(V::x) s) { return cx<V>(a.x * s, a.y * s); }

__device__ __forceinline__ void sincospi_t(float a, float* s, float* c) { sincospif(a, s, c); }
__device__ __forceinline__ void sincospi_t(double a, double* s, double* c) { sincospi(a, s, c); }

// Y / |Y| (numpy's exp(1j angle(Y)) up to rounding); (+-1, 0) for a zero bin, by the sign of its real part
template <typename V> __device__ __forceinline__ V unit_phase(V y) {
  const auto r = hypot(y.x, y.y);
  if (r == 0) return cx<V>(signbit(y.x) ? -1 : 1, 0);
  return cx<V>(y.x / r, y.y / r);
}

// s = log(max(p, tiny)), tiny the dtype's smallest normal number: finite for a bin of zero power
__device__ __forceinline__ float log_power(float p) { return logf(fmaxf(p, FLT_MIN)); }
__device__ __forceinline__ double log_power(double p) { return log(fmax(p, DBL_MIN)); }

// one post-filtered bin (k >= 1): Y / |Y| exp(s' / 2) with s' = a s + c, ac = (a, c); a bin of zero power stays 0
template <typename V> __device__ __forceinline__ V postfilter_bin(V y, V ac) {
  using T = decltype(V::x);
  const T p = y.x * y.x + y.y * y.y;
  if (p == T(0)) return cx<V>(0, 0);
  return scale(unit_phase(y), exp((ac.x * log_power(p) + ac.y) * T(0.5)));
}

}  // namespace nnk
