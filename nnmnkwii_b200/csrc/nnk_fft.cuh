// nnk_fft.cuh -- complex arithmetic and the per-bin operations of the modulation-spectrum kernels, shared by
// csrc/nnk_modspec.cu (utterance level), csrc/nnk_ms_segment.cu (segment level) and csrc/nnk_ms_gen.cu
// (generation, both levels).
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

// ---- block-wide real FFT of n = 2 M points, the scheme of modspec_kernel (csrc/nnk_modspec.cu) ------------------
// The n real points are packed as z_t = x_2t + i x_2t+1 into M complex values at bit-reversed positions
// (z[__brev(t) >> (32 - LOGM)]), tw[j] = W^j = e^{-2 pi i j / n} for j < M.  NT threads of one CTA run the stages,
// with a barrier after each.

// decimation in time: bit-reversed in, natural out (Z = FFT_M of the packed points)
template <int LOGN, int NT, typename V>
__device__ __forceinline__ void block_fft_dit(V* z, const V* tw, int tid) {
  constexpr int LOGM = LOGN - 1, M = 1 << LOGM;
#pragma unroll
  for (int s = 1; s <= LOGM; ++s) {
    const int half = 1 << (s - 1);
    for (int j = tid; j < M / 2; j += NT) {
      const int p = j & (half - 1), i0 = ((j >> (s - 1)) << s) + p, i1 = i0 + half;
      const V u = z[i0], v = cmul(z[i1], tw[p << (LOGN - s)]);
      z[i0] = cadd(u, v);
      z[i1] = csub(u, v);
    }
    __syncthreads();
  }
}

// decimation in frequency, inverse: natural in, bit-reversed out.  After rfft_pack_pair on every pair, z holds
// n irfft(C) packed like the input: frame t is component (t & 1) of z[__brev(t >> 1) >> (32 - LOGM)].
template <int LOGN, int NT, typename V>
__device__ __forceinline__ void block_ifft_dif(V* z, const V* tw, int tid) {
  constexpr int LOGM = LOGN - 1, M = 1 << LOGM;
#pragma unroll
  for (int s = LOGM; s >= 1; --s) {
    const int half = 1 << (s - 1);
    for (int j = tid; j < M / 2; j += NT) {
      const int p = j & (half - 1), i0 = ((j >> (s - 1)) << s) + p, i1 = i0 + half;
      const V u = z[i0], v = z[i1];
      z[i0] = cadd(u, v);
      z[i1] = cmul(csub(u, v), conj_(tw[p << (LOGN - s)]));
    }
    __syncthreads();
  }
}

// the same two transforms run by the 32 lanes of one warp on the warp's own z, with __syncwarp between stages
// (csrc/nnk_ms_gen.cu's segment-level trial kernel; nnk_ms_segment.cu keeps its own copy for now)
template <int LOGN, typename V>
__device__ __forceinline__ void warp_fft_dit(V* z, const V* tw, int lane) {
  constexpr int LOGM = LOGN - 1, M = 1 << LOGM;
#pragma unroll
  for (int s = 1; s <= LOGM; ++s) {
    const int half = 1 << (s - 1);
    for (int j = lane; j < M / 2; j += 32) {
      const int p = j & (half - 1), i0 = ((j >> (s - 1)) << s) + p, i1 = i0 + half;
      const V u = z[i0], v = cmul(z[i1], tw[p << (LOGN - s)]);
      z[i0] = cadd(u, v);
      z[i1] = csub(u, v);
    }
    __syncwarp();
  }
}

template <int LOGN, typename V>
__device__ __forceinline__ void warp_ifft_dif(V* z, const V* tw, int lane) {
  constexpr int LOGM = LOGN - 1, M = 1 << LOGM;
#pragma unroll
  for (int s = LOGM; s >= 1; --s) {
    const int half = 1 << (s - 1);
    for (int j = lane; j < M / 2; j += 32) {
      const int p = j & (half - 1), i0 = ((j >> (s - 1)) << s) + p, i1 = i0 + half;
      const V u = z[i0], v = z[i1];
      z[i0] = cadd(u, v);
      z[i1] = cmul(csub(u, v), conj_(tw[p << (LOGN - s)]));
    }
    __syncwarp();
  }
}

// bins k and M - k (k = 0 .. M / 2) of the real spectrum X from Z; pair 0 is (0, M), both from Z_0
template <typename V>
__device__ __forceinline__ void rfft_bin_pair(const V* z, const V* tw, int k, int M, V& Xk, V& Xj) {
  using T = decltype(V::x);
  if (k == 0) {
    const V z0 = z[0];
    Xk = cx<V>(z0.x + z0.y, 0);
    Xj = cx<V>(z0.x - z0.y, 0);
  } else {
    const V zk = z[k], zj = z[M - k];
    const V E = cx<V>((zk.x + zj.x) * T(0.5), (zk.y - zj.y) * T(0.5));
    const V O = cx<V>((zk.y + zj.y) * T(0.5), (zj.x - zk.x) * T(0.5));
    const V WO = cmul(tw[k], O);
    Xk = cadd(E, WO);
    Xj = conj_(csub(E, WO));
  }
}

// the inverse's input at bins k and M - k from the half spectrum C there, in place of rfft_bin_pair's z entries;
// imaginary parts of bins 0 and n / 2 are ignored, as irfft does
template <typename V>
__device__ __forceinline__ void rfft_pack_pair(V* z, const V* tw, int k, int M, V Ck, V Cj) {
  if (k == 0) {
    z[0] = cx<V>(Ck.x + Cj.x, Ck.x - Cj.x);
  } else {
    const V w = tw[k];
    const V A = cadd(Ck, conj_(Cj)), Bd = csub(Ck, conj_(Cj));
    z[k] = cadd(A, times_i(cmul(conj_(w), Bd)));
    if (M - k != k) z[M - k] = cadd(conj_(A), times_i(cmul(w, conj_(Bd))));
  }
}

}  // namespace nnk
