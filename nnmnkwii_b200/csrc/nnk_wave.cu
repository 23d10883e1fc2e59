// nnk_wave.cu -- waveform and F0 preprocessing: F0 interpolation, pre-emphasis and its inverse, mu-law.
//
// Replaces nnmnkwii/preprocessing/f0.py (interp1d) and generic.py:56-226 (the mu-law family,
// preemphasis, inv_preemphasis).
//
// f0_interp_kernel<T, KIND>: one CTA per row.  A forward walk over tiles of F0_BLOCK frames carries the
// last voiced index (block max-scan) and stores it per frame in the workspace; a backward walk carries the
// next voiced index (block min-scan) and evaluates the kind in float64 with the operation order of the
// scipy routine the reference reaches (de Boor k = 1 for slinear, np.interp / interp1d._call_linear for
// linear), with _rn intrinsics and no contraction.  Frames 0 and len - 1 take the first / last voiced
// value first, as the reference does.
//
// preemph_fir_kernel<T>: y[t] = (0 + x[t]) + (-c) * x[t - 1] (np.convolve's dot, which starts from 0).
//
// inv_preemphasis (y[t] = x[t] + c y[t - 1], scipy's _linear_filter order) in three kernels:
//   preemph_est_kernel<T>     each estimate segment's zero-state end value and c^len, float64
//   preemph_carry_kernel      one CTA per row: scan of the affine maps -> estimate of y before every
//                             warm-up start
//   preemph_spec_kernel<T>    one thread per chunk of IIR_L samples: start W samples early from the
//                             estimate, run the exact dtype recurrence, store the chunk, its start and
//                             end states
//   preemph_repair_kernel<T>  one CTA per row: walk the chunks in order, rerun a chunk whose start state
//                             differs bitwise from the true one until its output merges bitwise
// The recurrence is deterministic, so a trajectory that equals the true one bitwise at one sample equals
// it at every later sample: after the repair every output is the sequential result (DESIGN.md 3.13).
//
// mulaw_kernel<MODE, Tin, Tc, Ty, Tout>: the four mu-law functions, elementwise, in the reference's
// promotion chain (Tc: dtype of sign / log1p / pow, Ty: dtype of the companded value, Tout: result).
#include <math.h>

#include "nnk_common.cuh"

namespace nnk {

constexpr int F0_BLOCK = 256;
constexpr int PE_BLOCK = 256;
constexpr int PE_VEC_BYTES = 16;
constexpr int IIR_L = 1024;        // samples per chunk
constexpr int IIR_W_MAX = 4096;    // longest warm-up
constexpr int IIR_BLOCK = 128;     // threads of the estimate / speculation kernels
constexpr int IIR_SCAN = 256;      // threads of the carry scan and the repair walk
constexpr int MU_BLOCK = 256;

enum F0Kind { F0_LINEAR = 0, F0_SLINEAR = 1, F0_ZERO = 2, F0_NEAREST = 3, F0_NEAREST_UP = 4, F0_PREVIOUS = 5,
              F0_NEXT = 6 };

__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ uint32_t bits(float v) { return __float_as_uint(v); }
__device__ __forceinline__ uint64_t bits(double v) { return (uint64_t)__double_as_longlong(v); }

// ---- block scans ------------------------------------------------------------------------------------
__device__ __forceinline__ int shfl_up(int v, int d) { return __shfl_up_sync(0xffffffffu, v, d); }
__device__ __forceinline__ double2 shfl_up(double2 v, int d) {
  return make_double2(__shfl_up_sync(0xffffffffu, v.x, d), __shfl_up_sync(0xffffffffu, v.y, d));
}

// Inclusive scan of one value per thread in thread order, with an associative (not necessarily
// commutative) operator op(earlier, later).
template <typename V, typename Op>
__device__ __forceinline__ V block_scan(V v, Op op, V* sh_warp) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const V o = shfl_up(v, d);
    if (lane >= d) v = op(o, v);
  }
  if (lane == 31) sh_warp[warp] = v;
  __syncthreads();
  if (warp > 0) {
    V pre = sh_warp[0];
    for (int w = 1; w < warp; ++w) pre = op(pre, sh_warp[w]);
    v = op(pre, v);
  }
  __syncthreads();  // sh_warp may be reused by the next call
  return v;
}

// ---- F0 interpolation ---------------------------------------------------------------------------------
struct MaxOp { __device__ int operator()(int a, int b) const { return a > b ? a : b; } };
struct MinOp { __device__ int operator()(int a, int b) const { return a < b ? a : b; } };

template <typename T, int KIND>
__device__ __forceinline__ double f0_eval(double xa, double xb, double x, double ya, double yb) {
  if (KIND == F0_SLINEAR) {  // de Boor, k = 1: w = 1 / (xb - xa); (0 + ya h0) + yb h1
    const double w = __ddiv_rn(1.0, __dsub_rn(xb, xa));
    const double h0 = __dmul_rn(w, __dsub_rn(xb, x));
    const double h1 = __dmul_rn(w, __dsub_rn(x, xa));
    return __dadd_rn(__dmul_rn(ya, h0), __dmul_rn(yb, h1));
  } else if (KIND == F0_LINEAR) {
    if (sizeof(T) == 8) {  // float64 y: np.interp, with its retry from the right end on NaN
      const double slope = __ddiv_rn(__dsub_rn(yb, ya), __dsub_rn(xb, xa));
      double r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, xa)), ya);
      if (r != r) {
        r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, xb)), yb);
        if (r != r && ya == yb) r = ya;
      }
      return r;
    } else {  // float32 y: interp1d._call_linear
      const double dx = __dsub_rn(xb, xa);
      return __dadd_rn(__dmul_rn(__ddiv_rn(__dsub_rn(x, xa), dx), yb), __dmul_rn(__ddiv_rn(__dsub_rn(xb, x), dx), ya));
    }
  } else if (KIND == F0_ZERO || KIND == F0_PREVIOUS) {
    return ya;
  } else if (KIND == F0_NEXT) {
    return yb;
  } else {  // nearest: searchsorted over the midpoints, side left (ties down) or right (ties up)
    const double mid = __dadd_rn(__dmul_rn(xb, 0.5), __dmul_rn(xa, 0.5));
    if (KIND == F0_NEAREST) return x <= mid ? ya : yb;
    return x < mid ? ya : yb;
  }
}

template <typename T, int KIND>
__global__ void __launch_bounds__(F0_BLOCK) f0_interp_kernel(const T* __restrict__ x, T* __restrict__ out, int T_max,
                                                             const int32_t* __restrict__ lengths,
                                                             int32_t* __restrict__ prev_ws) {
  __shared__ int sh_warp[F0_BLOCK / 32];
  __shared__ int sh_first, sh_carry;
  const int b = blockIdx.x;
  const T* X = x + (size_t)b * T_max;
  T* Y = out + (size_t)b * T_max;
  int32_t* P = prev_ws + (size_t)b * T_max;
  int len = T_max;
  if (lengths) len = min(max(lengths[b], 0), T_max);
  for (int i = len + threadIdx.x; i < T_max; i += F0_BLOCK) Y[i] = X[i];  // beyond the length: unchanged
  if (threadIdx.x == 0) sh_first = INT_MAX;
  __syncthreads();
  // forward: last voiced index <= i (-1 if none)
  int carry = -1;
  for (int t0 = 0; t0 < len; t0 += F0_BLOCK) {
    const int i = t0 + threadIdx.x;
    const bool voiced = i < len && X[i] > T(0);
    if (voiced) atomicMin(&sh_first, i);
    int p = block_scan(voiced ? i : -1, MaxOp(), sh_warp);
    p = max(p, carry);
    if (i < len) P[i] = p;
    if (threadIdx.x == F0_BLOCK - 1) sh_carry = p;
    __syncthreads();
    carry = sh_carry;
    __syncthreads();
  }
  const int last = carry, first = sh_first;
  if (last < 0) {  // no voiced frame: the row is unchanged
    for (int i = threadIdx.x; i < len; i += F0_BLOCK) Y[i] = X[i];
    return;
  }
  const double y_first = (double)X[first], y_last = (double)X[last];
  // backward: next voiced index >= i (INT_MAX if none), and the output
  int ncarry = INT_MAX;
  const int n_tiles = (len + F0_BLOCK - 1) / F0_BLOCK;
  for (int tile = n_tiles - 1; tile >= 0; --tile) {
    const int i = tile * F0_BLOCK + (F0_BLOCK - 1 - threadIdx.x);  // thread order runs backwards in time
    const T v = i >= 0 && i < len ? X[i] : T(0);
    const bool voiced = i >= 0 && i < len && v > T(0);
    int nx = block_scan(voiced ? i : INT_MAX, MinOp(), sh_warp);
    nx = min(nx, ncarry);
    if (i >= 0 && i < len) {
      double r;
      if (i == 0) r = y_first;
      else if (i == len - 1) r = y_last;
      else if (!(v <= T(0))) r = (double)v;  // voiced, or NaN (neither voiced nor filled)
      else {
        const int pa = P[i];
        const int a = pa < 0 ? 0 : pa;
        const int bb = nx == INT_MAX ? len - 1 : nx;
        const double ya = pa < 0 ? y_first : (double)X[a];
        const double yb = nx == INT_MAX ? y_last : (double)X[bb];
        r = f0_eval<T, KIND>((double)a, (double)bb, (double)i, ya, yb);
      }
      Y[i] = (T)r;
    }
    if (threadIdx.x == F0_BLOCK - 1) sh_carry = nx;
    __syncthreads();
    ncarry = sh_carry;
    __syncthreads();
  }
}

// ---- pre-emphasis (FIR) -------------------------------------------------------------------------------
// Row r, samples [t0, t0 + V) per thread; 16-byte loads when the row start is aligned.
template <typename T>
__global__ void __launch_bounds__(PE_BLOCK) preemph_fir_kernel(const T* __restrict__ x, T* __restrict__ out, int64_t rows,
                                                               int64_t T_max, const int32_t* __restrict__ lengths, T nc,
                                                               bool vec) {
  constexpr int V = PE_VEC_BYTES / (int)sizeof(T);
  const int64_t per_row = (T_max + V - 1) / V;
  for (int64_t r = blockIdx.y; r < rows; r += gridDim.y) {
    const T* X = x + r * T_max;
    T* Y = out + r * T_max;
    const int64_t len = lengths ? min((int64_t)max(lengths[r], 0), T_max) : T_max;
    for (int64_t g = (int64_t)blockIdx.x * PE_BLOCK + threadIdx.x; g < per_row; g += (int64_t)gridDim.x * PE_BLOCK) {
      const int64_t t0 = g * V;
      T v[V];
      if (vec && t0 + V <= T_max) {
        if (sizeof(T) == 4) {
          const float4 q = __ldcs(reinterpret_cast<const float4*>(X + t0));
          reinterpret_cast<float*>(v)[0] = q.x; reinterpret_cast<float*>(v)[1] = q.y;
          reinterpret_cast<float*>(v)[2] = q.z; reinterpret_cast<float*>(v)[3] = q.w;
        } else {
          const double2 q = __ldcs(reinterpret_cast<const double2*>(X + t0));
          reinterpret_cast<double*>(v)[0] = q.x; reinterpret_cast<double*>(v)[1] = q.y;
        }
      } else {
#pragma unroll
        for (int k = 0; k < V; ++k) v[k] = t0 + k < T_max ? X[t0 + k] : T(0);
      }
      T prev = t0 > 0 ? X[t0 - 1] : T(0);
      T y[V];
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const int64_t t = t0 + k;
        const T s = add_rn(T(0), v[k]);
        y[k] = t >= len ? v[k] : (t == 0 ? s : add_rn(s, mul_rn(nc, prev)));
        prev = v[k];
      }
      if (vec && t0 + V <= T_max) {
        if (sizeof(T) == 4) {
          const float* f = reinterpret_cast<const float*>(y);
          __stcs(reinterpret_cast<float4*>(Y + t0), make_float4(f[0], f[1], f[2], f[3]));
        } else {
          const double* d = reinterpret_cast<const double*>(y);
          __stcs(reinterpret_cast<double2*>(Y + t0), make_double2(d[0], d[1]));
        }
      } else {
#pragma unroll
        for (int k = 0; k < V; ++k)
          if (t0 + k < T_max) Y[t0 + k] = y[k];
      }
    }
  }
}

// ---- inverse pre-emphasis (IIR) -------------------------------------------------------------------------
// One exact step of scipy's _linear_filter with b = [1, 0], a = [1, a1]: y = z + x; z' = x * 0 - y * a1.
template <typename T>
__device__ __forceinline__ T iir_step(T& z, T xt, T a1) {
  const T y = add_rn(z, xt);
  z = sub_rn(mul_rn(xt, T(0)), mul_rn(y, a1));
  return y;
}

struct IirShape {
  int64_t rows, T_max;
  int n_ck;   // chunks per row
  int W;      // warm-up samples
};

// Estimate segment m (m = 1 .. n_ck - 1) of a row ends at sample m L - W - 1: segment m covers
// [max(0, (m - 1) L - W), m L - W - 1].  est[2 k] = zero-state end value, est[2 k + 1] = c^len (float64).
template <typename T>
__global__ void __launch_bounds__(IIR_BLOCK) preemph_est_kernel(const T* __restrict__ x, IirShape s,
                                                                const int32_t* __restrict__ lengths, double c,
                                                                double* __restrict__ est) {
  const int64_t k = (int64_t)blockIdx.x * IIR_BLOCK + threadIdx.x;
  if (k >= s.rows * s.n_ck) return;
  const int64_t r = k / s.n_ck;
  const int m = (int)(k % s.n_ck);
  const int64_t len = lengths ? min((int64_t)max(lengths[r], 0), s.T_max) : s.T_max;
  const int64_t hi = (int64_t)m * IIR_L - s.W - 1;  // last sample of the segment
  double e = 0.0, p = 1.0;
  if (m > 0 && hi >= 0 && hi < len) {
    const T* X = x + r * s.T_max;
    for (int64_t t = max((int64_t)0, (int64_t)(m - 1) * IIR_L - s.W); t <= hi; ++t) {
      e = fma(c, e, (double)X[t]);
      p *= c;
    }
  }
  est[2 * k] = e;
  est[2 * k + 1] = p;
}

// One CTA per row: state[m] = e_m + p_m * state[m - 1] (state[0] = 0) as a scan of affine maps, in place
// of est[2 k]: the estimate of y at sample m L - W - 1.
__global__ void __launch_bounds__(IIR_SCAN) preemph_carry_kernel(IirShape s, double* __restrict__ est) {
  __shared__ double2 sh_warp[IIR_SCAN / 32];
  __shared__ double sh_carry;
  double* E = est + (size_t)blockIdx.x * s.n_ck * 2;
  if (threadIdx.x == 0) sh_carry = 0.0;
  __syncthreads();
  struct Compose {  // (p1, e1) then (p2, e2): y -> p2 (p1 y + e1) + e2
    __device__ double2 operator()(double2 f, double2 g) const { return make_double2(f.x * g.x, fma(g.x, f.y, g.y)); }
  };
  for (int m0 = 0; m0 < s.n_ck; m0 += IIR_SCAN) {
    const int m = m0 + threadIdx.x;
    double2 f = make_double2(1.0, 0.0);
    if (m < s.n_ck) f = make_double2(E[2 * m + 1], E[2 * m]);
    f = block_scan(f, Compose(), sh_warp);
    const double carry = sh_carry;
    const double st = fma(f.x, carry, f.y);
    if (m < s.n_ck) E[2 * m] = st;
    __syncthreads();
    if (threadIdx.x == IIR_SCAN - 1) sh_carry = st;
    __syncthreads();
  }
}

// One thread per chunk: outputs of [m L, m L + L) from a speculative start; spec[2 k] = y at m L - 1 (the
// state the chunk starts from), spec[2 k + 1] = y at the chunk's last sample.  Chunk 0, and a chunk whose
// warm-up would reach before sample 0, starts exactly from scipy's zero state.  Samples at or beyond the
// row's length are copied unchanged.
template <typename T>
__global__ void __launch_bounds__(IIR_BLOCK) preemph_spec_kernel(const T* __restrict__ x, T* __restrict__ out, IirShape s,
                                                                 const int32_t* __restrict__ lengths, T a1,
                                                                 const double* __restrict__ est, T* __restrict__ spec) {
  const int64_t k = (int64_t)blockIdx.x * IIR_BLOCK + threadIdx.x;
  if (k >= s.rows * s.n_ck) return;
  const int64_t r = k / s.n_ck;
  const int m = (int)(k % s.n_ck);
  const int64_t len = lengths ? min((int64_t)max(lengths[r], 0), s.T_max) : s.T_max;
  const T* X = x + r * s.T_max;
  T* Y = out + r * s.T_max;
  const int64_t c0 = (int64_t)m * IIR_L, c1 = min(c0 + IIR_L, s.T_max);
  for (int64_t t = max(c0, len); t < c1; ++t) Y[t] = X[t];
  const int64_t e1 = min(c1, len);
  if (c0 >= e1) return;
  const int64_t q = c0 - s.W - 1;  // the sample whose estimated y starts the warm-up
  T z = T(0), y_prev = T(0);
  int64_t t = 0;
  if (m > 0 && q >= 0) {
    y_prev = (T)est[2 * k];
    const T xq = X[q];
    z = sub_rn(mul_rn(xq, T(0)), mul_rn(y_prev, a1));
    t = q + 1;
  }
  for (; t < c0; ++t) y_prev = iir_step(z, X[t], a1);
  spec[2 * k] = y_prev;
  for (; t < e1; ++t) {
    y_prev = iir_step(z, X[t], a1);
    Y[t] = y_prev;
  }
  spec[2 * k + 1] = y_prev;
}

// One CTA per row.  Chunk m is exact when its start state equals the true end state of chunk m - 1
// bitwise; otherwise thread 0 reruns it from the true state and stops at the first output that equals the
// stored one bitwise.  Tiles of IIR_SCAN chunks are tested in parallel, so only mismatching chunks are
// walked.  counters[0] += chunks rerun, counters[1] += samples rewritten.
template <typename T>
__global__ void __launch_bounds__(IIR_SCAN) preemph_repair_kernel(const T* __restrict__ x, T* __restrict__ out, IirShape s,
                                                                  const int32_t* __restrict__ lengths, T a1,
                                                                  const T* __restrict__ spec,
                                                                  unsigned long long* __restrict__ counters) {
  __shared__ unsigned sh_mask[IIR_SCAN / 32];
  __shared__ int sh_any;
  const int64_t r = blockIdx.x;
  const int64_t len = lengths ? min((int64_t)max(lengths[r], 0), s.T_max) : s.T_max;
  const int n_live = (int)((len + IIR_L - 1) / IIR_L);
  const T* X = x + r * s.T_max;
  T* Y = out + r * s.T_max;
  const T* S = spec + (size_t)r * s.n_ck * 2;
  T true_end = n_live > 0 ? S[1] : T(0);  // chunk 0 is exact
  bool end_is_spec = true;                 // true_end == S[2 (m - 1) + 1]
  unsigned long long n_chunks = 0, n_samples = 0;
  for (int m0 = 1; m0 < n_live; m0 += IIR_SCAN) {
    const int m = m0 + threadIdx.x;
    bool bad = false;
    if (m < n_live) bad = bits(S[2 * m]) != bits(S[2 * (m - 1) + 1]);
    const unsigned ballot = __ballot_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0) sh_mask[threadIdx.x >> 5] = ballot;
    if (threadIdx.x == 0) sh_any = 0;
    __syncthreads();
    if (bad) sh_any = 1;
    __syncthreads();
    if (threadIdx.x == 0 && (sh_any || !end_is_spec)) {
      const int m_end = min(m0 + IIR_SCAN, n_live);
      int mm = m0;
      while (mm < m_end) {
        if (end_is_spec) {  // jump to the next flagged chunk
          int w = (mm - m0) >> 5;
          unsigned msk = sh_mask[w] & (0xffffffffu << ((mm - m0) & 31));
          while (!msk && ++w < IIR_SCAN / 32) msk = sh_mask[w];
          if (!msk) break;
          mm = m0 + w * 32 + __ffs(msk) - 1;
          if (mm >= m_end) break;
          true_end = S[2 * (mm - 1) + 1];
        }
        const T start = S[2 * mm];
        if (bits(start) == bits(true_end)) {
          true_end = S[2 * mm + 1];
          end_is_spec = true;
          ++mm;
          continue;
        }
        // rerun chunk mm from the true state
        ++n_chunks;
        const int64_t c0 = (int64_t)mm * IIR_L, e1 = min(c0 + IIR_L, len);
        T z = sub_rn(mul_rn(X[c0 - 1], T(0)), mul_rn(true_end, a1));
        bool merged = false;
        T yv = true_end;
        for (int64_t t = c0; t < e1; ++t) {
          yv = iir_step(z, X[t], a1);
          if (bits(yv) == bits(Y[t])) { merged = true; break; }
          Y[t] = yv;
          ++n_samples;
        }
        if (merged) {
          true_end = S[2 * mm + 1];
          end_is_spec = true;
        } else {
          true_end = yv;
          end_is_spec = false;
        }
        ++mm;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0 && n_chunks) {
    atomicAdd(counters, n_chunks);
    atomicAdd(counters + 1, n_samples);
  }
}

// W: samples for a perturbation of the start state to decay below the dtype's rounding unit,
// ln(2^-p) / ln|c| (p = 24 or 53), rounded up to 32 and capped at IIR_W_MAX; 0 when |c| >= 1 or c is not
// finite (the repair walk is then the sequential filter).
static int iir_warmup(double c, int dtype) {
  const double a = fabs(c);
  if (!(a < 1.0) || a == 0.0) return 0;
  const double w = (dtype == NNK_F32 ? -24.0 : -53.0) * 0.6931471805599453 / log(a);
  if (!(w < IIR_W_MAX)) return IIR_W_MAX;
  return ((int)ceil(w) + 31) / 32 * 32;
}

static IirShape iir_shape(int64_t rows, int64_t T_max, double c, int dtype) {
  IirShape s{};
  s.rows = rows;
  s.T_max = T_max;
  s.n_ck = (int)((T_max + IIR_L - 1) / IIR_L);
  s.W = iir_warmup(c, dtype);
  return s;
}

static int64_t iir_ws_bytes(const IirShape& s, int dtype) {
  const int64_t n = s.rows * (int64_t)s.n_ck;
  const int64_t es = dtype == NNK_F32 ? 4 : 8;
  return n * 16 + ((n * 2 * es + 15) / 16) * 16;
}

// ---- mu-law ---------------------------------------------------------------------------------------------
// float32 log1p / pow are evaluated in float64 and rounded once.
__device__ __forceinline__ float log1p_t(float v) { return __double2float_rn(log1p((double)v)); }
__device__ __forceinline__ double log1p_t(double v) { return log1p(v); }
__device__ __forceinline__ float pow_t(float b, float e) { return __double2float_rn(pow((double)b, (double)e)); }
__device__ __forceinline__ double pow_t(double b, double e) { return pow(b, e); }
template <typename T> __device__ __forceinline__ T sign_np(T v) {  // np.sign: -1, 0, +1, NaN
  return v > T(0) ? T(1) : (v < T(0) ? T(-1) : (v == T(0) ? T(0) : v));
}
template <typename Tin, typename T> __device__ __forceinline__ T to_t(Tin v) { return (T)v; }
template <> __device__ __forceinline__ float to_t<long long, float>(long long v) { return __ll2float_rn(v); }
template <> __device__ __forceinline__ float to_t<int, float>(int v) { return __int2float_rn(v); }
template <> __device__ __forceinline__ float to_t<double, float>(double v) { return __double2float_rn(v); }

// MODE 0 mulaw, 1 inv_mulaw, 2 mulaw_quantize, 3 inv_mulaw_quantize.
template <int MODE, typename Tin, typename Tc, typename Ty, typename Tout>
__global__ void __launch_bounds__(MU_BLOCK) mulaw_kernel(const Tin* __restrict__ x, Tout* __restrict__ out, int64_t n,
                                                         double mu) {
  const Tc mu_c = (Tc)mu;
  for (int64_t i = (int64_t)blockIdx.x * MU_BLOCK + threadIdx.x; i < n; i += (int64_t)gridDim.x * MU_BLOCK) {
    if (MODE == 0 || MODE == 2) {
      const Tc v = (Tc)x[i];
      const Tc t = mul_rn(sign_np(v), log1p_t(mul_rn(mu_c, fabs(v))));
      const Ty y = div_rn((Ty)t, (Ty)log1p(mu));  // / np.log1p(mu): float64 for NumPy, the tensor's dtype for torch
      if (MODE == 0) {
        out[i] = (Tout)y;
      } else {
        const Ty q = mul_rn(div_rn(add_rn(y, Ty(1)), Ty(2)), (Ty)mu);
        out[i] = (Tout)__double2ll_rz((double)q);
      }
    } else {
      Tc v;
      if (MODE == 3) v = sub_rn(div_rn(mul_rn(Tc(2), to_t<Tin, Tc>(x[i])), mu_c), Tc(1));
      else v = (Tc)x[i];
      const Tc s = mul_rn(sign_np(v), (Tc)(1.0 / mu));
      const Tc p = sub_rn(pow_t((Tc)(1.0 + mu), fabs(v)), Tc(1));
      out[i] = (Tout)mul_rn(s, p);
    }
  }
}

template <int MODE, typename Tin, typename Tc, typename Ty, typename Tout>
static void launch_mulaw(const void* x, void* out, int64_t n, double mu, cudaStream_t st) {
  int64_t g = (n + MU_BLOCK - 1) / MU_BLOCK;
  if (g > (int64_t)kNumSMs * 16) g = (int64_t)kNumSMs * 16;
  mulaw_kernel<MODE, Tin, Tc, Ty, Tout><<<(unsigned)g, MU_BLOCK, 0, st>>>(reinterpret_cast<const Tin*>(x),
                                                                         reinterpret_cast<Tout*>(out), n, mu);
}

template <typename T>
static void launch_f0(const void* x, void* out, int B, int T_max, const int32_t* lengths, int kind, int32_t* ws,
                      cudaStream_t st) {
  const T* xp = reinterpret_cast<const T*>(x);
  T* op = reinterpret_cast<T*>(out);
  switch (kind) {
    case F0_LINEAR: f0_interp_kernel<T, F0_LINEAR><<<B, F0_BLOCK, 0, st>>>(xp, op, T_max, lengths, ws); break;
    case F0_SLINEAR: f0_interp_kernel<T, F0_SLINEAR><<<B, F0_BLOCK, 0, st>>>(xp, op, T_max, lengths, ws); break;
    case F0_ZERO: f0_interp_kernel<T, F0_ZERO><<<B, F0_BLOCK, 0, st>>>(xp, op, T_max, lengths, ws); break;
    case F0_NEAREST: f0_interp_kernel<T, F0_NEAREST><<<B, F0_BLOCK, 0, st>>>(xp, op, T_max, lengths, ws); break;
    case F0_NEAREST_UP: f0_interp_kernel<T, F0_NEAREST_UP><<<B, F0_BLOCK, 0, st>>>(xp, op, T_max, lengths, ws); break;
    case F0_PREVIOUS: f0_interp_kernel<T, F0_PREVIOUS><<<B, F0_BLOCK, 0, st>>>(xp, op, T_max, lengths, ws); break;
    default: f0_interp_kernel<T, F0_NEXT><<<B, F0_BLOCK, 0, st>>>(xp, op, T_max, lengths, ws); break;
  }
}

template <typename T>
static int run_preemph(const void* x, void* out, int64_t rows, int64_t T_max, const int32_t* lengths, double coef,
                       int inverse, void* workspace, int64_t workspace_bytes, unsigned long long* counters,
                       int dtype, cudaStream_t st) {
  const T* xp = reinterpret_cast<const T*>(x);
  T* op = reinterpret_cast<T*>(out);
  const T c = (T)coef;  // np.array([1.0, -coef], x.dtype)
  if (!inverse) {
    const int V = PE_VEC_BYTES / (int)sizeof(T);
    const bool vec = T_max % V == 0 && ((uintptr_t)x % PE_VEC_BYTES) == 0 && ((uintptr_t)out % PE_VEC_BYTES) == 0;
    const int64_t per_row = (T_max + V - 1) / V;
    int64_t gx = (per_row + PE_BLOCK - 1) / PE_BLOCK;
    int64_t gy = rows < 65535 ? rows : 65535;
    const int64_t cap = (int64_t)kNumSMs * 32;
    if (gx > cap) gx = cap;
    if (gx * gy > cap * 8 && gy > 1) gy = (cap * 8 + gx - 1) / gx;
    preemph_fir_kernel<T><<<dim3((unsigned)gx, (unsigned)gy), PE_BLOCK, 0, st>>>(xp, op, rows, T_max, lengths, -c, vec);
    count_launch();
    NNK_CUDA_CHECK(cudaGetLastError());
    return NNK_OK;
  }
  NNK_REQUIRE(counters, NNK_ERR_ARG, "NULL counters");
  NNK_REQUIRE(rows <= 0x7fffffff, NNK_ERR_ARG, "too many rows");
  const IirShape s = iir_shape(rows, T_max, (double)c, dtype);
  NNK_REQUIRE(workspace && workspace_bytes >= iir_ws_bytes(s, dtype), NNK_ERR_WORKSPACE,
              "preemphasis workspace too small");
  double* est = reinterpret_cast<double*>(workspace);
  const int64_t n = rows * (int64_t)s.n_ck;
  T* spec = reinterpret_cast<T*>(reinterpret_cast<char*>(workspace) + n * 16);
  const T a1 = -c;
  NNK_CUDA_CHECK(cudaMemsetAsync(counters, 0, 2 * sizeof(unsigned long long), st));
  const unsigned g = (unsigned)((n + IIR_BLOCK - 1) / IIR_BLOCK);
  preemph_est_kernel<T><<<g, IIR_BLOCK, 0, st>>>(xp, s, lengths, (double)c, est);
  preemph_carry_kernel<<<(unsigned)rows, IIR_SCAN, 0, st>>>(s, est);
  preemph_spec_kernel<T><<<g, IIR_BLOCK, 0, st>>>(xp, op, s, lengths, a1, est, spec);
  preemph_repair_kernel<T><<<(unsigned)rows, IIR_SCAN, 0, st>>>(xp, op, s, lengths, a1, spec, counters);
  count_launch(4);
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

}  // namespace nnk

using namespace nnk;

extern "C" int64_t nnk_f0_interp_workspace_bytes(int32_t B, int32_t T_max) {
  return (int64_t)(B > 0 ? B : 0) * (T_max > 0 ? T_max : 0) * 4;
}

extern "C" int nnk_f0_interp(const void* x, void* out, int32_t dtype, int32_t B, int32_t T_max, const int32_t* lengths,
                             int32_t kind, void* workspace, int64_t workspace_bytes, void* stream) {
  NNK_REQUIRE(out, NNK_ERR_ARG, "NULL output");
  DeviceGuard guard(out);
  NNK_REQUIRE(dtype == NNK_F32 || dtype == NNK_F64, NNK_ERR_ARG, "bad dtype");
  NNK_REQUIRE(kind >= F0_LINEAR && kind <= F0_NEXT, NNK_ERR_ARG, "bad kind");
  NNK_REQUIRE(B >= 0 && T_max >= 0, NNK_ERR_ARG, "bad size");
  if (B == 0 || T_max == 0) return NNK_OK;
  NNK_REQUIRE(x, NNK_ERR_ARG, "NULL input");
  NNK_REQUIRE(workspace && workspace_bytes >= nnk_f0_interp_workspace_bytes(B, T_max), NNK_ERR_WORKSPACE,
              "f0 workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* ws = reinterpret_cast<int32_t*>(workspace);
  if (dtype == NNK_F32) launch_f0<float>(x, out, B, T_max, lengths, kind, ws, st);
  else launch_f0<double>(x, out, B, T_max, lengths, kind, ws, st);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

extern "C" int64_t nnk_preemphasis_workspace_bytes(int32_t dtype, int64_t rows, int64_t T_max, double coef,
                                                   int32_t inverse) {
  if (!inverse || rows <= 0 || T_max <= 0) return 0;
  const double c = dtype == NNK_F32 ? (double)(float)coef : coef;
  return iir_ws_bytes(iir_shape(rows, T_max, c, dtype), dtype);
}

extern "C" int nnk_preemphasis(const void* x, void* out, int32_t dtype, int64_t rows, int64_t T_max,
                               const int32_t* lengths, double coef, int32_t inverse, void* workspace,
                               int64_t workspace_bytes, unsigned long long* counters, void* stream) {
  NNK_REQUIRE(out, NNK_ERR_ARG, "NULL output");
  DeviceGuard guard(out);
  NNK_REQUIRE(dtype == NNK_F32 || dtype == NNK_F64, NNK_ERR_ARG, "bad dtype");
  NNK_REQUIRE(rows >= 0 && T_max >= 0, NNK_ERR_ARG, "bad size");
  if (rows == 0 || T_max == 0) return NNK_OK;
  NNK_REQUIRE(x, NNK_ERR_ARG, "NULL input");
  NNK_REQUIRE((T_max + IIR_L - 1) / IIR_L <= 0x7fffffff, NNK_ERR_ARG, "row too long");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == NNK_F32)
    return run_preemph<float>(x, out, rows, T_max, lengths, coef, inverse, workspace, workspace_bytes, counters, dtype, st);
  return run_preemph<double>(x, out, rows, T_max, lengths, coef, inverse, workspace, workspace_bytes, counters, dtype, st);
}

extern "C" int nnk_mulaw(const void* x, int32_t in_type, void* out, int32_t mode, int32_t variant, int64_t n, double mu,
                         void* stream) {
  NNK_REQUIRE(out, NNK_ERR_ARG, "NULL output");
  DeviceGuard guard(out);
  NNK_REQUIRE(mode >= 0 && mode <= 3, NNK_ERR_ARG, "bad mode");
  NNK_REQUIRE(n >= 0, NNK_ERR_ARG, "bad size");
  if (n == 0) return NNK_OK;
  NNK_REQUIRE(x, NNK_ERR_ARG, "NULL input");
  cudaStream_t st = (cudaStream_t)stream;
  typedef long long i64;
  bool ok = true;
  if (mode == 0 || mode == 2) {
    // variant 0: float32 NumPy (float64 division), 1: float32 tensor, 2: float64
    const bool f32 = in_type == NNK_F32;
    ok = (variant == 2) == !f32 && (variant <= 2) && (in_type == NNK_F32 || in_type == NNK_F64);
    if (ok && mode == 0) {
      if (variant == 0) launch_mulaw<0, float, float, double, double>(x, out, n, mu, st);
      else if (variant == 1) launch_mulaw<0, float, float, float, float>(x, out, n, mu, st);
      else launch_mulaw<0, double, double, double, double>(x, out, n, mu, st);
    } else if (ok) {
      if (variant == 0) launch_mulaw<2, float, float, double, i64>(x, out, n, mu, st);
      else if (variant == 1) launch_mulaw<2, float, float, float, i64>(x, out, n, mu, st);
      else launch_mulaw<2, double, double, double, i64>(x, out, n, mu, st);
    }
  } else if (mode == 1) {
    ok = (in_type == NNK_F32 && variant == 1) || (in_type == NNK_F64 && variant == 2);
    if (ok && variant == 1) launch_mulaw<1, float, float, float, float>(x, out, n, mu, st);
    else if (ok) launch_mulaw<1, double, double, double, double>(x, out, n, mu, st);
  } else {
    // variant 1: float32 chain from float32 / float64 / int32 / int64 codes, 2: float64 chain (Python scalar)
    if (variant == 2) {
      ok = in_type == NNK_F64;
      if (ok) launch_mulaw<3, double, double, double, double>(x, out, n, mu, st);
    } else if (variant == 1) {
      switch (in_type) {
        case NNK_F32: launch_mulaw<3, float, float, float, float>(x, out, n, mu, st); break;
        case NNK_F64: launch_mulaw<3, double, float, float, float>(x, out, n, mu, st); break;
        case NNK_I32: launch_mulaw<3, int, float, float, float>(x, out, n, mu, st); break;
        case NNK_I64: launch_mulaw<3, i64, float, float, float>(x, out, n, mu, st); break;
        default: ok = false;
      }
    } else {
      ok = false;
    }
  }
  NNK_REQUIRE(ok, NNK_ERR_ARG, "bad input type / variant for this mode");
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}
