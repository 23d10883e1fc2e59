// nnk_modspec.cu -- modulation spectrum: preprocessing.modspec / inv_modspec / modspec_smoothing and the
// gradient of autograd.ModSpec (C ABI: include/nnk_b200.h).
//
// modspec_kernel<T, LOGN>: one CTA per (utterance, feature column).  The n real frames are packed as
// z_t = x_{2t} + i x_{2t+1} (M = n / 2 complex points) into shared memory in bit-reversed order, and an
// in-place radix-2 decimation-in-time FFT gives Z in natural order.  One pass over the bin pairs (k, M - k)
// splits Z into the real spectrum X_k = E_k + W^k O_k, X_{M-k} = conj(E_k - W^k O_k) (E, O: the spectra of the
// even and odd frames, W = e^{-2 pi i / n}), applies the mode's operation, and -- for the modes that go back to
// frames -- packs the new half spectrum C into Z'_k = (C_k + conj(C_{M-k})) + i conj(W^k) (C_k - conj(C_{M-k})),
// in place.  A decimation-in-frequency inverse FFT of Z' leaves n irfft(C) in bit-reversed order, read straight
// into the output frames.  The spectrum never leaves shared memory.  Twiddles W^j, j < M, are one table per CTA
// (sincospi), which also serves the FFT stages (e^{-2 pi i p / len} = W^{p n / len}).
//
// The MS post-filter (postfilters.modspec_post_filter) is two modes of the same kernel: the log power, whose
// moments over utterances are the filter's statistics, and the filter itself, which rescales each bin's log
// power in the bin-pair pass and goes back to frames like smoothing.
#include "nnk_common.cuh"
#include "nnk_fft.cuh"

namespace nnk {

constexpr int MS_MAX_THREADS = 256;
constexpr int MS_LOGN_MIN = 8, MS_LOGN_MAX = 12;  // n = 256 .. 4096

struct MsArgs {
  const void* in;
  const void* in2;
  void* out;
  void* out2;
  int B, T_in, T_out, D;
  const int32_t* lengths;
  double fwd_scale, inv_scale;
  int limit_bin, log_domain, mode;
};

template <int LOGN> constexpr int ms_threads() { return (1 << (LOGN - 2)) < MS_MAX_THREADS ? (1 << (LOGN - 2)) : MS_MAX_THREADS; }

// PF selects the post-filter instance (modes 4 and 5); the other instance runs modes 0 to 3.  Separate instances
// keep log / exp out of the register allocation of modes 0 to 3: one runtime switch over all six modes gave the
// float64 instances 64 registers and 24-36 B of spills instead of 72-80 registers and none.
template <typename T, int LOGN, bool PF>
__global__ void __launch_bounds__(ms_threads<LOGN>()) modspec_kernel(MsArgs a) {
  using V = typename Cx<T>::V;
  constexpr int N = 1 << LOGN, LOGM = LOGN - 1, M = N / 2, NT = ms_threads<LOGN>();
  constexpr int K = M + 1;
  extern __shared__ __align__(16) unsigned char ms_smem[];
  V* z = reinterpret_cast<V*>(ms_smem);
  V* tw = z + M;
  const int tid = threadIdx.x, d = blockIdx.x, D = a.D;
  const int mode = a.mode;
  const bool reads_x = PF || mode != NNK_MS_INVERSE;
  const bool writes_frames = PF ? mode == NNK_MS_POSTFILTER : mode != NNK_MS_POWER;
  const T fs = (T)a.fwd_scale;
  for (int j = tid; j < M; j += NT) {  // W^j = e^{-2 pi i j / n}
    T s, c;
    sincospi_t(T(2 * j) / T(N), &s, &c);
    tw[j] = cx<V>(c, -s);
  }
  for (int b = blockIdx.y; b < a.B; b += gridDim.y) {
    int cap = N;
    if (reads_x) cap = min(cap, a.T_in);
    if (writes_frames) cap = min(cap, a.T_out);
    const int len = a.lengths ? min(max(a.lengths[b], 0), cap) : cap;
    const size_t spec_row = (size_t)b * K * D + d;  // bin 0 of column d in a (B, K, D) array
    if (reads_x) {
      const T* x = reinterpret_cast<const T*>(a.in) + (size_t)b * a.T_in * D + d;
      for (int t = tid; t < M; t += NT) {
        const T x0 = 2 * t < len ? x[(size_t)(2 * t) * D] : T(0);
        const T x1 = 2 * t + 1 < len ? x[(size_t)(2 * t + 1) * D] : T(0);
        z[__brev(t) >> (32 - LOGM)] = cx<V>(x0, x1);
      }
      __syncthreads();
#pragma unroll
      for (int s = 1; s <= LOGM; ++s) {  // decimation in time: bit-reversed in, natural out
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
    // bin pairs (k, M - k), k = 0 .. M / 2; pair 0 is (0, M), both from Z_0
    for (int k = tid; k <= M / 2; k += NT) {
      const int j = M - k;
      V Ck, Cj;  // the half spectrum that goes back to frames, at bins k and j
      if (!PF && mode == NNK_MS_INVERSE) {
        const T* P = reinterpret_cast<const T*>(a.in) + spec_row;
        const V* Ph = reinterpret_cast<const V*>(a.in2) + spec_row;
        Ck = scale(Ph[(size_t)k * D], sqrt(P[(size_t)k * D]));
        Cj = scale(Ph[(size_t)j * D], sqrt(P[(size_t)j * D]));
      } else {
        V Xk, Xj;
        if (k == 0) {
          const V z0 = z[0];
          Xk = cx<V>(z0.x + z0.y, 0);
          Xj = cx<V>(z0.x - z0.y, 0);
        } else {
          const V zk = z[k], zj = z[j];
          const V E = cx<V>((zk.x + zj.x) * T(0.5), (zk.y - zj.y) * T(0.5));
          const V O = cx<V>((zk.y + zj.y) * T(0.5), (zj.x - zk.x) * T(0.5));
          const V WO = cmul(tw[k], O);
          Xk = cadd(E, WO);
          Xj = conj_(csub(E, WO));
        }
        const V Yk = scale(Xk, fs), Yj = scale(Xj, fs);
        if (!writes_frames) {  // power (PF: log power)
          T* P = reinterpret_cast<T*>(a.out) + spec_row;
          V* Ph = reinterpret_cast<V*>(a.out2) + spec_row;
          const T pk = Yk.x * Yk.x + Yk.y * Yk.y;
          P[(size_t)k * D] = PF ? log_power(pk) : pk;
          if (!PF && a.out2) Ph[(size_t)k * D] = unit_phase(Yk);
          if (j != k) {
            const T pj = Yj.x * Yj.x + Yj.y * Yj.y;
            P[(size_t)j * D] = PF ? log_power(pj) : pj;
            if (!PF && a.out2) Ph[(size_t)j * D] = unit_phase(Yj);
          }
          continue;
        }
        if (PF) {  // bin 0 keeps the column's level; the (a, c) table is shared by every utterance
          const V* AC = reinterpret_cast<const V*>(a.in2) + d;
          Ck = k == 0 ? Yk : postfilter_bin(Yk, AC[(size_t)k * D]);
          Cj = postfilter_bin(Yj, AC[(size_t)j * D]);
        } else if (mode == NNK_MS_SMOOTH) {
          Ck = k < a.limit_bin ? Yk : (a.log_domain ? unit_phase(Yk) : cx<V>(0, 0));
          Cj = j < a.limit_bin ? Yj : (a.log_domain ? unit_phase(Yj) : cx<V>(0, 0));
        } else {  // gradient: sum over k of G_k Y_k e^{+i phi k t}, bins 0 and n / 2 counted twice
          const T* G = reinterpret_cast<const T*>(a.in2) + spec_row;
          const T gk = G[(size_t)k * D], gj = G[(size_t)j * D];
          Ck = scale(Yk, k == 0 ? T(2) * gk : gk);
          Cj = scale(Yj, j == M ? T(2) * gj : gj);
        }
      }
      if (k == 0) {  // imaginary parts of bins 0 and n / 2 are ignored, as irfft does
        z[0] = cx<V>(Ck.x + Cj.x, Ck.x - Cj.x);
      } else {
        const V w = tw[k];
        const V A = cadd(Ck, conj_(Cj)), Bd = csub(Ck, conj_(Cj));
        z[k] = cadd(A, times_i(cmul(conj_(w), Bd)));
        // at bin j: (C_j + conj(C_k)) + i conj(W^j) (C_j - conj(C_k)) = conj(A) + i W conj(Bd)
        if (j != k) z[j] = cadd(conj_(A), times_i(cmul(w, conj_(Bd))));
      }
    }
    if (!writes_frames) {
      __syncthreads();  // z is rewritten by the next utterance
      continue;
    }
    __syncthreads();
#pragma unroll
    for (int s = LOGM; s >= 1; --s) {  // decimation in frequency, inverse: natural in, bit-reversed out
      const int half = 1 << (s - 1);
      for (int j = tid; j < M / 2; j += NT) {
        const int p = j & (half - 1), i0 = ((j >> (s - 1)) << s) + p, i1 = i0 + half;
        const V u = z[i0], v = z[i1];
        z[i0] = cadd(u, v);
        z[i1] = cmul(csub(u, v), conj_(tw[p << (LOGN - s)]));
      }
      __syncthreads();
    }
    const T os = (T)(!PF && mode == NNK_MS_GRAD ? a.fwd_scale : a.inv_scale);
    T* y = reinterpret_cast<T*>(a.out) + (size_t)b * a.T_out * D + d;
    for (int t = tid; t < a.T_out; t += NT) {
      T v = T(0);
      if (t < len) {
        const V q = z[__brev(t >> 1) >> (32 - LOGM)];
        v = ((t & 1) ? q.y : q.x) * os;
      }
      y[(size_t)t * D] = v;
    }
    __syncthreads();
  }
}

template <typename T, int LOGN, bool PF>
static int launch_modspec(const MsArgs& a, cudaStream_t st) {
  constexpr int M = 1 << (LOGN - 1);
  const size_t smem = 2 * M * sizeof(typename Cx<T>::V);
  if (smem > 48 * 1024)  // per device: cheap enough to set on every launch
    NNK_CUDA_CHECK(cudaFuncSetAttribute(modspec_kernel<T, LOGN, PF>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)smem));
  const dim3 grid((unsigned)a.D, (unsigned)(a.B < 65535 ? a.B : 65535));
  modspec_kernel<T, LOGN, PF><<<grid, ms_threads<LOGN>(), smem, st>>>(a);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

template <typename T, bool PF>
static int dispatch_modspec(int logn, const MsArgs& a, cudaStream_t st) {
  switch (logn) {
    case 8: return launch_modspec<T, 8, PF>(a, st);
    case 9: return launch_modspec<T, 9, PF>(a, st);
    case 10: return launch_modspec<T, 10, PF>(a, st);
    case 11: return launch_modspec<T, 11, PF>(a, st);
    default: return launch_modspec<T, 12, PF>(a, st);
  }
}

}  // namespace nnk

using namespace nnk;

extern "C" int nnk_modspec(int32_t mode, int32_t dtype, int32_t n, const void* in, const void* in2, void* out,
                           void* out2, int32_t B, int32_t T_in, int32_t T_out, int32_t D, const int32_t* lengths,
                           double fwd_scale, double inv_scale, int32_t limit_bin, int32_t log_domain, void* stream) {
  NNK_REQUIRE(mode >= NNK_MS_POWER && mode <= NNK_MS_POSTFILTER, NNK_ERR_ARG, "bad mode");
  NNK_REQUIRE(dtype == NNK_F32 || dtype == NNK_F64, NNK_ERR_ARG, "bad dtype");
  int logn = 0;
  while (logn < 31 && (1 << logn) < n) ++logn;
  NNK_REQUIRE(n > 0 && (1 << logn) == n && logn >= MS_LOGN_MIN && logn <= MS_LOGN_MAX, NNK_ERR_ARG,
              "n must be 256, 512, 1024, 2048 or 4096");
  NNK_REQUIRE(B >= 0 && T_in >= 0 && T_out >= 0 && D >= 0, NNK_ERR_ARG, "bad size");
  const bool spectrum = mode == NNK_MS_POWER || mode == NNK_MS_LOGPOWER;
  if (B == 0 || D == 0 || (!spectrum && T_out == 0)) return NNK_OK;  // nothing to write
  NNK_REQUIRE(out, NNK_ERR_ARG, "NULL output");
  DeviceGuard guard(out);
  // utterances of no frames are an empty x: nothing is read from it
  NNK_REQUIRE(in || (mode != NNK_MS_INVERSE && T_in == 0), NNK_ERR_ARG, "NULL input");
  NNK_REQUIRE(in2 || mode == NNK_MS_POWER || mode == NNK_MS_SMOOTH || mode == NNK_MS_LOGPOWER, NNK_ERR_ARG,
              "NULL second input");
  NNK_REQUIRE(!out2 || mode < NNK_MS_LOGPOWER, NNK_ERR_ARG, "out2 must be NULL for the log power and the post-filter");
  MsArgs a{in, in2, out, out2, B, T_in, T_out, D, lengths, fwd_scale, inv_scale, limit_bin, log_domain, mode};
  cudaStream_t st = (cudaStream_t)stream;
  if (mode >= NNK_MS_LOGPOWER)
    return dtype == NNK_F32 ? dispatch_modspec<float, true>(logn, a, st) : dispatch_modspec<double, true>(logn, a, st);
  return dtype == NNK_F32 ? dispatch_modspec<float, false>(logn, a, st) : dispatch_modspec<double, false>(logn, a, st);
}
