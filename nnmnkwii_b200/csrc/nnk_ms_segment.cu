// nnk_ms_segment.cu -- segment-level modulation spectrum: the log power of every windowed segment (the statistics
// of postfilters.modspec_statistics(segment=L)) and the segment-level MS post-filter with its overlap-add
// (postfilters.modspec_post_filter(segment=L)).  C ABI: nnk_ms_segment in include/nnk_b200.h.
//
// ms_segment_kernel<T, LOGN, FILTER>: one CTA per (utterance, tile of P hop blocks, group of DG adjacent columns).
// Hop block i is frames [i H, (i + 1) H); it is covered by segments i and i + 1 (segment j starts at (j - 1) H),
// so the tile of blocks [p, p + P) needs segments p .. p + P and frames [(p - 1) H, (p + P + 1) H), which are
// staged once into shared memory with coalesced row loads (rows are D-contiguous).  The edge segments p and
// p + P are also computed by the neighbouring tiles: recomputing one segment costs less than exchanging it.
//
// Each warp takes one (segment, column) at a time: the L windowed frames, zero-padded to n, are packed as
// z_t = x_2t + i x_2t+1 into the warp's own n / 2 complex values of shared memory, and the radix-2 FFT, the
// bin-pair split and the inverse FFT are the ones of csrc/nnk_modspec.cu, with __syncwarp between stages instead
// of __syncthreads.  The statistics instance writes the log power and stops there.  The filter instance applies
// the (a, c) gain of each bin (the group's table is staged once per CTA), runs the inverse FFT and adds the
// segment's first L frames into the tile's result in shared memory.  Segments of one parity do not overlap, so
// the even segments write their frames and, after a barrier, the odd ones add theirs: every frame is the sum of
// its two segments' values (one IEEE addition, whose result does not depend on the order), without atomics.
// The tile is then stored once, with coalesced row stores, zeros past the utterance's length.
#include "nnk_common.cuh"
#include "nnk_fft.cuh"

namespace nnk {

constexpr int SEG_THREADS = 256, SEG_WARPS = SEG_THREADS / 32;
constexpr int SEG_LOGN_MIN = 5, SEG_LOGN_MAX = 9;  // n = 32 .. 512
constexpr int SEG_TILE_FRAMES = 256;               // frames of a tile, rounded to an even number of hop blocks
// columns of a group: 64 B of a float32 row, 64 B of a float64 row
template <typename T> constexpr int seg_cols() { return sizeof(T) == 4 ? 16 : 8; }

// hop blocks of a tile: even (the two parities of segments cover every frame of the tile once each), at least 2
static inline int seg_tile_blocks(int H) {
  const int q = (SEG_TILE_FRAMES / H) & ~1;
  return q > 2 ? q : 2;
}

struct SegArgs {
  const void* x;
  const void* table;
  void* out;
  int B, T, D, L, P, tiles;
  const int32_t* lengths;
  const int64_t* seg_off;
};

// FILTER selects the post-filter instance; the other writes the log power.  Separate instances keep exp and the
// inverse FFT out of the statistics' register allocation, as for modspec_kernel's PF.
template <typename T, int LOGN, bool FILTER>
__global__ void __launch_bounds__(SEG_THREADS) ms_segment_kernel(SegArgs a) {
  using V = typename Cx<T>::V;
  constexpr int N = 1 << LOGN, M = N / 2, LOGM = LOGN - 1, K = M + 1, DG = seg_cols<T>(), DP = DG + 1;
  extern __shared__ __align__(16) unsigned char seg_smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int L = a.L, H = L / 2, P = a.P, D = a.D, T_pad = a.T;
  const int b = blockIdx.x / a.tiles, p = (blockIdx.x % a.tiles) * P;  // utterance, first hop block of the tile
  const int d0 = blockIdx.y * DG, nd = min(DG, D - d0);
  const int len = a.lengths ? min(max(a.lengths[b], 0), T_pad) : T_pad;
  const int J = len ? (len + H - 1) / H + 1 : 0;  // segments of the utterance
  V* tw = reinterpret_cast<V*>(seg_smem);         // W^j = e^{-2 pi i j / n}, j < M
  V* z = tw + M + warp * M;                       // this warp's FFT
  V* acs = tw + M + SEG_WARPS * M;                // FILTER: (a, c) of the group, [column][bin]
  T* win = reinterpret_cast<T*>(acs + (FILTER ? DG * K : 0));
  T* xs = win + L;                // frames (p - 1) H .. (p + P + 1) H - 1 of the group, [frame][column]
  T* ys = xs + (P + 2) * H * DP;  // FILTER: frames p H .. (p + P) H - 1 of the result, [frame][column]
  T* out = reinterpret_cast<T*>(a.out);
  const size_t row0 = (size_t)b * T_pad;  // frame 0 of utterance b
  if (FILTER && p * H >= len) {  // the tile lies past the utterance: zeros
    for (int i = tid; i < P * H * DG; i += SEG_THREADS) {
      const int f = p * H + i / DG, c = i % DG;
      if (f < T_pad && c < nd) out[(row0 + f) * D + d0 + c] = T(0);
    }
    return;
  }
  if (!FILTER && p >= J) return;
  for (int j = tid; j < M; j += SEG_THREADS) {
    T s, c;
    sincospi_t(T(2 * j) / T(N), &s, &c);
    tw[j] = cx<V>(c, -s);
  }
  for (int m = tid; m < L; m += SEG_THREADS) {  // periodic Hann window
    T s, c;
    sincospi_t(T(2 * m) / T(L), &s, &c);
    win[m] = T(0.5) - T(0.5) * c;
  }
  const T* x = reinterpret_cast<const T*>(a.x);
  const int f0 = (p - 1) * H;
  for (int i = tid; i < (P + 2) * H * DG; i += SEG_THREADS) {
    const int r = i / DG, c = i % DG, f = f0 + r;
    xs[r * DP + c] = c < nd && f >= 0 && f < len ? x[(row0 + f) * D + d0 + c] : T(0);
  }
  if (FILTER) {
    const V* AC = reinterpret_cast<const V*>(a.table);
    for (int i = tid; i < K * DG; i += SEG_THREADS) {
      const int k = i / DG, c = i % DG;
      acs[c * K + k] = c < nd ? AC[(size_t)k * D + d0 + c] : cx<V>(0, 0);
    }
  }
  __syncthreads();
  // the statistics take segments p .. p + P - 1 (each segment once over the tiles); the filter p .. p + P, the
  // even local indices q in phase 0 and the odd ones in phase 1
  for (int phase = 0; phase < (FILTER ? 2 : 1); ++phase) {
    const int nseg = FILTER ? (phase ? P / 2 : P / 2 + 1) : min(P, J - p);
    for (int item = warp; item < nseg * nd; item += SEG_WARPS) {
      const int c = item % nd, q = FILTER ? 2 * (item / nd) + phase : item / nd, j = p + q;
      __syncwarp();  // the previous item's reads of z are done
      if (FILTER && j >= J) {  // the segment starts past the utterance: it adds nothing
        if (phase == 0)
          for (int m = lane; m < L; m += 32) {
            const int r = (q - 1) * H + m;
            if (r >= 0 && r < P * H) ys[r * DP + c] = T(0);
          }
        continue;
      }
      const T* xc = xs + q * H * DP + c;
      for (int t = lane; t < M; t += 32) {
        const int m0 = 2 * t, m1 = 2 * t + 1;
        const T x0 = m0 < L ? win[m0] * xc[m0 * DP] : T(0);
        const T x1 = m1 < L ? win[m1] * xc[m1 * DP] : T(0);
        z[__brev(t) >> (32 - LOGM)] = cx<V>(x0, x1);
      }
      __syncwarp();
#pragma unroll
      for (int s = 1; s <= LOGM; ++s) {  // decimation in time: bit-reversed in, natural out
        const int half = 1 << (s - 1);
        for (int i = lane; i < M / 2; i += 32) {
          const int pp = i & (half - 1), i0 = ((i >> (s - 1)) << s) + pp, i1 = i0 + half;
          const V u = z[i0], v = cmul(z[i1], tw[pp << (LOGN - s)]);
          z[i0] = cadd(u, v);
          z[i1] = csub(u, v);
        }
        __syncwarp();
      }
      // bin pairs (k, M - k), k = 0 .. M / 2; pair 0 is (0, M), both from Z_0
      for (int k = lane; k <= M / 2; k += 32) {
        const int jb = M - k;
        V Yk, Yj;
        if (k == 0) {
          const V z0 = z[0];
          Yk = cx<V>(z0.x + z0.y, 0);
          Yj = cx<V>(z0.x - z0.y, 0);
        } else {
          const V zk = z[k], zj = z[jb];
          const V E = cx<V>((zk.x + zj.x) * T(0.5), (zk.y - zj.y) * T(0.5));
          const V O = cx<V>((zk.y + zj.y) * T(0.5), (zj.x - zk.x) * T(0.5));
          const V WO = cmul(tw[k], O);
          Yk = cadd(E, WO);
          Yj = conj_(csub(E, WO));
        }
        if (!FILTER) {  // (S, D, K): the bins of one (segment, column) are contiguous
          T* S = out + ((size_t)(a.seg_off[b] + j) * D + d0 + c) * K;
          S[k] = log_power(Yk.x * Yk.x + Yk.y * Yk.y);
          if (jb != k) S[jb] = log_power(Yj.x * Yj.x + Yj.y * Yj.y);
          continue;
        }
        const V* ac = acs + c * K;  // bin 0 keeps the segment's level
        const V Ck = k == 0 ? Yk : postfilter_bin(Yk, ac[k]);
        const V Cj = postfilter_bin(Yj, ac[jb]);
        if (k == 0) {  // imaginary parts of bins 0 and n / 2 are ignored, as irfft does
          z[0] = cx<V>(Ck.x + Cj.x, Ck.x - Cj.x);
        } else {
          const V w = tw[k];
          const V A = cadd(Ck, conj_(Cj)), Bd = csub(Ck, conj_(Cj));
          z[k] = cadd(A, times_i(cmul(conj_(w), Bd)));
          if (jb != k) z[jb] = cadd(conj_(A), times_i(cmul(w, conj_(Bd))));
        }
      }
      if (!FILTER) continue;
      __syncwarp();
#pragma unroll
      for (int s = LOGM; s >= 1; --s) {  // decimation in frequency, inverse: natural in, bit-reversed out
        const int half = 1 << (s - 1);
        for (int i = lane; i < M / 2; i += 32) {
          const int pp = i & (half - 1), i0 = ((i >> (s - 1)) << s) + pp, i1 = i0 + half;
          const V u = z[i0], v = z[i1];
          z[i0] = cadd(u, v);
          z[i1] = cmul(csub(u, v), conj_(tw[pp << (LOGN - s)]));
        }
        __syncwarp();
      }
      // overlap-add of frames 0 .. L - 1 of n irfft(C), scaled by 1 / n (exact: a power of two)
      for (int m = lane; m < L; m += 32) {
        const int r = (q - 1) * H + m;
        if (r < 0 || r >= P * H) continue;
        const V v2 = z[__brev(m >> 1) >> (32 - LOGM)];
        const T v = ((m & 1) ? v2.y : v2.x) * (T(1) / T(N));
        if (phase == 0)
          ys[r * DP + c] = v;
        else
          ys[r * DP + c] += v;
      }
    }
    __syncthreads();
  }
  if (FILTER) {
    for (int i = tid; i < P * H * DG; i += SEG_THREADS) {
      const int r = i / DG, c = i % DG, f = p * H + r;
      if (f < T_pad && c < nd) out[(row0 + f) * D + d0 + c] = f < len ? ys[r * DP + c] : T(0);
    }
  }
}

template <typename T, int LOGN, bool FILTER>
static size_t seg_smem_bytes(int L, int P) {
  using V = typename Cx<T>::V;
  constexpr int M = 1 << (LOGN - 1), DG = seg_cols<T>(), DP = DG + 1;
  const size_t H = L / 2;
  return sizeof(V) * ((size_t)M * (1 + SEG_WARPS) + (FILTER ? (size_t)DG * (M + 1) : 0)) +
         sizeof(T) * (L + (P + 2) * H * DP + (FILTER ? P * H * DP : 0));
}

template <typename T, int LOGN, bool FILTER>
static int launch_ms_segment(const SegArgs& a, cudaStream_t st) {
  const size_t smem = seg_smem_bytes<T, LOGN, FILTER>(a.L, a.P);
  if (smem > 48 * 1024)  // per device: cheap enough to set on every launch
    NNK_CUDA_CHECK(cudaFuncSetAttribute(ms_segment_kernel<T, LOGN, FILTER>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 grid((unsigned)a.B * (unsigned)a.tiles, (unsigned)((a.D + seg_cols<T>() - 1) / seg_cols<T>()));
  ms_segment_kernel<T, LOGN, FILTER><<<grid, SEG_THREADS, smem, st>>>(a);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

template <typename T, bool FILTER>
static int dispatch_ms_segment(int logn, const SegArgs& a, cudaStream_t st) {
  switch (logn) {
    case 5: return launch_ms_segment<T, 5, FILTER>(a, st);
    case 6: return launch_ms_segment<T, 6, FILTER>(a, st);
    case 7: return launch_ms_segment<T, 7, FILTER>(a, st);
    case 8: return launch_ms_segment<T, 8, FILTER>(a, st);
    default: return launch_ms_segment<T, 9, FILTER>(a, st);
  }
}

}  // namespace nnk

using namespace nnk;

extern "C" int nnk_ms_segment(int32_t mode, int32_t dtype, int32_t n, int32_t L, const void* x, const void* table,
                              void* out, int32_t B, int32_t T, int32_t D, const int32_t* lengths,
                              const int64_t* seg_off, void* stream) {
  NNK_REQUIRE(mode == NNK_MSSEG_LOGPOWER || mode == NNK_MSSEG_POSTFILTER, NNK_ERR_ARG, "bad mode");
  NNK_REQUIRE(dtype == NNK_F32 || dtype == NNK_F64, NNK_ERR_ARG, "bad dtype");
  int logn = 0;
  while (logn < 31 && (1 << logn) < n) ++logn;
  NNK_REQUIRE(n > 0 && (1 << logn) == n && logn >= SEG_LOGN_MIN && logn <= SEG_LOGN_MAX, NNK_ERR_ARG,
              "n must be 32, 64, 128, 256 or 512");
  NNK_REQUIRE(L >= 4 && L <= n && L % 2 == 0, NNK_ERR_ARG, "L must be even with 4 <= L <= n");
  NNK_REQUIRE(B >= 0 && T >= 0 && D >= 0, NNK_ERR_ARG, "bad size");
  if (B == 0 || T == 0 || D == 0) return NNK_OK;  // nothing to write
  const bool filter = mode == NNK_MSSEG_POSTFILTER;
  NNK_REQUIRE(x && out, NNK_ERR_ARG, "NULL x or output");
  NNK_REQUIRE(filter ? table != nullptr : seg_off != nullptr, NNK_ERR_ARG, "NULL table (post-filter) or seg_off");
  const int H = L / 2, P = seg_tile_blocks(H);
  // the filter covers the T frames of every utterance (zeros past its length); the statistics its segments
  const int64_t tiles = filter ? ((int64_t)T + (int64_t)P * H - 1) / ((int64_t)P * H)
                               : (((int64_t)T + H - 1) / H + 1 + P - 1) / P;
  const int dg = dtype == NNK_F32 ? seg_cols<float>() : seg_cols<double>();
  NNK_REQUIRE((int64_t)B * tiles <= 0x7fffffff && (D + dg - 1) / dg <= 65535, NNK_ERR_UNSUPPORTED,
              "batch too large for one launch");
  DeviceGuard guard(out);
  SegArgs a{x, table, out, B, T, D, L, P, (int)tiles, lengths, seg_off};
  cudaStream_t st = (cudaStream_t)stream;
  if (filter)
    return dtype == NNK_F32 ? dispatch_ms_segment<float, true>(logn, a, st) : dispatch_ms_segment<double, true>(logn, a, st);
  return dtype == NNK_F32 ? dispatch_ms_segment<float, false>(logn, a, st) : dispatch_ms_segment<double, false>(logn, a, st);
}
