// nnk_stats.cu -- corpus normalisation: per-column statistics and the per-column affine maps.
//
// Replaces the per-utterance Python loops of nnmnkwii/preprocessing/generic.py:
//   meanvar / meanstd (:496-602)  scikit-learn's _incremental_mean_and_var once per utterance
//   minmax            (:605-636)  np.minimum / np.maximum once per utterance
//   scale, inv_scale, minmax_scale, inv_minmax_scale (:639-828)  one NumPy expression each
//
// frame_stats_kernel: one pass over the valid rows computes count, mean, m2 (sum of squared deviations),
// min and max of every column, in float64 whatever the input dtype.  A tile is up to tile_rows rows of one
// utterance; a block owns a strip of CW columns (thread = column, RS row slices) and a fixed, strided set
// of tiles.  Within a tile each thread keeps shifted sums s1 = sum(x - K), s2 = sum((x - K)^2) with K
// its first value of the tile (no division per element), and turns them into (n, mean, m2) at the end
// of the tile; tiles, then the RS row slices, then the blocks combine with Chan's pairwise formula.
// The last block to finish (ticket) folds the incoming state and the block partials in index order, so
// two identical calls are bit-identical.  ~6 float64 operations per element: HBM bound.
//
// column_affine_kernel: out = (x - a[c]) / b[c] or x * b[c] + a[c] with the _rn intrinsics (no FMA
// contraction, IEEE division), i.e. bit-identical to the NumPy expression evaluated in the same dtype.
#include "nnk_common.cuh"

namespace nnk {

constexpr int ST_BLOCK = 256;           // threads per block at most (CW * RS)
constexpr int ST_LOAD_BYTES = 64;      // bytes of loads in flight per thread: 16 float32 or 8 float64 rows
constexpr int ST_ROWS_PER_THREAD = 64;  // rows a thread reads per tile
constexpr int ST_BLOCKS_PER_SM = 3;  // resident 256-thread blocks per SM (<= 80 registers)
constexpr int ST_THREADS_PER_SM = 816; // 65536 registers / 80: the grid is one wave of resident blocks
constexpr int ST_FOLD_UNROLL = 4;     // partials in flight per thread in the final fold

struct StatsParams {
  const void* x;
  int64_t ld;
  const int64_t* utt_off;
  const int32_t* lengths;
  int D, CW, RS, max_rows, tile_rows, tiles_per_utt;
  int64_t n_tiles;
  double* part;           // [gridDim.x][5][D]: n, mean, m2, min, max of every block
  unsigned int* ticket;
  double* state;          // [1 + 4 D]: count, mean, m2, min, max (in and out)
};

// NaN-propagating min / max (np.minimum / np.maximum): once a NaN is in, it stays
template <typename T> __device__ __forceinline__ T nan_min(T m, T v) { return (v < m || v != v) ? v : m; }
template <typename T> __device__ __forceinline__ T nan_max(T m, T v) { return (v > m || v != v) ? v : m; }

// (na, ma, qa) <- (na, ma, qa) + (nb, mb, qb): Chan, Golub & LeVeque's pairwise update of (n, mean, m2)
__device__ __forceinline__ void chan_merge(double& na, double& ma, double& qa, double nb, double mb, double qb) {
  if (nb == 0.0) return;
  if (na == 0.0) { na = nb; ma = mb; qa = qb; return; }
  const double n = na + nb;
  const double delta = mb - ma;
  const double f = nb / n;
  ma = ma + delta * f;
  qa = qa + qb + delta * delta * (na * f);
  na = n;
}

template <typename T>
__global__ void __launch_bounds__(ST_BLOCK, ST_BLOCKS_PER_SM) frame_stats_kernel(const __grid_constant__ StatsParams p) {
  __shared__ double sh_n[ST_BLOCK], sh_mean[ST_BLOCK], sh_m2[ST_BLOCK], sh_mn[ST_BLOCK], sh_mx[ST_BLOCK];
  __shared__ bool last;
  constexpr int ST_UNROLL = ST_LOAD_BYTES / (int)sizeof(T);
  const int D = p.D, RS = p.RS;
  const int cl = threadIdx.x % p.CW, rs = threadIdx.x / p.CW;
  const int c = blockIdx.y * p.CW + cl;
  const bool col_ok = c < D;
  const T* X = reinterpret_cast<const T*>(p.x) + (col_ok ? c : 0);
  double n = 0.0, mean = 0.0, m2 = 0.0;
  T mn = T(INFINITY), mx = T(-INFINITY);
  for (int64_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    const int u = (int)(tile / p.tiles_per_utt);
    const int r0 = (int)(tile % p.tiles_per_utt) * p.tile_rows;
    const int64_t off = p.utt_off[u];
    int64_t len = p.utt_off[u + 1] - off;
    if (p.lengths) len = min(len, (int64_t)max(p.lengths[u], 0));
    len = min(len, (int64_t)p.max_rows);
    if (r0 >= len) continue;
    const int nr = (int)min(len - r0, (int64_t)p.tile_rows);  // rows of this tile
    const T* base = X + (off + r0) * p.ld;
    int cnt = 0;
    double K = 0.0, s1 = 0.0, s2 = 0.0;
    for (int r = rs; r < nr; r += RS * ST_UNROLL) {
      T v[ST_UNROLL];
#pragma unroll
      for (int k = 0; k < ST_UNROLL; ++k) {
        const int rr = r + k * RS;
        v[k] = T(0);
        if (col_ok && rr < nr) v[k] = ld_stream(base + (int64_t)rr * p.ld);
      }
      if (cnt == 0) K = (double)v[0];  // the shift: first value of the tile (r < nr here)
#pragma unroll
      for (int k = 0; k < ST_UNROLL; ++k) {
        if (r + k * RS < nr) {
          const double d = (double)v[k] - K;
          s1 += d;
          s2 = fma(d, d, s2);
          mn = nan_min(mn, v[k]);
          mx = nan_max(mx, v[k]);
          ++cnt;
        }
      }
    }
    if (cnt) {
      const double tn = (double)cnt;
      const double q = s1 / tn;
      double tm2 = s2 - s1 * q;
      if (tm2 < 0.0) tm2 = 0.0;  // rounding of a (near) constant column; a NaN passes through
      chan_merge(n, mean, m2, tn, K + q, tm2);
    }
  }
  // row slices of the block, in order
  sh_n[threadIdx.x] = n; sh_mean[threadIdx.x] = mean; sh_m2[threadIdx.x] = m2;
  sh_mn[threadIdx.x] = (double)mn; sh_mx[threadIdx.x] = (double)mx;
  __syncthreads();
  if (rs == 0 && col_ok) {
    double bmn = (double)mn, bmx = (double)mx;
    for (int s = 1; s < RS; ++s) {
      const int t = s * p.CW + cl;
      chan_merge(n, mean, m2, sh_n[t], sh_mean[t], sh_m2[t]);
      bmn = nan_min(bmn, sh_mn[t]);
      bmx = nan_max(bmx, sh_mx[t]);
    }
    double* P = p.part + (size_t)blockIdx.x * 5 * D;
    P[c] = n; P[D + c] = mean; P[2 * D + c] = m2; P[3 * D + c] = bmn; P[4 * D + c] = bmx;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(p.ticket, 1u) == gridDim.x * gridDim.y - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  // the incoming state first, then the block partials in index order
  const double n_in = __ldcg(p.state);
  const int G = gridDim.x;
  double n_out = n_in;
  for (int cc = threadIdx.x; cc < D; cc += blockDim.x) {
    double fn = n_in, fm = __ldcg(p.state + 1 + cc), fq = __ldcg(p.state + 1 + D + cc);
    double fmn = __ldcg(p.state + 1 + 2 * D + cc), fmx = __ldcg(p.state + 1 + 3 * D + cc);
    for (int b0 = 0; b0 < G; b0 += ST_FOLD_UNROLL) {  // (n, mean, m2), then min / max: fewer live registers
      double pn[ST_FOLD_UNROLL], pm[ST_FOLD_UNROLL], pq[ST_FOLD_UNROLL];
#pragma unroll
      for (int k = 0; k < ST_FOLD_UNROLL; ++k) {
        pn[k] = pm[k] = pq[k] = 0.0;
        if (b0 + k < G) {
          const double* P = p.part + (size_t)(b0 + k) * 5 * D + cc;
          pn[k] = __ldcg(P); pm[k] = __ldcg(P + D); pq[k] = __ldcg(P + 2 * D);
        }
      }
#pragma unroll
      for (int k = 0; k < ST_FOLD_UNROLL; ++k) chan_merge(fn, fm, fq, pn[k], pm[k], pq[k]);
    }
    for (int b0 = 0; b0 < G; b0 += 2 * ST_FOLD_UNROLL) {
      double pa[2 * ST_FOLD_UNROLL], pb[2 * ST_FOLD_UNROLL];
#pragma unroll
      for (int k = 0; k < 2 * ST_FOLD_UNROLL; ++k) {
        pa[k] = INFINITY; pb[k] = -INFINITY;
        if (b0 + k < G) {
          const double* P = p.part + (size_t)(b0 + k) * 5 * D + cc;
          pa[k] = __ldcg(P + 3 * D); pb[k] = __ldcg(P + 4 * D);
        }
      }
#pragma unroll
      for (int k = 0; k < 2 * ST_FOLD_UNROLL; ++k) {
        fmn = nan_min(fmn, pa[k]);
        fmx = nan_max(fmx, pb[k]);
      }
    }
    p.state[1 + cc] = fm; p.state[1 + D + cc] = fq; p.state[1 + 2 * D + cc] = fmn; p.state[1 + 3 * D + cc] = fmx;
    n_out = fn;  // the same for every column
  }
  __syncthreads();  // every thread has read state[0]
  if (threadIdx.x == 0) {
    p.state[0] = n_out;
    *p.ticket = 0u;
  }
}

struct StatsShape {
  int CW, RS, nstrips, tile_rows, tiles_per_utt, grid;
  int64_t n_tiles;
};

static StatsShape stats_shape(int n_utt, int max_rows, int D) {
  StatsShape s{};
  s.nstrips = (D + ST_BLOCK - 1) / ST_BLOCK;
  if (s.nstrips < 1) s.nstrips = 1;
  const int w = (D + s.nstrips - 1) / s.nstrips;
  s.CW = (w + 31) / 32 * 32;
  if (s.CW < 32) s.CW = 32;
  s.RS = ST_BLOCK / s.CW;
  s.tile_rows = ST_ROWS_PER_THREAD * s.RS;
  s.tiles_per_utt = (max_rows + s.tile_rows - 1) / s.tile_rows;
  s.n_tiles = (int64_t)n_utt * s.tiles_per_utt;
  int bps = ST_THREADS_PER_SM / (s.CW * s.RS);
  if (bps > 8) bps = 8;
  int64_t g = (int64_t)kNumSMs * bps / s.nstrips;
  if (g > s.n_tiles) g = s.n_tiles;
  s.grid = (int)(g < 1 ? 1 : g);
  return s;
}

static int64_t stats_ws_bytes(const StatsShape& s, int D) { return 64 + (int64_t)s.grid * 5 * D * 8; }

// ---- per-column affine map ---------------------------------------------------------------------------
constexpr int AF_BLOCK = 256;
constexpr int AF_UNROLL = 4;

__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }

// Element e = row * D + col of a contiguous matrix; a thread walks e, e + AF_BLOCK, ... and advances its
// column incrementally, so no division per element and any D keeps every lane busy.
template <typename Tin, typename T, int FORM>
__global__ void __launch_bounds__(AF_BLOCK) column_affine_kernel(const Tin* __restrict__ x, const T* __restrict__ a,
                                                                 const T* __restrict__ b, T* __restrict__ out,
                                                                 int64_t n, int D) {
  const int64_t stride = (int64_t)gridDim.x * AF_BLOCK * AF_UNROLL;
  const int step_c = AF_BLOCK % D, stride_c = (int)(stride % D);
  int64_t e0 = (int64_t)blockIdx.x * AF_BLOCK * AF_UNROLL + threadIdx.x;
  int c = (int)(e0 % D);
  for (; e0 < n; e0 += stride) {
    Tin v[AF_UNROLL];
    int cc[AF_UNROLL];
    int cu = c;
#pragma unroll
    for (int k = 0; k < AF_UNROLL; ++k) {
      const int64_t e = e0 + (int64_t)k * AF_BLOCK;
      cc[k] = cu;
      v[k] = Tin(0);
      if (e < n) v[k] = ld_stream(x + e);
      cu += step_c;
      if (cu >= D) cu -= D;
    }
#pragma unroll
    for (int k = 0; k < AF_UNROLL; ++k) {
      const int64_t e = e0 + (int64_t)k * AF_BLOCK;
      if (e < n) {
        const T xv = (T)v[k];
        const T r = FORM == 0 ? div_rn(sub_rn(xv, __ldg(a + cc[k])), __ldg(b + cc[k]))
                              : add_rn(mul_rn(xv, __ldg(b + cc[k])), __ldg(a + cc[k]));
        st_stream(out + e, r);
      }
    }
    c += stride_c;
    if (c >= D) c -= D;
  }
}

template <typename Tin, typename T>
static void launch_affine(const void* x, const void* a, const void* b, void* out, int64_t n, int D, int form,
                          cudaStream_t st) {
  int64_t g = (n + AF_BLOCK * AF_UNROLL - 1) / (AF_BLOCK * AF_UNROLL);
  if (g > (int64_t)kNumSMs * 16) g = (int64_t)kNumSMs * 16;
  const Tin* xp = reinterpret_cast<const Tin*>(x);
  const T* ap = reinterpret_cast<const T*>(a);
  const T* bp = reinterpret_cast<const T*>(b);
  T* op = reinterpret_cast<T*>(out);
  if (form == 0) column_affine_kernel<Tin, T, 0><<<(unsigned)g, AF_BLOCK, 0, st>>>(xp, ap, bp, op, n, D);
  else column_affine_kernel<Tin, T, 1><<<(unsigned)g, AF_BLOCK, 0, st>>>(xp, ap, bp, op, n, D);
}

// segment_moments_kernel (nnk_segment_moments): per-segment column mean and population variance, two passes.
// Block = 32 columns x SM_RS row slices of one segment; slice k sums rows k, k + SM_RS, ... in order and the
// slices are folded in index order, so the result depends only on the segment's rows.
constexpr int SM_RS = 8;

template <typename Tin>
__global__ void __launch_bounds__(32 * SM_RS)
    segment_moments_kernel(const Tin* __restrict__ x, int D, int64_t ld, const int64_t* __restrict__ utt_off,
                           const int32_t* __restrict__ utt_len, int u0, double* __restrict__ mean,
                           double* __restrict__ var) {
  __shared__ double part[SM_RS][32];
  __shared__ double col_mean[32];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c = blockIdx.x * 32 + tx;
  const int u = u0 + blockIdx.y;
  const int64_t r0 = utt_off[u];
  const int64_t n = utt_len ? (int64_t)utt_len[u] : utt_off[u + 1] - r0;
  const bool on = c < D;
  const Tin* col = x + r0 * ld + (on ? c : 0);
  double s = 0.0;
  if (on)
    for (int64_t r = ty; r < n; r += SM_RS) s += (double)col[r * ld];
  part[ty][tx] = s;
  __syncthreads();
  if (ty == 0) {
    double t = 0.0;
#pragma unroll
    for (int k = 0; k < SM_RS; ++k) t += part[k][tx];
    col_mean[tx] = t / (double)n;
  }
  __syncthreads();
  const double m = col_mean[tx];
  double s2 = 0.0;
  if (on)
    for (int64_t r = ty; r < n; r += SM_RS) {
      const double d = (double)col[r * ld] - m;
      s2 = fma(d, d, s2);
    }
  __syncthreads();
  part[ty][tx] = s2;
  __syncthreads();
  if (ty == 0 && on) {
    double t = 0.0;
#pragma unroll
    for (int k = 0; k < SM_RS; ++k) t += part[k][tx];
    var[(int64_t)u * D + c] = t / (double)n;
    if (mean) mean[(int64_t)u * D + c] = m;
  }
}

}  // namespace nnk

using namespace nnk;

extern "C" int64_t nnk_frame_stats_workspace_bytes(int32_t n_utt, int32_t max_rows, int32_t D) {
  if (n_utt < 1) n_utt = 1;
  if (max_rows < 1) max_rows = 1;
  if (D < 1) D = 1;
  return stats_ws_bytes(stats_shape(n_utt, max_rows, D), D);
}

extern "C" int nnk_frame_stats(const void* X, int32_t dtype, int32_t D, int64_t ld, const int64_t* utt_off,
                               const int32_t* lengths, int32_t n_utt, int32_t max_rows, double* state,
                               void* workspace, int64_t workspace_bytes, void* stream) {
  NNK_REQUIRE(state, NNK_ERR_ARG, "NULL state");
  DeviceGuard guard(state);
  NNK_REQUIRE(dtype == NNK_F32 || dtype == NNK_F64, NNK_ERR_ARG, "bad dtype");
  NNK_REQUIRE(D >= 1 && n_utt >= 0 && max_rows >= 0 && ld >= D, NNK_ERR_ARG, "bad size");
  if (n_utt == 0 || max_rows == 0) return NNK_OK;  // no rows: the state is the result
  NNK_REQUIRE(X && utt_off, NNK_ERR_ARG, "NULL input");
  cudaStream_t st = (cudaStream_t)stream;
  const StatsShape s = stats_shape(n_utt, max_rows, D);
  NNK_REQUIRE(workspace && workspace_bytes >= stats_ws_bytes(s, D), NNK_ERR_WORKSPACE, "stats workspace too small");
  StatsParams p{};
  p.x = X; p.ld = ld; p.utt_off = utt_off; p.lengths = lengths;
  p.D = D; p.CW = s.CW; p.RS = s.RS; p.max_rows = max_rows; p.tile_rows = s.tile_rows;
  p.tiles_per_utt = s.tiles_per_utt; p.n_tiles = s.n_tiles;
  char* w = reinterpret_cast<char*>(workspace);
  p.ticket = reinterpret_cast<unsigned int*>(w);
  p.part = reinterpret_cast<double*>(w + 64);
  p.state = state;
  NNK_CUDA_CHECK(cudaMemsetAsync(p.ticket, 0, sizeof(unsigned int), st));
  const dim3 grid((unsigned)s.grid, (unsigned)s.nstrips);
  const unsigned threads = (unsigned)(s.CW * s.RS);
  if (dtype == NNK_F32) frame_stats_kernel<float><<<grid, threads, 0, st>>>(p);
  else frame_stats_kernel<double><<<grid, threads, 0, st>>>(p);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

extern "C" int nnk_column_affine(const void* x, int32_t x_dtype, int32_t dtype, int64_t n_rows, int32_t D,
                                 const void* a, const void* b, int32_t form, void* out, void* stream) {
  NNK_REQUIRE(out, NNK_ERR_ARG, "NULL output");
  DeviceGuard guard(out);
  NNK_REQUIRE((x_dtype == NNK_F32 || x_dtype == NNK_F64) && (dtype == NNK_F32 || dtype == NNK_F64) &&
                  !(x_dtype == NNK_F64 && dtype == NNK_F32),
              NNK_ERR_ARG, "bad dtype (x float32 / float64, computed in float32 only for float32 x)");
  NNK_REQUIRE(form == 0 || form == 1, NNK_ERR_ARG, "bad form");
  NNK_REQUIRE(n_rows >= 0 && D >= 1, NNK_ERR_ARG, "bad size");
  if (n_rows == 0) return NNK_OK;
  NNK_REQUIRE(x && a && b, NNK_ERR_ARG, "NULL input");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n = n_rows * D;
  if (dtype == NNK_F32) launch_affine<float, float>(x, a, b, out, n, D, form, st);
  else if (x_dtype == NNK_F32) launch_affine<float, double>(x, a, b, out, n, D, form, st);
  else launch_affine<double, double>(x, a, b, out, n, D, form, st);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

extern "C" int nnk_segment_moments(const void* X, int32_t dtype, int32_t D, int64_t ld, const int64_t* utt_off,
                                   const int32_t* utt_len, int32_t n_utt, double* mean, double* var, void* stream) {
  NNK_REQUIRE(dtype == NNK_F32 || dtype == NNK_F64, NNK_ERR_ARG, "dtype must be NNK_F32 or NNK_F64");
  NNK_REQUIRE(D >= 0 && n_utt >= 0 && ld >= D, NNK_ERR_ARG, "bad sizes");
  if (D == 0 || n_utt == 0) return NNK_OK;
  NNK_REQUIRE(X && utt_off && var, NNK_ERR_ARG, "NULL device pointer");
  DeviceGuard guard(var);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 block(32, SM_RS);
  for (int u0 = 0; u0 < n_utt; u0 += 65535) {
    const dim3 grid((D + 31) / 32, n_utt - u0 < 65535 ? n_utt - u0 : 65535);
    if (dtype == NNK_F32)
      segment_moments_kernel<float><<<grid, block, 0, st>>>((const float*)X, D, ld, utt_off, utt_len, u0, mean, var);
    else
      segment_moments_kernel<double><<<grid, block, 0, st>>>((const double*)X, D, ld, utt_off, utt_len, u0, mean, var);
    count_launch();
    NNK_CUDA_CHECK(cudaGetLastError());
  }
  return NNK_OK;
}
