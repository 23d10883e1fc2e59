// nnk_kmeans.cu -- k-means initialisation of baseline.gmm.GaussianMixture on sm_90a, float64 throughout.
//
// Device restatement of scikit-learn 1.9's KMeans(n_init=1) (Lloyd) and k-means++ seeding, step for step:
//   km_colsum_kernel / km_colfold_kernel : X_mean = X.mean(axis=0) and mean(var(X, axis=0)) (the tolerance),
//                          fixed-order column sums; every later kernel reads widen(x) - X_mean, nothing is copied.
//   k-means++ (one step per centre, no host synchronisation; the host pre-draws the uniforms):
//     km_pp_search_kernel : per trial, r = u * current_pot and the first row whose inclusive prefix sum of
//                           closest_dist_sq reaches r (searchsorted side="left", clipped to N - 1);
//     km_pp_dist_kernel   : per row, max(-2 x.c + |c|^2 + |x|^2, 0) for every candidate (sklearn's
//                           _euclidean_distances order), min with closest_dist_sq, per-chunk potentials;
//     km_pp_pick_kernel   : fold the potentials, first argmin, record the centre.
//   Lloyd (one iteration per nnk_kmeans_lloyd):
//     km_centers_kernel   : centres transposed and their squared norms;
//     km_assign_kernel    : label = first argmin_j |c_j|^2 - 2 x.c_j, changed-label count and per-chunk cluster
//                           sums / counts in one pass over a frame tile in shared memory;
//     km_fold_kernel      : cluster sums and weights, chunk partials summed in chunk order;
//     km_update_kernel    : _average_centers (multiply by 1 / weight) and _center_shift, unless a cluster is
//                           empty: then the host relocates first (see nnk_kmeans_relocate_dist).
//   km_reloc_dist_kernel  : ((x - c_old[label])^2).sum() per row, for _relocate_empty_clusters_dense.
//   km_inertia_kernel / km_inertia_fold_kernel : _inertia_dense and the number of distinct labels.
// Every reduction has a fixed shape that depends only on (N, D, K), so runs are bit-identical.
#include <float.h>
#include <math.h>
#include <math_constants.h>

#include "nnk_common.cuh"

namespace nnk {

constexpr int KM_MAX_D = 128;
constexpr int KM_MAX_K = 128;
constexpr int KM_MAX_TRIALS = 8;         // 2 + int(log(K)) <= 6 for K <= 128
constexpr int KM_KP = 128;               // padded cluster stride of the transposed centres
constexpr int KM_THREADS = 256;
constexpr int KM_COL_CHUNK = 1024;       // column sums: rows per block
constexpr int PP_CHUNK = 1024;           // k-means++: contiguous rows per block (the prefix-sum search order)
constexpr int PP_WARPS = KM_THREADS / 32;
constexpr int LL_FPW = 8;                // Lloyd assignment: frames per warp
constexpr int LL_WARPS = 8;
constexpr int LL_FT = LL_FPW * LL_WARPS; // frames per tile
constexpr int LL_TARGET_BLOCKS = 2 * kNumSMs;

// int64 slots at the start of the workspace
constexpr int IW_CAND = 0;               // [KM_MAX_TRIALS] candidate rows of the current step
constexpr int IW_BEST = KM_MAX_TRIALS;   // best trial of the last step
constexpr int IW_SLOTS = 16;

struct KmLayout {
  int64_t n_col, n_pp, ll_chunk, n_ll, n_in;
  int trials;
  size_t col, pot, ppart, dtrial, ct, cn, lpart, ipart, seen, total;  // offsets in 8-byte words
};

static inline size_t round4(size_t v) { return (v + 3) & ~(size_t)3; }

static int km_trials(int K) { return 2 + (int)floor(log((double)K)); }  // sklearn: 2 + int(np.log(n_clusters))

static KmLayout km_layout(int64_t N, int D, int K) {
  KmLayout L{};
  L.trials = km_trials(K);
  L.n_col = (N + KM_COL_CHUNK - 1) / KM_COL_CHUNK;
  L.n_pp = (N + PP_CHUNK - 1) / PP_CHUNK;
  const int64_t per = (N + LL_TARGET_BLOCKS - 1) / LL_TARGET_BLOCKS;
  L.ll_chunk = (per + LL_FT - 1) / LL_FT * LL_FT;
  L.n_ll = (N + L.ll_chunk - 1) / L.ll_chunk;
  L.n_in = (N + KM_THREADS - 1) / KM_THREADS;
  size_t o = IW_SLOTS;
  L.col = o;    o += round4((size_t)L.n_col * D);
  L.pot = o;    o += 4;
  L.ppart = o;  o += round4((size_t)L.trials * L.n_pp);
  L.dtrial = o; o += round4((size_t)L.trials * N);
  L.ct = o;     o += (size_t)D * KM_KP;
  L.cn = o;     o += KM_KP;
  L.lpart = o;  o += round4((size_t)L.n_ll * ((size_t)K * (D + 1) + 1));
  L.ipart = o;  o += round4((size_t)L.n_in);
  L.seen = o;   o += round4((size_t)K);
  L.total = o;
  return L;
}

struct KmParams {
  const void* X;
  int64_t N, x_ld;
  int D, K;
  int step, n_tr;       // k-means++: centre index and trials of this launch
  int64_t first;
  const double* rand;
  double* centers;
  double* sums;
  double* weights;
  int32_t* labels;
  int64_t* indices;
  double* mean;
  double* dist;
  double* out_centers;
  double* status;
  double* ws;
  int64_t* iw;
  KmLayout L;
};

template <typename T> __device__ __forceinline__ double ldx(const T* p) { return (double)__ldg(p); }
template <typename T> __device__ __forceinline__ double xc(const KmParams& p, int64_t i, int d) {
  return ldx(static_cast<const T*>(p.X) + i * p.x_ld + d) - p.mean[d];
}

// sklearn's _euclidean_dense_dense (squared): four products summed left to right per step, then the tail;
// explicit roundings so that nothing is contracted into an FMA
__device__ __forceinline__ double sq4(double a0, double a1, double a2, double a3) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(a0, a0), __dmul_rn(a1, a1)), __dmul_rn(a2, a2)), __dmul_rn(a3, a3));
}

// numpy's pairwise_sum for n <= 128 (one block: eight accumulators, then ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)))
template <typename F>
__device__ double np_pairwise_sum(F v, int n) {
  if (n < 8) {
    double s = 0.0;
    for (int i = 0; i < n; ++i) s = __dadd_rn(s, v(i));
    return s;
  }
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = v(j);
  int i = 8;
  for (; i < n - (n % 8); i += 8)
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], v(i + j));
  double s = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                       __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; ++i) s = __dadd_rn(s, v(i));
  return s;
}

// fixed-shape block reduction: thread t sums entries t, t + 256, ... in order, then a fixed tree
__device__ double km_block_fold(const double* v, int64_t n) {
  __shared__ double red[KM_THREADS];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += KM_THREADS) s += v[i];
  __syncthreads();
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = KM_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

__device__ __forceinline__ double warp_sum(double s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

// ---- column means and the tolerance ----------------------------------------------------------------------
// SQ = false: partial column sums of x; SQ = true: of (x - mean)^2.  Thread d owns column d.
template <typename T, bool SQ>
__global__ void __launch_bounds__(KM_MAX_D) km_colsum_kernel(const __grid_constant__ KmParams p) {
  const int d = threadIdx.x;
  if (d >= p.D) return;
  const T* X = static_cast<const T*>(p.X);
  const int64_t n0 = (int64_t)blockIdx.x * KM_COL_CHUNK, n1 = min(p.N, n0 + KM_COL_CHUNK);
  const double m = SQ ? p.mean[d] : 0.0;
  double s = 0.0;
  for (int64_t i = n0; i < n1; ++i) {
    const double v = ldx(X + i * p.x_ld + d);
    if (SQ) {
      const double c = v - m;
      s = fma(c, c, s);
    } else {
      s += v;
    }
  }
  p.ws[p.L.col + (size_t)blockIdx.x * p.D + d] = s;
}

template <bool SQ>
__global__ void __launch_bounds__(KM_MAX_D) km_colfold_kernel(const __grid_constant__ KmParams p) {
  __shared__ double var[KM_MAX_D];
  const int d = threadIdx.x;
  if (d < p.D) {
    double s = 0.0;
    for (int64_t c = 0; c < p.L.n_col; ++c) s += p.ws[p.L.col + (size_t)c * p.D + d];
    if (SQ) var[d] = s / (double)p.N;
    else p.mean[d] = s / (double)p.N;
  }
  if (!SQ) return;
  __syncthreads();
  if (d == 0) {
    double s = 0.0;
    for (int e = 0; e < p.D; ++e) s += var[e];
    p.status[NNK_KM_VAR_MEAN] = s / (double)p.D;
  }
}

__global__ void km_zero_mean_kernel(const __grid_constant__ KmParams p) {
  if ((int)threadIdx.x < p.D) p.mean[threadIdx.x] = 0.0;
}

// ---- k-means++ -------------------------------------------------------------------------------------------
// First index i < n with base + v[0] + ... + v[i] >= r (n if none), over a block of KM_THREADS threads:
// thread t owns a contiguous run of entries; the runs' sums are scanned in a fixed tree, then each thread walks
// its run in order.  *before = the running sum before entry i.
__device__ int64_t block_first_geq(const double* v, int64_t n, double base, double r, double* before) {
  __shared__ double scan[KM_THREADS];
  __shared__ unsigned long long hit;
  __shared__ double hit_before;
  const int t = threadIdx.x;
  const int64_t per = (n + KM_THREADS - 1) / KM_THREADS;
  const int64_t lo = min(n, (int64_t)t * per), hi = min(n, lo + per);
  double g = 0.0;
  for (int64_t j = lo; j < hi; ++j) g += v[j];
  __syncthreads();
  scan[t] = g;
  if (t == 0) hit = (unsigned long long)n;
  __syncthreads();
  for (int off = 1; off < KM_THREADS; off <<= 1) {
    const double add = (t >= off) ? scan[t - off] : 0.0;
    __syncthreads();
    scan[t] += add;
    __syncthreads();
  }
  double run = base + ((t > 0) ? scan[t - 1] : 0.0);
  int64_t mine = n;
  double mine_before = 0.0;
  for (int64_t j = lo; j < hi; ++j) {
    const double prev = run;
    run += v[j];
    if (run >= r) {
      mine = j;
      mine_before = prev;
      atomicMin(&hit, (unsigned long long)j);
      break;
    }
  }
  __syncthreads();
  if (mine < n && (unsigned long long)mine == hit) hit_before = mine_before;
  __syncthreads();
  const int64_t res = (int64_t)hit;
  if (before && res < n) *before = hit_before;
  __syncthreads();
  return res;
}

// one block per trial of step p.step >= 1
__global__ void __launch_bounds__(KM_THREADS) km_pp_search_kernel(const __grid_constant__ KmParams p) {
  const int t = blockIdx.x;
  const int64_t best = p.iw[IW_BEST];
  const double r = p.rand[(size_t)(p.step - 1) * p.L.trials + t] * p.ws[p.L.pot];
  double base = 0.0;
  const int64_t b = block_first_geq(p.ws + p.L.ppart + (size_t)best * p.L.n_pp, p.L.n_pp, 0.0, r, &base);
  int64_t cand = p.N - 1;
  if (b < p.L.n_pp) {
    const int64_t row0 = b * PP_CHUNK, nrows = min((int64_t)PP_CHUNK, p.N - row0);
    int64_t i = block_first_geq(p.ws + p.L.dtrial + (size_t)best * p.N + row0, nrows, base, r, nullptr);
    if (i >= nrows) i = nrows - 1;  // rounding between the chunk-level and the row-level sums
    cand = min(row0 + i, p.N - 1);
  }
  if (threadIdx.x == 0) p.iw[IW_CAND + t] = cand;
}

// warp per row, lanes along the features (d = lane + 32 e)
template <int EPL, typename T>
__global__ void __launch_bounds__(KM_THREADS) km_pp_dist_kernel(const __grid_constant__ KmParams p) {
  __shared__ double wpot[PP_WARPS][KM_MAX_TRIALS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n_tr = p.n_tr;
  double cv[KM_MAX_TRIALS][EPL], cn[KM_MAX_TRIALS], pot[KM_MAX_TRIALS];
#pragma unroll
  for (int t = 0; t < KM_MAX_TRIALS; ++t) {
    pot[t] = 0.0;
    cn[t] = 0.0;
    if (t < n_tr) {
      const int64_t c = (p.step == 0) ? p.first : p.iw[IW_CAND + t];
      double s = 0.0;
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int d = lane + 32 * e;
        cv[t][e] = (d < p.D) ? xc<T>(p, c, d) : 0.0;
        s = fma(cv[t][e], cv[t][e], s);
      }
      cn[t] = warp_sum(s);
    } else {
#pragma unroll
      for (int e = 0; e < EPL; ++e) cv[t][e] = 0.0;
    }
  }
  const double* closest = p.ws + p.L.dtrial + (size_t)p.iw[IW_BEST] * p.N;
  double* dtr = p.ws + p.L.dtrial;
  const int64_t r0 = (int64_t)blockIdx.x * PP_CHUNK, r1 = min(p.N, r0 + PP_CHUNK);
  for (int64_t i = r0 + warp; i < r1; i += PP_WARPS) {
    double xv[EPL], s = 0.0;
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      const int d = lane + 32 * e;
      xv[e] = (d < p.D) ? xc<T>(p, i, d) : 0.0;
      s = fma(xv[e], xv[e], s);
    }
    const double xn = warp_sum(s);
    const double cl = (p.step == 0) ? CUDART_INF : closest[i];
    double dv[KM_MAX_TRIALS];
#pragma unroll
    for (int t = 0; t < KM_MAX_TRIALS; ++t) {
      if (t < n_tr) {
        double q = 0.0;
#pragma unroll
        for (int e = 0; e < EPL; ++e) q = fma(xv[e], cv[t][e], q);
        const double dot = warp_sum(q);
        const double dist = fmax(__dadd_rn(__dadd_rn(-2.0 * dot, cn[t]), xn), 0.0);
        dv[t] = fmin(cl, dist);
        pot[t] += dv[t];
      }
    }
    __syncwarp();  // every lane has read closest[i] before it is overwritten (trial `best` may alias it)
    if (lane == 0) {
#pragma unroll
      for (int t = 0; t < KM_MAX_TRIALS; ++t)
        if (t < n_tr) dtr[(size_t)t * p.N + i] = dv[t];
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int t = 0; t < KM_MAX_TRIALS; ++t) wpot[warp][t] = pot[t];
  }
  __syncthreads();
  if (threadIdx.x < n_tr) {
    double s = 0.0;
    for (int w = 0; w < PP_WARPS; ++w) s += wpot[w][threadIdx.x];
    p.ws[p.L.ppart + (size_t)threadIdx.x * p.L.n_pp + blockIdx.x] = s;
  }
}

template <typename T>
__global__ void __launch_bounds__(KM_THREADS) km_pp_pick_kernel(const __grid_constant__ KmParams p) {
  __shared__ double pots[KM_MAX_TRIALS];
  __shared__ int64_t cand;
  for (int t = 0; t < p.n_tr; ++t) {
    const double s = km_block_fold(p.ws + p.L.ppart + (size_t)t * p.L.n_pp, p.L.n_pp);
    if (threadIdx.x == 0) pots[t] = s;
  }
  if (threadIdx.x == 0) {
    int best = 0;
    for (int t = 1; t < p.n_tr; ++t)
      if (pots[t] < pots[best]) best = t;
    p.ws[p.L.pot] = pots[best];
    p.iw[IW_BEST] = best;
    cand = (p.step == 0) ? p.first : p.iw[IW_CAND + best];
    p.indices[p.step] = cand;
  }
  __syncthreads();
  for (int d = threadIdx.x; d < p.D; d += blockDim.x) p.centers[(size_t)p.step * p.D + d] = xc<T>(p, cand, d);
}

// ---- Lloyd -----------------------------------------------------------------------------------------------
// centres transposed (D x KM_KP) and sklearn's centers_squared_norms
__global__ void __launch_bounds__(KM_THREADS) km_centers_kernel(const __grid_constant__ KmParams p) {
  const int D = p.D, K = p.K;
  double* ct = p.ws + p.L.ct;
  for (int e = threadIdx.x; e < D * K; e += blockDim.x) {
    const int k = e / D, d = e - k * D;
    ct[(size_t)d * KM_KP + k] = p.centers[e];
  }
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    double s = 0.0;
    for (int d = 0; d < D; ++d) s = fma(p.centers[(size_t)k * D + d], p.centers[(size_t)k * D + d], s);
    p.ws[p.L.cn + k] = s;
  }
}

// One block per chunk of L.ll_chunk frames, in tiles of LL_FT frames (centred, in shared memory).  Warp w labels
// frames w * LL_FPW ..; lanes run along the clusters (j = lane + 32 e, e < EPL), the transposed centres come
// through L1.  UPDATE: thread d <= D then adds the tile's frames into the chunk's cluster sums in frame order.
template <int EPL, typename T, bool UPDATE>
__global__ void __launch_bounds__(KM_THREADS) km_assign_kernel(const __grid_constant__ KmParams p) {
  extern __shared__ __align__(16) double sm[];
  const int D = p.D, K = p.K, W = D + 1;
  double* mean = sm;                            // [D]
  double* xs = mean + D;                        // [LL_FT][D]
  double* acc = xs + (size_t)LL_FT * D;         // [K][D + 1] (UPDATE)
  int* lab = reinterpret_cast<int*>(acc + (UPDATE ? (size_t)K * W : 0));  // [LL_FT]
  __shared__ int changed_w[LL_WARPS];
  const T* X = static_cast<const T*>(p.X);
  const double* ct = p.ws + p.L.ct;
  const double* cn = p.ws + p.L.cn;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int d = threadIdx.x; d < D; d += blockDim.x) mean[d] = p.mean[d];
  if (UPDATE)
    for (int o = threadIdx.x; o < K * W; o += blockDim.x) acc[o] = 0.0;
  double cnl[EPL];
#pragma unroll
  for (int e = 0; e < EPL; ++e) {
    const int j = lane + 32 * e;
    cnl[e] = (j < K) ? cn[j] : 0.0;
  }
  int changed = 0;
  const int64_t n0 = (int64_t)blockIdx.x * p.L.ll_chunk, n1 = min(p.N, n0 + p.L.ll_chunk);
  for (int64_t t0 = n0; t0 < n1; t0 += LL_FT) {
    const int nf = (int)min((int64_t)LL_FT, n1 - t0);
    __syncthreads();
    for (int e = threadIdx.x; e < nf * D; e += blockDim.x) {
      const int f = e / D, d = e - f * D;
      xs[e] = ldx(X + (t0 + f) * p.x_ld + d) - mean[d];
    }
    __syncthreads();
    const double* xw = xs + (size_t)warp * LL_FPW * D;
    double a[LL_FPW][EPL];
#pragma unroll
    for (int f = 0; f < LL_FPW; ++f)
#pragma unroll
      for (int e = 0; e < EPL; ++e) a[f][e] = 0.0;
    const int nfw = min(LL_FPW, nf - warp * LL_FPW);
    if (nfw > 0) {
      for (int d = 0; d < D; ++d) {
        double c[EPL];
#pragma unroll
        for (int e = 0; e < EPL; ++e) c[e] = __ldg(ct + (size_t)d * KM_KP + lane + 32 * e);
#pragma unroll
        for (int f = 0; f < LL_FPW; ++f) {
          const double v = (f < nfw) ? xw[(size_t)f * D + d] : 0.0;
#pragma unroll
          for (int e = 0; e < EPL; ++e) a[f][e] = fma(v, c[e], a[f][e]);
        }
      }
    }
#pragma unroll
    for (int f = 0; f < LL_FPW; ++f) {
      if (f >= nfw) break;
      double bv = CUDART_INF;
      int bj = K;
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int j = lane + 32 * e;
        const double dist = cnl[e] + (-2.0 * a[f][e]);  // BLAS: -2 X.C^T + 1.0 * |c|^2
        if (j < K && dist < bv) { bv = dist; bj = j; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {  // first minimum: the smaller index wins a tie
        const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
        if (ov < bv || (ov == bv && oj < bj)) { bv = ov; bj = oj; }
      }
      if (lane == 0) {
        const int fr = warp * LL_FPW + f;
        const int64_t i = t0 + fr;
        if (p.labels[i] != bj) ++changed;
        p.labels[i] = bj;
        if (UPDATE) lab[fr] = bj;
      }
    }
    if (UPDATE) {
      __syncthreads();
      const int d = threadIdx.x;
      if (d <= D)
        for (int f = 0; f < nf; ++f) acc[(size_t)lab[f] * W + d] += (d < D) ? xs[(size_t)f * D + d] : 1.0;
    }
  }
  if (!UPDATE) {
    if (lane == 0) changed_w[warp] = changed;
    __syncthreads();
    return;
  }
  if (lane == 0) changed_w[warp] = changed;
  __syncthreads();
  const size_t stride = (size_t)K * W + 1;
  double* out = p.ws + p.L.lpart + (size_t)blockIdx.x * stride;
  for (int o = threadIdx.x; o < K * W; o += blockDim.x) out[o] = acc[o];
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < LL_WARPS; ++w) s += changed_w[w];
    out[K * W] = (double)s;
  }
}

// one thread per (k, d <= D) and one for the changed count: chunk partials in chunk order
__global__ void __launch_bounds__(KM_THREADS) km_fold_kernel(const __grid_constant__ KmParams p) {
  const int D = p.D, K = p.K, W = D + 1;
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o > K * W) return;
  const size_t stride = (size_t)K * W + 1;
  double s = 0.0;
  for (int64_t c = 0; c < p.L.n_ll; ++c) s += p.ws[p.L.lpart + (size_t)c * stride + o];
  if (o == K * W) {
    p.status[NNK_KM_CHANGED] = s;
    return;
  }
  const int k = o / W, d = o - k * W;
  if (d < D) p.sums[(size_t)k * D + d] = s;
  else p.weights[k] = s;
}

// _average_centers + _center_shift, thread k owns centre k.  force == 0 and an empty cluster: only count them
// (the host relocates, then calls nnk_kmeans_average, which runs this with force == 1).
__global__ void __launch_bounds__(KM_MAX_K) km_update_kernel(const __grid_constant__ KmParams p, int force) {
  __shared__ double shift2[KM_MAX_K];
  __shared__ int n_empty, amax;
  const int D = p.D, K = p.K, k = threadIdx.x;
  if (k == 0) {
    int ne = 0, am = 0;
    for (int j = 0; j < K; ++j) {
      if (p.weights[j] == 0.0) ++ne;
      if (p.weights[j] > p.weights[am]) am = j;  // np.argmax: the first maximum
    }
    n_empty = ne;
    amax = am;
    p.status[NNK_KM_EMPTY] = (double)ne;
  }
  __syncthreads();
  if (n_empty > 0 && !force) return;
  if (k < K) {
    // sklearn averages rows in order and copies the heaviest row into an empty one: a row before it is still
    // a sum, a row after it already the average
    const double wk = p.weights[k];
    const int src = (wk > 0.0) ? k : amax;
    const bool avg = (wk > 0.0) || (amax < k);
    const double alpha = avg ? __ddiv_rn(1.0, p.weights[src]) : 1.0;
    const double* s = p.sums + (size_t)src * D;
    double* c = p.centers + (size_t)k * D;
    double res = 0.0;
    int d = 0;
    for (; d + 4 <= D; d += 4) {
      double nv[4], df[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        nv[q] = avg ? __dmul_rn(s[d + q], alpha) : s[d + q];
        df[q] = __dsub_rn(nv[q], c[d + q]);
      }
      res = __dadd_rn(res, sq4(df[0], df[1], df[2], df[3]));
#pragma unroll
      for (int q = 0; q < 4; ++q) c[d + q] = nv[q];
    }
    for (; d < D; ++d) {
      const double nv = avg ? __dmul_rn(s[d], alpha) : s[d];
      const double df = __dsub_rn(nv, c[d]);
      res = __dadd_rn(res, __dmul_rn(df, df));
      c[d] = nv;
    }
    const double sh = sqrt(res);
    shift2[k] = __dmul_rn(sh, sh);
  }
  __syncthreads();
  if (k == 0) p.status[NNK_KM_SHIFT] = np_pairwise_sum([&](int j) { return shift2[j]; }, K);
}

// ((X - centers_old[labels]) ** 2).sum(axis=1), numpy's pairwise order along the row
template <typename T>
__global__ void __launch_bounds__(KM_THREADS) km_reloc_dist_kernel(const __grid_constant__ KmParams p) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.N) return;
  const double* c = p.centers + (size_t)p.labels[i] * p.D;
  p.dist[i] = np_pairwise_sum([&](int d) {
    const double df = __dsub_rn(xc<T>(p, i, d), c[d]);
    return __dmul_rn(df, df);
  }, p.D);
}

// _inertia_dense: per row _euclidean_dense_dense(x, c[label]), block partials in a fixed tree
template <typename T>
__global__ void __launch_bounds__(KM_THREADS) km_inertia_kernel(const __grid_constant__ KmParams p) {
  __shared__ double red[KM_THREADS];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double res = 0.0;
  if (i < p.N) {
    const int lb = p.labels[i];
    const double* c = p.centers + (size_t)lb * p.D;
    int d = 0;
    for (; d + 4 <= p.D; d += 4)
      res = __dadd_rn(res, sq4(__dsub_rn(xc<T>(p, i, d), c[d]), __dsub_rn(xc<T>(p, i, d + 1), c[d + 1]),
                               __dsub_rn(xc<T>(p, i, d + 2), c[d + 2]), __dsub_rn(xc<T>(p, i, d + 3), c[d + 3])));
    for (; d < p.D; ++d) {
      const double df = __dsub_rn(xc<T>(p, i, d), c[d]);
      res = __dadd_rn(res, __dmul_rn(df, df));
    }
    p.ws[p.L.seen + lb] = 1.0;
  }
  red[threadIdx.x] = res;
  __syncthreads();
  for (int w = KM_THREADS / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) p.ws[p.L.ipart + blockIdx.x] = red[0];
}

__global__ void __launch_bounds__(KM_THREADS) km_inertia_fold_kernel(const __grid_constant__ KmParams p) {
  const double s = km_block_fold(p.ws + p.L.ipart, p.L.n_in);
  if (threadIdx.x == 0) {
    p.status[NNK_KM_INERTIA] = s;
    int n = 0;
    for (int k = 0; k < p.K; ++k) n += (p.ws[p.L.seen + k] != 0.0);
    p.status[NNK_KM_DISTINCT] = (double)n;
  }
  for (int e = threadIdx.x; e < p.K * p.D; e += blockDim.x) p.out_centers[e] = p.centers[e] + p.mean[e % p.D];
}

}  // namespace nnk

using namespace nnk;

static int km_check(const nnk_kmeans_args_t* a, KmParams& p) {
  NNK_REQUIRE(a != nullptr, NNK_ERR_ARG, "NULL args");
  NNK_REQUIRE(a->D >= 1 && a->D <= KM_MAX_D, NNK_ERR_UNSUPPORTED, "k-means supports 1 <= n_features <= 128");
  NNK_REQUIRE(a->K >= 1 && a->K <= KM_MAX_K, NNK_ERR_UNSUPPORTED, "k-means supports 1 <= n_clusters <= 128");
  NNK_REQUIRE(a->N >= a->K && a->N <= INT32_MAX, NNK_ERR_ARG, "k-means needs n_clusters <= n_samples < 2^31");
  NNK_REQUIRE(a->dtype == NNK_F32 || a->dtype == NNK_F64, NNK_ERR_ARG, "dtype must be NNK_F32 or NNK_F64");
  NNK_REQUIRE(a->x_ld >= a->D, NNK_ERR_ARG, "x_ld < D");
  NNK_REQUIRE(a->X && a->centers && a->sums && a->weights && a->labels && a->mean && a->status, NNK_ERR_ARG,
              "NULL pointer");
  p = KmParams{};
  p.L = km_layout(a->N, a->D, a->K);
  NNK_REQUIRE(a->workspace != nullptr && a->workspace_bytes >= p.L.total * sizeof(double), NNK_ERR_WORKSPACE,
              "workspace smaller than nnk_kmeans_workspace_bytes()");
  p.X = a->X; p.N = a->N; p.x_ld = a->x_ld; p.D = a->D; p.K = a->K; p.first = a->first; p.rand = a->rand;
  p.centers = a->centers; p.sums = a->sums; p.weights = a->weights; p.labels = a->labels; p.indices = a->indices;
  p.mean = a->mean; p.dist = a->dist; p.out_centers = a->out_centers; p.status = a->status;
  p.ws = (double*)a->workspace;
  p.iw = (int64_t*)a->workspace;
  return NNK_OK;
}

template <typename Kernel, typename... Extra>
static int km_launch(Kernel kernel, dim3 grid, int threads, size_t smem, cudaStream_t st, const KmParams& p,
                     Extra... extra) {
  if (smem > 48 * 1024) NNK_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<grid, threads, smem, st>>>(p, extra...);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

#define KM_TRY(expr)          \
  do {                        \
    const int _rc = (expr);   \
    if (_rc) return _rc;      \
  } while (0)

template <typename T>
static int prepare_t(const nnk_kmeans_args_t* a, const KmParams& p, cudaStream_t st) {
  if (!a->centre) return km_launch(km_zero_mean_kernel, dim3(1), KM_MAX_D, 0, st, p);
  KM_TRY(km_launch(km_colsum_kernel<T, false>, dim3((unsigned)p.L.n_col), KM_MAX_D, 0, st, p));
  KM_TRY(km_launch(km_colfold_kernel<false>, dim3(1), KM_MAX_D, 0, st, p));
  KM_TRY(km_launch(km_colsum_kernel<T, true>, dim3((unsigned)p.L.n_col), KM_MAX_D, 0, st, p));
  return km_launch(km_colfold_kernel<true>, dim3(1), KM_MAX_D, 0, st, p);
}

template <int EPL, typename T>
static int seed_t(KmParams p, cudaStream_t st) {
  for (int c = 0; c < p.K; ++c) {
    p.step = c;
    p.n_tr = (c == 0) ? 1 : p.L.trials;
    if (c > 0) KM_TRY(km_launch(km_pp_search_kernel, dim3((unsigned)p.n_tr), KM_THREADS, 0, st, p));
    KM_TRY(km_launch(km_pp_dist_kernel<EPL, T>, dim3((unsigned)p.L.n_pp), KM_THREADS, 0, st, p));
    KM_TRY(km_launch(km_pp_pick_kernel<T>, dim3(1), KM_THREADS, 0, st, p));
  }
  return NNK_OK;
}

template <typename T>
static int seed_d(const KmParams& p, cudaStream_t st) {
  switch ((p.D + 31) / 32) {
    case 1: return seed_t<1, T>(p, st);
    case 2: return seed_t<2, T>(p, st);
    case 3: return seed_t<3, T>(p, st);
    default: return seed_t<4, T>(p, st);
  }
}

static size_t assign_smem(const KmParams& p, bool update) {
  return sizeof(double) * ((size_t)p.D + (size_t)LL_FT * p.D + (update ? (size_t)p.K * (p.D + 1) : 0)) +
         sizeof(int) * LL_FT;
}

template <int EPL, typename T>
static int assign_t(const KmParams& p, bool update, cudaStream_t st) {
  const dim3 grid((unsigned)p.L.n_ll);
  if (update) return km_launch(km_assign_kernel<EPL, T, true>, grid, KM_THREADS, assign_smem(p, true), st, p);
  return km_launch(km_assign_kernel<EPL, T, false>, grid, KM_THREADS, assign_smem(p, false), st, p);
}

template <typename T>
static int assign_d(const KmParams& p, bool update, cudaStream_t st) {
  switch ((p.K + 31) / 32) {
    case 1: return assign_t<1, T>(p, update, st);
    case 2: return assign_t<2, T>(p, update, st);
    case 3: return assign_t<3, T>(p, update, st);
    default: return assign_t<4, T>(p, update, st);
  }
}

extern "C" size_t nnk_kmeans_workspace_bytes(int64_t N, int32_t D, int32_t K) {
  if (D < 1 || D > KM_MAX_D || K < 1 || K > KM_MAX_K || N < K || N > INT32_MAX) return 0;
  return km_layout(N, D, K).total * sizeof(double);
}

extern "C" int nnk_kmeans_prepare(const nnk_kmeans_args_t* a, void* stream) {
  KmParams p;
  KM_TRY(km_check(a, p));
  DeviceGuard guard(a->X);
  cudaStream_t st = (cudaStream_t)stream;
  return (a->dtype == NNK_F32) ? prepare_t<float>(a, p, st) : prepare_t<double>(a, p, st);
}

extern "C" int nnk_kmeans_seed(const nnk_kmeans_args_t* a, void* stream) {
  KmParams p;
  KM_TRY(km_check(a, p));
  NNK_REQUIRE(a->indices != nullptr && (a->K == 1 || a->rand != nullptr), NNK_ERR_ARG, "NULL indices / rand");
  NNK_REQUIRE(a->first >= 0 && a->first < a->N, NNK_ERR_ARG, "first centre out of range");
  DeviceGuard guard(a->X);
  cudaStream_t st = (cudaStream_t)stream;
  NNK_CUDA_CHECK(cudaMemsetAsync(p.iw, 0, IW_SLOTS * sizeof(int64_t), st));
  return (a->dtype == NNK_F32) ? seed_d<float>(p, st) : seed_d<double>(p, st);
}

extern "C" int nnk_kmeans_lloyd(const nnk_kmeans_args_t* a, void* stream) {
  KmParams p;
  KM_TRY(km_check(a, p));
  DeviceGuard guard(a->X);
  cudaStream_t st = (cudaStream_t)stream;
  const bool update = a->update != 0;
  KM_TRY(km_launch(km_centers_kernel, dim3(1), KM_THREADS, 0, st, p));
  KM_TRY((a->dtype == NNK_F32) ? assign_d<float>(p, update, st) : assign_d<double>(p, update, st));
  if (!update) return NNK_OK;
  const int n = p.K * (p.D + 1) + 1;
  KM_TRY(km_launch(km_fold_kernel, dim3((unsigned)((n + KM_THREADS - 1) / KM_THREADS)), KM_THREADS, 0, st, p));
  return km_launch(km_update_kernel, dim3(1), KM_MAX_K, 0, st, p, 0);
}

extern "C" int nnk_kmeans_average(const nnk_kmeans_args_t* a, void* stream) {
  KmParams p;
  KM_TRY(km_check(a, p));
  DeviceGuard guard(a->X);
  return km_launch(km_update_kernel, dim3(1), KM_MAX_K, 0, (cudaStream_t)stream, p, 1);
}

extern "C" int nnk_kmeans_relocate_dist(const nnk_kmeans_args_t* a, void* stream) {
  KmParams p;
  KM_TRY(km_check(a, p));
  NNK_REQUIRE(a->dist != nullptr, NNK_ERR_ARG, "NULL dist");
  DeviceGuard guard(a->X);
  const dim3 grid((unsigned)((p.N + KM_THREADS - 1) / KM_THREADS));
  cudaStream_t st = (cudaStream_t)stream;
  if (a->dtype == NNK_F32) return km_launch(km_reloc_dist_kernel<float>, grid, KM_THREADS, 0, st, p);
  return km_launch(km_reloc_dist_kernel<double>, grid, KM_THREADS, 0, st, p);
}

extern "C" int nnk_kmeans_inertia(const nnk_kmeans_args_t* a, void* stream) {
  KmParams p;
  KM_TRY(km_check(a, p));
  NNK_REQUIRE(a->out_centers != nullptr, NNK_ERR_ARG, "NULL out_centers");
  DeviceGuard guard(a->X);
  cudaStream_t st = (cudaStream_t)stream;
  NNK_CUDA_CHECK(cudaMemsetAsync(p.ws + p.L.seen, 0, (size_t)p.K * sizeof(double), st));
  const dim3 grid((unsigned)p.L.n_in);
  if (a->dtype == NNK_F32) KM_TRY(km_launch(km_inertia_kernel<float>, grid, KM_THREADS, 0, st, p));
  else KM_TRY(km_launch(km_inertia_kernel<double>, grid, KM_THREADS, 0, st, p));
  return km_launch(km_inertia_fold_kernel, dim3(1), KM_THREADS, 0, st, p);
}
