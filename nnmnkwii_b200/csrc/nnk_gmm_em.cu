// nnk_gmm_em.cu -- EM fit of a full-covariance Gaussian mixture on sm_90a, float64 throughout.
//
// The device side of baseline.gmm.GaussianMixture (a drop-in for sklearn.mixture.GaussianMixture with
// covariance_type="full"), following scikit-learn 1.9's operation order where it matters for parity:
//   em_estep_kernel    : per tile of frames and every component k, y = X U_k - (mu_k U_k) (the product first,
//                        then the precomputed row), log_prob = -1/2 (D log 2pi + sum y^2) + log_det_k + log w_k;
//                        per frame sklearn's _logsumexp (maxima excluded, log1p(s / m) + log(m) + max);
//                        resp = exp(log_prob - lse); one partial of sum lse per tile.
//   em_lse_fold_kernel : lower bound = (fixed-order sum of the tile partials) / N.
//   em_stats_kernel    : per chunk of frames, partials of nk = sum r and sum r x for every component.
//   em_stats_fold      : nk = sum r + 10 eps, means = sum r x / nk, fixed order over the chunks.
//   em_cov_kernel      : per (chunk, component), the centred sum (r (x - mu))^T (x - mu) (sklearn's two-pass
//                        form; sum r x x^T - nk mu mu^T cancels badly when |mu| >> sigma).
//   em_cov_fold_kernel : covariances = (fixed-order sum of the chunk partials) / nk + reg_covar I, and the
//                        weights nk / N (sklearn's _initialize) or nk / sum nk (its _m_step).
//   em_factor_kernel   : one CTA per component: Cholesky C = L L^T (a non-positive pivot sets the status
//                        word and the CTA leaves), precisions_cholesky = L^-T, then log_det = sum log diag U,
//                        log w and mu U for the next E-step.
// Every reduction has a fixed shape that depends only on (N, D, K), so runs are bit-identical.  X may be
// float32 (widened on load) or float64.  Plain FP64 CUDA-core arithmetic, register-blocked; no tensor cores.
#include <float.h>
#include <math.h>
#include <math_constants.h>

#include "nnk_common.cuh"

namespace nnk {

constexpr int EM_MAX_D = 128;
constexpr int EM_MAX_K = 128;
constexpr int ES_FPW = 8;                  // E-step: frames per warp
constexpr int ES_WARPS = 4;
constexpr int ES_FT = ES_FPW * ES_WARPS;   // E-step: frames per block
constexpr int ST_CHUNK = 1024;             // statistics: frames per block
constexpr int ST_SUB = 32;                 // statistics: frames staged at a time
constexpr int CV_SUB = 32;                 // covariance: frames staged at a time
constexpr int CV_TARGET_BLOCKS = 4 * kNumSMs;
constexpr int FOLD_THREADS = 256;

struct EmLayout {
  int64_t n_tiles, n_stat, n_cov, cov_chunk;
  size_t lse, stat, nk, cov, logw, logdet, muu, total;  // offsets in doubles
};

static inline size_t round4(size_t v) { return (v + 3) & ~(size_t)3; }

static EmLayout em_layout(int64_t N, int D, int K) {
  EmLayout L{};
  L.n_tiles = (N + ES_FT - 1) / ES_FT;
  L.n_stat = (N + ST_CHUNK - 1) / ST_CHUNK;
  int64_t n_cov = (CV_TARGET_BLOCKS + K - 1) / K;
  const int64_t by_len = (N + 255) / 256;  // at least 256 frames per chunk
  if (n_cov > by_len) n_cov = by_len;
  if (n_cov < 1) n_cov = 1;
  L.cov_chunk = ((N + n_cov - 1) / n_cov + CV_SUB - 1) / CV_SUB * CV_SUB;
  L.n_cov = (N + L.cov_chunk - 1) / L.cov_chunk;
  size_t o = 0;
  L.lse = o;    o += round4((size_t)L.n_tiles);
  L.stat = o;   o += round4((size_t)L.n_stat * K * (D + 1));
  L.nk = o;     o += round4((size_t)K);
  L.cov = o;    o += round4((size_t)L.n_cov * K * D * D);
  L.logw = o;   o += round4((size_t)K);
  L.logdet = o; o += round4((size_t)K);
  L.muu = o;    o += round4((size_t)K * D);
  L.total = o;
  return L;
}

struct EmParams {
  const void* X;
  int64_t N, x_ld;
  int D, K;
  double* resp;
  double* weights;
  double* means;
  double* cov;
  double* prec_chol;
  double* lower_bound;
  double reg_covar;
  double c0;  // D log(2 pi), evaluated on the host like sklearn's n_features * math.log(2 * math.pi)
  int weight_norm;
  int factor;
  int32_t* status;
  double* ws;
  EmLayout L;
};

template <typename T> __device__ __forceinline__ double ldx(const T* p) { return (double)__ldg(p); }

// ---- E-step ------------------------------------------------------------------------------------------------
// Lanes run along the output dimension j (EPL outputs per lane, D <= 32 EPL), each warp keeps ES_FPW frames x EPL
// outputs in registers; the tile's frames sit in shared memory (broadcast reads), U_k rows come through L1.
template <int EPL, typename T>
__global__ void __launch_bounds__(ES_WARPS * 32) em_estep_kernel(const __grid_constant__ EmParams p) {
  extern __shared__ __align__(16) double sm[];
  const int D = p.D, K = p.K;
  double* xs = sm;                            // [ES_FT][D]
  double* lps = xs + (size_t)ES_FT * D;       // [ES_FT][K]
  double* lsef = lps + (size_t)ES_FT * K;     // [ES_FT]
  const int64_t t0 = (int64_t)blockIdx.x * ES_FT;
  const int nf = (int)min((int64_t)ES_FT, p.N - t0);
  const T* X = static_cast<const T*>(p.X);
  for (int e = threadIdx.x; e < ES_FT * D; e += blockDim.x) {
    const int f = e / D, d = e - f * D;
    xs[e] = (f < nf) ? ldx(X + (t0 + f) * p.x_ld + d) : 0.0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double* xw = xs + (size_t)warp * ES_FPW * D;
  const double* logw = p.ws + p.L.logw;
  const double* logdet = p.ws + p.L.logdet;
  const double* muu = p.ws + p.L.muu;
  for (int k = 0; k < K; ++k) {
    const double* U = p.prec_chol + (size_t)k * D * D;
    double acc[ES_FPW][EPL];
#pragma unroll
    for (int f = 0; f < ES_FPW; ++f)
#pragma unroll
      for (int e = 0; e < EPL; ++e) acc[f][e] = 0.0;
    for (int i = 0; i < D; ++i) {
      double u[EPL];
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int j = lane + 32 * e;
        u[e] = (j < D) ? __ldg(U + (size_t)i * D + j) : 0.0;
      }
#pragma unroll
      for (int f = 0; f < ES_FPW; ++f) {
        const double v = xw[(size_t)f * D + i];
#pragma unroll
        for (int e = 0; e < EPL; ++e) acc[f][e] = fma(v, u[e], acc[f][e]);
      }
    }
    double mu[EPL];
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      const int j = lane + 32 * e;
      mu[e] = (j < D) ? muu[(size_t)k * D + j] : 0.0;
    }
    const double ld = logdet[k], lw = logw[k];
#pragma unroll
    for (int f = 0; f < ES_FPW; ++f) {
      double s = 0.0;
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const double y = acc[f][e] - mu[e];
        s = fma(y, y, s);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) lps[(size_t)(warp * ES_FPW + f) * K + k] = (-0.5 * (p.c0 + s) + ld) + lw;
    }
  }
  __syncwarp();
  // per-frame logsumexp (sklearn.utils._array_api._logsumexp) and the responsibilities
  for (int q = 0; q < ES_FPW; ++q) {
    const int f = warp * ES_FPW + q;
    if (f >= nf) break;
    const double* row = lps + (size_t)f * K;
    double mx = -CUDART_INF;
    for (int k = lane; k < K; k += 32) mx = fmax(mx, row[k]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const double shift = isfinite(mx) ? mx : 0.0;
    double cnt = 0.0, s = 0.0;
    for (int k = lane; k < K; k += 32) {
      const double v = row[k];
      if (v == mx) cnt += 1.0;
      else s += exp(v - shift);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      s += __shfl_xor_sync(0xffffffffu, s, o);
    }
    if (s != 0.0) s = s / cnt;
    const double lse = log1p(s) + log(cnt) + mx;
    double* r = p.resp + (t0 + f) * K;
    for (int k = lane; k < K; k += 32) r[k] = exp(row[k] - lse);
    if (lane == 0) lsef[f] = lse;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int f = 0; f < nf; ++f) s += lsef[f];
    p.ws[p.L.lse + blockIdx.x] = s;
  }
}

// fixed-shape block reduction: thread t sums entries t, t + 256, ... in order, then a fixed tree
__device__ double block_fold(const double* v, int64_t n) {
  __shared__ double red[FOLD_THREADS];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += FOLD_THREADS) s += v[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = FOLD_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  return red[0];
}

__global__ void __launch_bounds__(FOLD_THREADS) em_lse_fold_kernel(const __grid_constant__ EmParams p) {
  const double s = block_fold(p.ws + p.L.lse, p.L.n_tiles);
  if (threadIdx.x == 0) *p.lower_bound = s / (double)p.N;
}

// ---- M-step: sufficient statistics -----------------------------------------------------------------------
// partial[c][k][d] = sum over the chunk of r[n][k] x[n][d] (d < D) and sum r[n][k] (d == D)
template <typename T>
__global__ void __launch_bounds__(256) em_stats_kernel(const __grid_constant__ EmParams p) {
  extern __shared__ __align__(16) double sm[];
  const int D = p.D, K = p.K, W = D + 1, KW = K * (D + 1);
  double* acc = sm;                       // [K][D + 1]
  double* rs = acc + KW;                  // [ST_SUB][K]
  double* xs = rs + (size_t)ST_SUB * K;   // [ST_SUB][D]
  const T* X = static_cast<const T*>(p.X);
  for (int o = threadIdx.x; o < KW; o += blockDim.x) acc[o] = 0.0;
  const int64_t n0 = (int64_t)blockIdx.x * ST_CHUNK, n1 = min(p.N, n0 + ST_CHUNK);
  for (int64_t s0 = n0; s0 < n1; s0 += ST_SUB) {
    const int ns = (int)min((int64_t)ST_SUB, n1 - s0);
    __syncthreads();
    for (int e = threadIdx.x; e < ns * K; e += blockDim.x) rs[e] = p.resp[s0 * K + e];
    for (int e = threadIdx.x; e < ns * D; e += blockDim.x) {
      const int f = e / D, d = e - f * D;
      xs[e] = ldx(X + (s0 + f) * p.x_ld + d);
    }
    __syncthreads();
    for (int o = threadIdx.x; o < KW; o += blockDim.x) {
      const int k = o / W, d = o - k * W;
      double a = 0.0;
      if (d < D) {
        for (int f = 0; f < ns; ++f) a = fma(rs[f * K + k], xs[f * D + d], a);
      } else {
        for (int f = 0; f < ns; ++f) a += rs[f * K + k];
      }
      acc[o] += a;
    }
  }
  __syncthreads();
  double* out = p.ws + p.L.stat + (size_t)blockIdx.x * KW;
  for (int o = threadIdx.x; o < KW; o += blockDim.x) out[o] = acc[o];
}

// one thread per (k, d): nk and means, summing the chunk partials in chunk order
__global__ void __launch_bounds__(256) em_stats_fold_kernel(const __grid_constant__ EmParams p) {
  const int D = p.D, W = D + 1, KW = p.K * W;
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= KW) return;
  const int k = o / W, d = o - k * W;
  const double* part = p.ws + p.L.stat;
  double nk = 0.0, sx = 0.0;
  for (int64_t c = 0; c < p.L.n_stat; ++c) {
    nk += part[c * KW + (size_t)k * W + D];
    if (d < D) sx += part[c * KW + o];
  }
  nk += 10.0 * DBL_EPSILON;
  if (d < D) p.means[(size_t)k * D + d] = sx / nk;
  else p.ws[p.L.nk + k] = nk;
}

// ---- M-step: covariances -----------------------------------------------------------------------------------
// One block per (chunk, component): 16 x 16 threads, thread (ty, tx) owns rows ty + 16 a and columns tx + 16 b,
// a, b < TI (D <= 16 TI).  (r (x - mu))_i and (x - mu)_j are staged per sub-tile of frames, rows padded to 16 TI.
template <int TI, typename T>
__global__ void __launch_bounds__(256) em_cov_kernel(const __grid_constant__ EmParams p) {
  extern __shared__ __align__(16) double sm[];
  constexpr int DS = 16 * TI;
  const int D = p.D, K = p.K, k = blockIdx.y;
  double* rd = sm;                        // [CV_SUB][DS]  r (x - mu)
  double* dd = rd + CV_SUB * DS;          // [CV_SUB][DS]  x - mu
  double* mus = dd + CV_SUB * DS;         // [D]
  const T* X = static_cast<const T*>(p.X);
  for (int d = threadIdx.x; d < D; d += blockDim.x) mus[d] = p.means[(size_t)k * D + d];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double acc[TI][TI];
#pragma unroll
  for (int a = 0; a < TI; ++a)
#pragma unroll
    for (int b = 0; b < TI; ++b) acc[a][b] = 0.0;
  const int64_t n0 = (int64_t)blockIdx.x * p.L.cov_chunk, n1 = min(p.N, n0 + p.L.cov_chunk);
  for (int64_t s0 = n0; s0 < n1; s0 += CV_SUB) {
    const int ns = (int)min((int64_t)CV_SUB, n1 - s0);
    __syncthreads();
    for (int e = threadIdx.x; e < CV_SUB * DS; e += blockDim.x) {
      const int f = e / DS, d = e - f * DS;
      double df = 0.0, r = 0.0;
      if (f < ns && d < D) {
        df = ldx(X + (s0 + f) * p.x_ld + d) - mus[d];
        r = p.resp[(s0 + f) * K + k];
      }
      dd[e] = df;
      rd[e] = r * df;
    }
    __syncthreads();
    for (int f = 0; f < ns; ++f) {
      double av[TI], bv[TI];
#pragma unroll
      for (int a = 0; a < TI; ++a) av[a] = rd[f * DS + ty + 16 * a];
#pragma unroll
      for (int b = 0; b < TI; ++b) bv[b] = dd[f * DS + tx + 16 * b];
#pragma unroll
      for (int a = 0; a < TI; ++a)
#pragma unroll
        for (int b = 0; b < TI; ++b) acc[a][b] = fma(av[a], bv[b], acc[a][b]);
    }
  }
  double* out = p.ws + p.L.cov + ((size_t)blockIdx.x * K + k) * D * D;
#pragma unroll
  for (int a = 0; a < TI; ++a)
#pragma unroll
    for (int b = 0; b < TI; ++b) {
      const int i = ty + 16 * a, j = tx + 16 * b;
      if (i < D && j < D) out[(size_t)i * D + j] = acc[a][b];
    }
}

__global__ void __launch_bounds__(256) em_cov_fold_kernel(const __grid_constant__ EmParams p) {
  const int D = p.D, K = p.K, k = blockIdx.x;
  const double nk = p.ws[p.L.nk + k];
  const size_t DD = (size_t)D * D, stride = (size_t)K * DD;
  const double* part = p.ws + p.L.cov + (size_t)k * DD;
  for (int e = threadIdx.x; e < (int)DD; e += blockDim.x) {
    double s = 0.0;
    for (int64_t c = 0; c < p.L.n_cov; ++c) s += part[c * stride + e];
    double v = s / nk;
    if (e / D == e % D) v += p.reg_covar;
    p.cov[(size_t)k * DD + e] = v;
  }
  if (threadIdx.x == 0 && p.weight_norm != 2) {
    double den = (double)p.N;
    if (p.weight_norm == 1) {
      den = 0.0;
      for (int c = 0; c < K; ++c) den += p.ws[p.L.nk + c];
    }
    p.weights[k] = nk / den;
  }
}

// ---- factorisation: one CTA per component, thread i owns row i (D <= 128 threads) -------------------------------
__global__ void __launch_bounds__(EM_MAX_D) em_factor_kernel(const __grid_constant__ EmParams p) {
  extern __shared__ __align__(16) double sm[];
  const int D = p.D, k = blockIdx.x, i = threadIdx.x;
  const int S = D + 1;  // odd-ish row stride: thread-per-row accesses spread over the banks
  double* A = sm;       // [D][D + 1]
  double* Ld = A + (size_t)D * S;
  double* U = p.prec_chol + (size_t)k * D * D;
  if (p.factor) {
    const double* C = p.cov + (size_t)k * D * D;
    for (int e = threadIdx.x; e < D * D; e += blockDim.x) {
      const int r = e / D, c = e - r * D;
      if (c <= r) A[r * S + c] = C[e];  // the lower triangle, as LAPACK's potrf('L') reads it
    }
    __syncthreads();
    // right-looking Cholesky, column j at a time
    for (int j = 0; j < D; ++j) {
      const double piv = A[j * S + j];
      if (!(piv > 0.0)) {  // non-positive or NaN pivot: uniform exit, the host raises
        if (i == 0) atomicExch(p.status, 1);
        return;
      }
      const double ljj = sqrt(piv);
      if (i == j) Ld[j] = ljj;
      if (i > j && i < D) A[i * S + j] = A[i * S + j] / ljj;
      __syncthreads();
      if (i > j && i < D) {
        const double lij = A[i * S + j];
        for (int c = j + 1; c <= i; ++c) A[i * S + c] -= lij * A[c * S + j];
      }
      __syncthreads();
    }
    // Z = L^-1 column c by thread c (forward substitution against e_c), kept in the upper triangle of row c:
    // A[c][r] = Z[r][c] = U[c][r] for r >= c
    if (i < D) {
      A[i * S + i] = 1.0 / Ld[i];
      for (int r = i + 1; r < D; ++r) {
        double s = 0.0;
        for (int j = i; j < r; ++j) s = fma(A[r * S + j], A[i * S + j], s);
        A[i * S + r] = -s / Ld[r];
      }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < D * D; e += blockDim.x) {
      const int r = e / D, c = e - r * D;
      U[e] = (c >= r) ? A[r * S + c] : 0.0;
    }
    __syncthreads();
  }
  // derived per-component constants of the E-step
  if (i < D) {
    const double* mu = p.means + (size_t)k * D;
    double s = 0.0;
    for (int r = 0; r < D; ++r) s = fma(mu[r], U[(size_t)r * D + i], s);
    p.ws[p.L.muu + (size_t)k * D + i] = s;
  }
  if (i == 0) {
    double ld = 0.0;
    for (int r = 0; r < D; ++r) ld += log(U[(size_t)r * D + r]);
    p.ws[p.L.logdet + k] = ld;
    p.ws[p.L.logw + k] = log(p.weights[k]);
  }
}

}  // namespace nnk

using namespace nnk;

static int em_check(const nnk_gmm_em_args_t* a, EmParams& p) {
  NNK_REQUIRE(a != nullptr, NNK_ERR_ARG, "NULL args");
  NNK_REQUIRE(a->D >= 1 && a->D <= EM_MAX_D, NNK_ERR_ARG, "GMM EM supports 1 <= n_features <= 128");
  NNK_REQUIRE(a->K >= 1 && a->K <= EM_MAX_K, NNK_ERR_ARG, "GMM EM supports 1 <= n_components <= 128");
  NNK_REQUIRE(a->N >= 1 && a->N <= ((int64_t)1 << 40), NNK_ERR_ARG, "bad number of samples");
  NNK_REQUIRE(a->dtype == NNK_F32 || a->dtype == NNK_F64, NNK_ERR_ARG, "dtype must be NNK_F32 or NNK_F64");
  NNK_REQUIRE(a->x_ld >= a->D, NNK_ERR_ARG, "x_ld < D");
  NNK_REQUIRE(a->X && a->resp && a->weights && a->means && a->covariances && a->prec_chol && a->lower_bound && a->status,
              NNK_ERR_ARG, "NULL pointer");
  p = EmParams{};
  p.L = em_layout(a->N, a->D, a->K);
  NNK_REQUIRE(a->workspace != nullptr && a->workspace_bytes >= p.L.total * sizeof(double), NNK_ERR_WORKSPACE,
              "workspace smaller than nnk_gmm_em_workspace_bytes()");
  p.X = a->X; p.N = a->N; p.x_ld = a->x_ld; p.D = a->D; p.K = a->K;
  p.resp = a->resp; p.weights = a->weights; p.means = a->means; p.cov = a->covariances; p.prec_chol = a->prec_chol;
  p.lower_bound = a->lower_bound; p.reg_covar = a->reg_covar; p.c0 = (double)a->D * log(2.0 * M_PI);
  p.weight_norm = a->weight_norm; p.factor = a->factor; p.status = a->status; p.ws = (double*)a->workspace;
  return NNK_OK;
}

template <typename Kernel>
static int em_launch(Kernel kernel, dim3 grid, int threads, size_t smem, cudaStream_t st, const EmParams& p) {
  if (smem > 48 * 1024) NNK_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<grid, threads, smem, st>>>(p);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

template <int EPL, typename T>
static int estep_t(const EmParams& p, cudaStream_t st) {
  const size_t smem = sizeof(double) * ((size_t)ES_FT * p.D + (size_t)ES_FT * p.K + ES_FT);
  return em_launch(em_estep_kernel<EPL, T>, dim3((unsigned)p.L.n_tiles), ES_WARPS * 32, smem, st, p);
}

template <typename T>
static int estep_d(const EmParams& p, cudaStream_t st) {
  switch ((p.D + 31) / 32) {
    case 1: return estep_t<1, T>(p, st);
    case 2: return estep_t<2, T>(p, st);
    case 3: return estep_t<3, T>(p, st);
    default: return estep_t<4, T>(p, st);
  }
}

template <int TI, typename T>
static int cov_t(const EmParams& p, cudaStream_t st) {
  const size_t smem = sizeof(double) * (2 * (size_t)CV_SUB * 16 * TI + p.D);
  return em_launch(em_cov_kernel<TI, T>, dim3((unsigned)p.L.n_cov, (unsigned)p.K), 256, smem, st, p);
}

template <typename T>
static int mstep_d(const EmParams& p, cudaStream_t st) {
  const size_t ssm = sizeof(double) * ((size_t)p.K * (p.D + 1) + (size_t)ST_SUB * p.K + (size_t)ST_SUB * p.D);
  int rc = em_launch(em_stats_kernel<T>, dim3((unsigned)p.L.n_stat), 256, ssm, st, p);
  if (rc) return rc;
  const int kw = p.K * (p.D + 1);
  rc = em_launch(em_stats_fold_kernel, dim3((unsigned)((kw + 255) / 256)), 256, 0, st, p);
  if (rc) return rc;
  switch ((p.D + 15) / 16) {
    case 1: rc = cov_t<1, T>(p, st); break;
    case 2: rc = cov_t<2, T>(p, st); break;
    case 3: rc = cov_t<3, T>(p, st); break;
    case 4: rc = cov_t<4, T>(p, st); break;
    case 5: rc = cov_t<5, T>(p, st); break;
    case 6: rc = cov_t<6, T>(p, st); break;
    case 7: rc = cov_t<7, T>(p, st); break;
    default: rc = cov_t<8, T>(p, st); break;
  }
  if (rc) return rc;
  return em_launch(em_cov_fold_kernel, dim3((unsigned)p.K), 256, 0, st, p);
}

extern "C" size_t nnk_gmm_em_workspace_bytes(int64_t N, int32_t D, int32_t K) {
  if (N < 1 || D < 1 || D > EM_MAX_D || K < 1 || K > EM_MAX_K) return 0;
  return em_layout(N, D, K).total * sizeof(double);
}

extern "C" int nnk_gmm_em_estep(const nnk_gmm_em_args_t* a, void* stream) {
  EmParams p;
  int rc = em_check(a, p);
  if (rc) return rc;
  DeviceGuard guard(a->X);
  cudaStream_t st = (cudaStream_t)stream;
  rc = (a->dtype == NNK_F32) ? estep_d<float>(p, st) : estep_d<double>(p, st);
  if (rc) return rc;
  return em_launch(em_lse_fold_kernel, dim3(1), FOLD_THREADS, 0, st, p);
}

extern "C" int nnk_gmm_em_mstep(const nnk_gmm_em_args_t* a, void* stream) {
  EmParams p;
  int rc = em_check(a, p);
  if (rc) return rc;
  NNK_REQUIRE(a->weight_norm >= 0 && a->weight_norm <= 2, NNK_ERR_ARG, "weight_norm must be 0, 1 or 2");
  DeviceGuard guard(a->X);
  cudaStream_t st = (cudaStream_t)stream;
  return (a->dtype == NNK_F32) ? mstep_d<float>(p, st) : mstep_d<double>(p, st);
}

extern "C" int nnk_gmm_em_factor(const nnk_gmm_em_args_t* a, void* stream) {
  EmParams p;
  int rc = em_check(a, p);
  if (rc) return rc;
  DeviceGuard guard(a->X);
  const size_t smem = sizeof(double) * ((size_t)p.D * (p.D + 1) + p.D);
  return em_launch(em_factor_kernel, dim3((unsigned)p.K), EM_MAX_D, smem, (cudaStream_t)stream, p);
}
