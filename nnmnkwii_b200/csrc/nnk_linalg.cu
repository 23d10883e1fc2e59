// nnk_linalg.cu -- inverse of a symmetric positive definite matrix from its Cholesky factor
// (nnmnkwii.util.linalg, util/linalg.py:7-36 and util/_linalg.pyx:45-71), float64, batched.
//
// Both kernels run one thread per column of the result: column c of (F F^T)^-1 is a forward
// substitution F y = e_c followed by a backward substitution F^T x = y, and depends on no other
// column.  The output buffer doubles as the per-column scratch for y, so no workspace is needed.
#include <math.h>

#include "nnk_common.cuh"

namespace nnk {
namespace {

constexpr int kBandBlock = 128;  // threads (columns) per CTA of the banded kernel
constexpr int kMaxBand = 9;      // widest band with a template instance (l + u + 1 of every MLPG window set)
constexpr int kDenseBlock = 64;  // threads (columns) per CTA of the dense kernel
constexpr int kDenseRows = 8;    // rows of one register tile of the dense substitutions
constexpr int kDenseK = 64;      // factor columns (forward) / rows (backward) staged per shared-memory chunk
constexpr int kMaxGridY = 65535;

__device__ __forceinline__ bool bad_pivot(double d) { return !(d != 0.0) || !isfinite(d); }

// cholesky_inv_banded: P = (R R^T)^-1 from the band R[t, t-j], 0 <= j < W, of a lower factor.
// The reference's row recurrences (util/_linalg.pyx:45-71), restated for one column c:
//   forward   g[t] = -(sum_{j=1..W-1, R[t,t-j] != 0} R[t,t-j] g[t-j]  - [t == c]) / R[t,t]   (t >= c; g = 0 above)
//   backward  P[t] = (g[t] - sum_{j=1..W-1, R[t+j,t] != 0} R[t+j,t] P[t+j]) / R[t,t]        (t = T-1 .. 0)
// The sums run in the reference's j order, products and sums rounded separately (NumPy multiplies the
// row by R and then adds), so each element is the reference's value bit for bit.  The last W-1 values
// of g (forward) and P (backward) stay in registers; g goes to P's rows t >= c and is read back once.
template <int W>
__global__ void __launch_bounds__(kBandBlock) cholinv_banded_kernel(const double* __restrict__ R, double* P, int T,
                                                                    int item0, unsigned long long* status) {
  const int b = blockIdx.y;
  const int c0 = blockIdx.x * kBandBlock;
  const int c = c0 + threadIdx.x;
  const bool active = c < T;
  R += (size_t)b * T * T;
  P += (size_t)b * T * T;
  if (active && bad_pivot(R[(size_t)c * T + c])) report_not_pd(status, item0 + b, 0, c + 1);

  double h[W > 1 ? W : 2];  // h[j] = g[t - j] (forward) or P[t + j] (backward) of this column
#pragma unroll
  for (int j = 0; j < W; ++j) h[j] = 0.0;
  for (int t = c0; t < T; ++t) {  // rows above c0 are zero in every column of this CTA
    double s = 0.0;
#pragma unroll
    for (int j = 1; j < W; ++j) {
      if (t - j >= 0) {
        const double r = R[(size_t)t * T + (t - j)];
        if (r != 0.0) s = __dadd_rn(s, __dmul_rn(r, h[j]));
      }
    }
    if (t == c) s = __dsub_rn(s, 1.0);
    double g = __ddiv_rn(-s, R[(size_t)t * T + t]);
    g = t >= c ? g : 0.0;
    if (active && t >= c) P[(size_t)t * T + c] = g;
#pragma unroll
    for (int j = W - 1; j > 1; --j) h[j] = h[j - 1];
    if (W > 1) h[1] = g;
  }
#pragma unroll
  for (int j = 0; j < W; ++j) h[j] = 0.0;
  for (int t = T - 1; t >= 0; --t) {
    double s = 0.0;
#pragma unroll
    for (int j = 1; j < W; ++j) {
      if (t + j < T) {
        const double r = R[(size_t)(t + j) * T + t];
        if (r != 0.0) s = __dadd_rn(s, __dmul_rn(r, h[j]));
      }
    }
    const double g = (active && t >= c) ? P[(size_t)t * T + c] : 0.0;
    const double p = __ddiv_rn(__dsub_rn(g, s), R[(size_t)t * T + t]);
    if (active) P[(size_t)t * T + c] = p;
#pragma unroll
    for (int j = W - 1; j > 1; --j) h[j] = h[j - 1];
    if (W > 1) h[1] = p;
  }
}

// cholesky_inv: P = (F F^T)^-1 with F = L (lower) or U^T (upper); only that triangle of the input is read.
// Column c solves F y = e_c for rows t >= c, then F^T x = y for rows t = N-1 .. c, so only the lower
// triangle of P is computed; each x[t] is also written to P[c, t], which makes P exactly symmetric
// (dpotri computes one triangle and the reference mirrors it, util/_linalg.pyx:12-22).
// Rows go in register tiles of kDenseRows: the contribution of every row outside the tile is summed
// from a shared-memory chunk of F (read by all threads of the CTA: a broadcast) against the column's own
// earlier results in P (one coalesced row of the CTA's columns per k); then the tile's triangle is solved.
template <bool LOWER>
__global__ void __launch_bounds__(kDenseBlock) cholinv_dense_kernel(const double* __restrict__ A, double* P, int N,
                                                                    int item0, unsigned long long* status) {
  constexpr int RB = kDenseRows, KC = kDenseK;
  __shared__ double Fs[RB][KC];  // chunk of F: Fs[r][k] = F[t0 + r, k0 + k] (forward), F[k0 + k, t0 + r] (backward)
  __shared__ double Fd[RB][RB];  // diagonal block: Fd[r][q] = F[t0 + r, t0 + q], q <= r
  const int b = blockIdx.y;
  const int c0 = blockIdx.x * kDenseBlock;
  const int c = c0 + threadIdx.x;
  const bool active = c < N;
  A += (size_t)b * N * N;
  P += (size_t)b * N * N;
  // F[i, k] with i >= k: lower reads L[i, k], upper reads U[k, i]
  auto F = [&](int i, int k) { return LOWER ? A[(size_t)i * N + k] : A[(size_t)k * N + i]; };
  if (active && bad_pivot(A[(size_t)c * N + c])) report_not_pd(status, item0 + b, 0, c + 1);

  auto stage_diag = [&](int t0) {
    for (int i = threadIdx.x; i < RB * RB; i += kDenseBlock) {
      const int r = i / RB, q = i % RB;
      Fd[r][q] = (q <= r && t0 + r < N) ? F(t0 + r, t0 + q) : 0.0;
    }
  };
  const int n_tiles = (N - c0 + RB - 1) / RB;

  // forward: y = F^-1 e_c into P[t, c], t >= c
  for (int m = 0; m < n_tiles; ++m) {
    const int t0 = c0 + m * RB;
    double acc[RB], yb[RB];
#pragma unroll
    for (int r = 0; r < RB; ++r) acc[r] = 0.0;
    for (int k0 = c0; k0 < t0; k0 += KC) {
      const int kn = min(KC, t0 - k0);
      __syncthreads();
      for (int i = threadIdx.x; i < RB * KC; i += kDenseBlock) {
        const int r = LOWER ? i / KC : i % RB, k = LOWER ? i % KC : i / RB;  // contiguous global reads
        Fs[r][k] = (k < kn && t0 + r < N) ? F(t0 + r, k0 + k) : 0.0;
      }
      __syncthreads();
#pragma unroll 4
      for (int k = 0; k < kn; ++k) {
        const double y = (active && k0 + k >= c) ? P[(size_t)(k0 + k) * N + c] : 0.0;
#pragma unroll
        for (int r = 0; r < RB; ++r) acc[r] = fma(Fs[r][k], y, acc[r]);
      }
    }
    __syncthreads();
    stage_diag(t0);
    __syncthreads();
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      const int t = t0 + r;
      double s = acc[r];
#pragma unroll
      for (int q = 0; q < r; ++q) s = fma(Fd[r][q], yb[q], s);
      double y = t < N ? ((t == c ? 1.0 : 0.0) - s) / Fd[r][r] : 0.0;
      y = t >= c ? y : 0.0;
      yb[r] = y;
      if (active && t >= c && t < N) P[(size_t)t * N + c] = y;
    }
  }

  // backward: x = F^-T y for t = N-1 .. c; x[t] replaces y[t] in P[t, c] and is mirrored to P[c, t]
  for (int m = n_tiles - 1; m >= 0; --m) {
    const int t0 = c0 + m * RB;
    double acc[RB], xb[RB];
#pragma unroll
    for (int r = 0; r < RB; ++r) acc[r] = 0.0;
    for (int k0 = t0 + RB; k0 < N; k0 += KC) {
      const int kn = min(KC, N - k0);
      __syncthreads();
      for (int i = threadIdx.x; i < RB * KC; i += kDenseBlock) {
        const int r = LOWER ? i % RB : i / KC, k = LOWER ? i / RB : i % KC;
        Fs[r][k] = k < kn ? F(k0 + k, t0 + r) : 0.0;
      }
      __syncthreads();
#pragma unroll 4
      for (int k = 0; k < kn; ++k) {
        const double x = (active && k0 + k >= c) ? P[(size_t)(k0 + k) * N + c] : 0.0;
#pragma unroll
        for (int r = 0; r < RB; ++r) acc[r] = fma(Fs[r][k], x, acc[r]);
      }
    }
    __syncthreads();
    stage_diag(t0);
    __syncthreads();
#pragma unroll
    for (int r = RB - 1; r >= 0; --r) {
      const int t = t0 + r;
      double s = acc[r];
#pragma unroll
      for (int q = r + 1; q < RB; ++q) s = fma(Fd[q][r], xb[q], s);
      const bool mine = active && t >= c && t < N;
      const double y = mine ? P[(size_t)t * N + c] : 0.0;
      const double x = mine ? (y - s) / Fd[r][r] : 0.0;
      xb[r] = x;
      if (mine) {
        P[(size_t)t * N + c] = x;
        if (t > c) P[(size_t)c * N + t] = x;
      }
    }
  }
}

template <int W>
void launch_banded(const double* R, double* P, int T, int B, unsigned long long* status, cudaStream_t st) {
  const int gx = (T + kBandBlock - 1) / kBandBlock;
  for (int b0 = 0; b0 < B; b0 += kMaxGridY) {
    const int nb = min(kMaxGridY, B - b0);
    cholinv_banded_kernel<W><<<dim3(gx, nb), kBandBlock, 0, st>>>(R + (size_t)b0 * T * T, P + (size_t)b0 * T * T, T,
                                                                 b0, status);
    count_launch();
  }
}

}  // namespace
}  // namespace nnk

using namespace nnk;

extern "C" int nnk_cholesky_inv(const double* L, int32_t lower, int32_t N, int32_t B, double* P, uint64_t* status_word,
                                void* stream) {
  NNK_REQUIRE(N >= 0 && B >= 0, NNK_ERR_ARG, "N and B must be >= 0");
  if (N == 0 || B == 0) return NNK_OK;
  NNK_REQUIRE(L && P && status_word, NNK_ERR_ARG, "NULL pointer");
  NNK_REQUIRE((const void*)L != (const void*)P, NNK_ERR_ARG, "P must not alias L (it is the substitutions' scratch)");
  DeviceGuard guard(P);
  cudaStream_t st = (cudaStream_t)stream;
  const int gx = (N + kDenseBlock - 1) / kDenseBlock;
  for (int b0 = 0; b0 < B; b0 += kMaxGridY) {
    const int nb = min(kMaxGridY, B - b0);
    const double* Lb = L + (size_t)b0 * N * N;
    double* Pb = P + (size_t)b0 * N * N;
    unsigned long long* s = (unsigned long long*)status_word;
    if (lower) cholinv_dense_kernel<true><<<dim3(gx, nb), kDenseBlock, 0, st>>>(Lb, Pb, N, b0, s);
    else cholinv_dense_kernel<false><<<dim3(gx, nb), kDenseBlock, 0, st>>>(Lb, Pb, N, b0, s);
    count_launch();
  }
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

extern "C" int nnk_cholesky_inv_banded(const double* R, int32_t width, int32_t T, int32_t B, double* P,
                                       uint64_t* status_word, void* stream) {
  NNK_REQUIRE(T >= 0 && B >= 0, NNK_ERR_ARG, "T and B must be >= 0");
  NNK_REQUIRE(width >= 1, NNK_ERR_ARG, "width must be >= 1");
  if (T == 0 || B == 0) return NNK_OK;
  NNK_REQUIRE(R && P && status_word, NNK_ERR_ARG, "NULL pointer");
  NNK_REQUIRE((const void*)R != (const void*)P, NNK_ERR_ARG, "P must not alias R (it holds R^-1 between the passes)");
  const int w = width < T ? width : T;  // rows beyond the matrix contribute nothing
  NNK_REQUIRE(w <= kMaxBand, NNK_ERR_UNSUPPORTED, "band width > 9 is not supported by the CUDA kernel");
  DeviceGuard guard(P);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* s = (unsigned long long*)status_word;
  switch (w) {
    case 1: launch_banded<1>(R, P, T, B, s, st); break;
    case 2: launch_banded<2>(R, P, T, B, s, st); break;
    case 3: launch_banded<3>(R, P, T, B, s, st); break;
    case 4: launch_banded<4>(R, P, T, B, s, st); break;
    case 5: launch_banded<5>(R, P, T, B, s, st); break;
    case 6: launch_banded<6>(R, P, T, B, s, st); break;
    case 7: launch_banded<7>(R, P, T, B, s, st); break;
    case 8: launch_banded<8>(R, P, T, B, s, st); break;
    default: launch_banded<9>(R, P, T, B, s, st); break;
  }
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}
