// nnk_postfilter.cu -- Merlin's mel-cepstral post-filter (nnmnkwii/postfilters/__init__.py:7-62), batched.
//
// Per frame c (D coefficients), weight w, warping a, order M, FFT length L the reference runs
//   r0   = c2acr(freqt(c,     M, -a), 0, L)        p_r0 = c2acr(freqt(w * c, M, -a), 0, L)
//   b0   = mc2b(w * c, a)[0]                       out  = b2mc([log(r0 / p_r0) / 2 + b0, mc2b(w * c, a)[1:]], a)
// mc2b and b2mc are exact inverses that differ only in coefficient 0, so out = w * c with
// out[0] += log(r0 / p_r0) / 2.  freqt is linear in c (a fixed (M+1) x D matrix F) and c2acr(., 0, L)
// is (1/L) sum_k exp(2 Re FFT_k), whose real part is a cosine map with bins k and L - k equal, so
//   r0(c) = (1/L) sum_{k=0}^{L/2} omega_k exp(2 (B c)_k),  B = Cos F  ((L/2+1) x D),  omega = 1, 2, .., 2, 1.
// The 1/L cancels in r0 / p_r0.
//
// postfilter_basis_kernel builds B once per (alpha, D, M, L) in float64: SPTK's freqt recursion run on
// each unit vector e_d (it truncates at order M, which the analytic warped-frequency map does not),
// then the cosine map through a table of cospi(2 m / L), m = k n mod L (exact arguments).  B is written
// in the filter kernel's B-fragment order (see pf_basis_index), zero-padded to 8-bin tiles and 16-wide
// k-steps, so a chunk of bins is one contiguous range.
//
// postfilter_kernel<T, KS>: a CTA of PF_WARPS warps takes 8 * PF_WARPS frames.  Warp rows 0-7 are c of
// its 8 frames, rows 8-15 are w * c of the same frames, so after the GEMM each lane holds both sums of
// its frame.  The A fragments (m16 x k16, KS = ceil(D / 16) k-steps) are loaded once straight from the
// strided rows into registers (every element is read by exactly one lane) and widened to float64; B
// streams through two shared-memory stages of PF_CH(KS) bin tiles by cp.async, from L2 where the whole
// basis stays (263 KB at D = 60, L = 1024).  The GEMM runs on the FP64 tensor cores
// (mma.sync.m16n8k16.f64 -> DMMA.16x8x16).  The epilogue of every bin tile takes exp(2 acc) in float64
// (libdevice exp, ~1 ulp), weights it by omega_k (0 past the last bin) and folds it into per-lane sums;
// a quad shuffle completes the sums of a frame, and the lanes write w * c with the column-0 correction
// in the input dtype.  No (frames x bins) intermediate leaves the SM.
// -DNNK_PF_NO_EXP replaces the exponential by 1 + 2 acc (a timing build that splits off the exp phase;
// its results are wrong).
#include "nnk_common.cuh"

namespace nnk {

constexpr int PF_WARPS = 8;                 // warps per CTA of the filter kernel
constexpr int PF_FRAMES = 8 * PF_WARPS;     // frames per CTA
constexpr int PF_MAX_KS = 8;                // D <= 128
constexpr int PF_MAX_FFTLEN = 8192;         // basis kernel: (M + 1 + L) doubles of shared memory
constexpr int pf_ch(int ks) { return ks >= 32 ? 1 : 32 / ks; }  // bin tiles per stage: 32 KB per stage

static inline int64_t pf_basis_elems(int D, int L) {
  const int64_t nt = ((int64_t)L / 2 + 1 + 7) / 8, ks = (D + 15) / 16;
  return nt * ks * 128;
}

// element (bin k, coefficient d) of B inside fragment (tile k / 8, k-step d / 16): lane = 4 (k % 8) + d % 4,
// value v = (d % 16) / 4 -- the B operand layout of mma.m16n8k16.f64 (b_v: k-row tig + 4 v, n-col groupID)
__device__ __forceinline__ int64_t pf_basis_index(int k, int d, int KS) {
  const int lane = 4 * (k & 7) + (d & 3), v = (d & 15) >> 2;
  return ((((int64_t)(k >> 3) * KS + (d >> 4)) * 32 + lane) << 2) + v;
}

// One CTA per coefficient d < 16 KS.  Thread 0 runs SPTK's freqt (freqt.c) on e_d in place in shared
// memory while the others fill the cosine table; then threads stride over the bins of the padded range.
__global__ void __launch_bounds__(256) postfilter_basis_kernel(double a, int D, int M, int L, int KS, int n_bins_pad,
                                                               double* __restrict__ basis) {
  extern __shared__ double sm[];
  double* g = sm;            // M + 1 freqt coefficients
  double* tab = sm + M + 1;  // L cosines
  const int d = blockIdx.x;
  if (d < D) {
    if (threadIdx.x == 0) {
      for (int j = 0; j <= M; ++j) g[j] = 0.0;
      // freqt(c1 = e_d, m1 = D - 1, c2 = g, m2 = M, a): for i = m1 .. 0 over c1[i]; steps with i > d
      // see zeros and leave g = 0
      const double b = 1.0 - a * a;
      for (int i = d; i >= 0; --i) {
        const double x = (i == d) ? 1.0 : 0.0;
        double d_prev = g[0];  // d[j - 1]: g[j - 1] before this step
        double g_prev = x + a * d_prev;
        g[0] = g_prev;
        if (M >= 1) {
          const double dj = g[1];
          g_prev = b * d_prev + a * dj;
          g[1] = g_prev;
          d_prev = dj;
        }
        for (int j = 2; j <= M; ++j) {
          const double dj = g[j];
          g_prev = d_prev + a * (dj - g_prev);
          g[j] = g_prev;
          d_prev = dj;
        }
      }
    }
    for (int m = threadIdx.x; m < L; m += blockDim.x) tab[m] = cospi((double)(2 * m) / (double)L);
  }
  __syncthreads();
  const int K = L / 2 + 1;
  for (int k = threadIdx.x; k < n_bins_pad; k += blockDim.x) {
    double s = 0.0;
    if (d < D && k < K)
      for (int n = 0; n <= M; ++n) s += tab[(int)(((int64_t)k * n) & (L - 1))] * g[n];
    basis[pf_basis_index(k, d, KS)] = s;
  }
}

struct PfParams {
  const void* x;
  void* out;
  int64_t x_ld, out_ld, N;
  const double* weight;
  const double* basis;
  int D, L, n_tiles;  // n_tiles = ceil((L/2 + 1) / 8)
};

__device__ __forceinline__ void mma_f64_16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src)
               : "memory");
}

__device__ __forceinline__ double pf_exp2x(double acc) {
#ifdef NNK_PF_NO_EXP
  return fma(2.0, acc, 1.0);
#else
  return exp(2.0 * acc);
#endif
}

template <typename T, int KS>
__global__ void __launch_bounds__(32 * PF_WARPS, KS <= 4 ? 2 : 1) postfilter_kernel(const __grid_constant__ PfParams p) {
  constexpr int CH = pf_ch(KS);
  constexpr int TILE_DBL = KS * 128;  // doubles of one bin tile (8 bins x 16 KS coefficients)
  extern __shared__ __align__(16) double stage[];  // 2 x CH x TILE_DBL
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int grp = lane >> 2, tig = lane & 3;
  const int64_t frame = (int64_t)blockIdx.x * PF_FRAMES + warp * 8 + grp;
  const bool live = frame < p.N;

  // A fragments: a[ks][2v] = c[frame][col], a[ks][2v + 1] = w[col] c[frame][col], col = 16 ks + tig + 4 v
  double a[KS][8];
  const T* xr = reinterpret_cast<const T*>(p.x) + (live ? frame : 0) * p.x_ld;
#pragma unroll
  for (int ks = 0; ks < KS; ++ks)
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int col = 16 * ks + tig + 4 * v;
      const double c = (live && col < p.D) ? (double)__ldg(xr + col) : 0.0;
      a[ks][2 * v] = c;
      a[ks][2 * v + 1] = col < p.D ? p.weight[col] * c : 0.0;
    }

  const int n_chunks = (p.n_tiles + CH - 1) / CH;
  auto issue = [&](int chunk) {
    const int t0 = chunk * CH, nt = min(CH, p.n_tiles - t0);
    const double* src = p.basis + (int64_t)t0 * TILE_DBL;
    double* dst = stage + (chunk & 1) * CH * TILE_DBL;
    for (int i = threadIdx.x; i < nt * TILE_DBL / 2; i += 32 * PF_WARPS) cp_async16(dst + 2 * i, src + 2 * i);
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  const int K = p.L / 2 + 1, half = p.L / 2;
  double s_c = 0.0, s_w = 0.0;  // this lane's share of sum_k omega_k exp(2 (B c)_k), rows grp and grp + 8
  issue(0);
#pragma unroll 1
  for (int chunk = 0; chunk < n_chunks; ++chunk) {
    if (chunk + 1 < n_chunks) {
      issue(chunk + 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const double* buf = stage + (chunk & 1) * CH * TILE_DBL;
    const int nt = min(CH, p.n_tiles - chunk * CH);
#pragma unroll 1
    for (int t = 0; t < nt; ++t) {
      double acc[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        const double2* bp = reinterpret_cast<const double2*>(buf + (t * KS + ks) * 128 + 4 * lane);
        const double2 b01 = bp[0], b23 = bp[1];
        const double b[4] = {b01.x, b01.y, b23.x, b23.y};
        mma_f64_16816(acc, a[ks], b);
      }
      // acc[0..1]: row grp (c), bins k0, k0 + 1; acc[2..3]: row grp + 8 (w * c), same bins
      const int k0 = 8 * (chunk * CH + t) + 2 * tig;
      const double om0 = k0 >= K ? 0.0 : (k0 == 0 || k0 == half) ? 1.0 : 2.0;
      const double om1 = k0 + 1 >= K ? 0.0 : (k0 + 1 == half) ? 1.0 : 2.0;
      s_c += om0 * pf_exp2x(acc[0]) + om1 * pf_exp2x(acc[1]);
      s_w += om0 * pf_exp2x(acc[2]) + om1 * pf_exp2x(acc[3]);
    }
    __syncthreads();  // every warp is done with this stage before the next issue overwrites it
  }
  s_c += __shfl_xor_sync(0xffffffffu, s_c, 1);
  s_w += __shfl_xor_sync(0xffffffffu, s_w, 1);
  s_c += __shfl_xor_sync(0xffffffffu, s_c, 2);
  s_w += __shfl_xor_sync(0xffffffffu, s_w, 2);
  if (!live) return;
  const double corr = 0.5 * log(s_c / s_w);  // log(r0 / p_r0) / 2; an all-zero frame gives s_c == s_w == L
  T* orow = reinterpret_cast<T*>(p.out) + frame * p.out_ld;
#pragma unroll
  for (int ks = 0; ks < KS; ++ks)
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int col = 16 * ks + tig + 4 * v;
      if (col < p.D) orow[col] = (T)(col == 0 ? a[ks][2 * v + 1] + corr : a[ks][2 * v + 1]);
    }
}

template <typename T, int KS>
static int pf_launch(const PfParams& p, cudaStream_t st) {
  const size_t smem = sizeof(double) * 2 * pf_ch(KS) * KS * 128;
  NNK_CUDA_CHECK(cudaFuncSetAttribute(postfilter_kernel<T, KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const unsigned grid = (unsigned)((p.N + PF_FRAMES - 1) / PF_FRAMES);
  postfilter_kernel<T, KS><<<grid, 32 * PF_WARPS, smem, st>>>(p);
  return NNK_OK;
}

template <typename T>
static int pf_dispatch(const PfParams& p, int KS, cudaStream_t st) {
  switch (KS) {
    case 1: return pf_launch<T, 1>(p, st);
    case 2: return pf_launch<T, 2>(p, st);
    case 3: return pf_launch<T, 3>(p, st);
    case 4: return pf_launch<T, 4>(p, st);
    case 5: return pf_launch<T, 5>(p, st);
    case 6: return pf_launch<T, 6>(p, st);
    case 7: return pf_launch<T, 7>(p, st);
    default: return pf_launch<T, 8>(p, st);
  }
}

static int pf_check_geometry(int32_t D, int32_t order, int32_t fftlen) {
  NNK_REQUIRE(D >= 1, NNK_ERR_ARG, "D must be >= 1");
  NNK_REQUIRE(fftlen >= 1 && (fftlen & (fftlen - 1)) == 0, NNK_ERR_ARG, "fftlen must be a power of two");
  NNK_REQUIRE(order >= 0, NNK_ERR_ARG, "minimum_phase_order must be >= 0");
  NNK_REQUIRE(order + 1 <= fftlen, NNK_ERR_ARG, "minimum_phase_order + 1 must not exceed fftlen");
  NNK_REQUIRE(D <= 16 * PF_MAX_KS, NNK_ERR_UNSUPPORTED, "more than 128 coefficients per frame");
  NNK_REQUIRE(fftlen <= PF_MAX_FFTLEN, NNK_ERR_UNSUPPORTED, "fftlen > 8192 is not supported by the basis kernel");
  return NNK_OK;
}

}  // namespace nnk

using namespace nnk;

extern "C" int64_t nnk_postfilter_basis_elems(int32_t D, int32_t fftlen) {
  if (D < 1 || D > 16 * PF_MAX_KS || fftlen < 1 || fftlen > PF_MAX_FFTLEN || (fftlen & (fftlen - 1))) return 0;
  return pf_basis_elems(D, fftlen);
}

extern "C" int nnk_postfilter_basis(double alpha, int32_t D, int32_t order, int32_t fftlen, double* basis,
                                    int64_t basis_elems, void* stream) {
  NNK_REQUIRE(basis, NNK_ERR_ARG, "NULL pointer");
  int rc = pf_check_geometry(D, order, fftlen);
  if (rc) return rc;
  NNK_REQUIRE(basis_elems == pf_basis_elems(D, fftlen), NNK_ERR_ARG, "basis_elems != nnk_postfilter_basis_elems(D, fftlen)");
  DeviceGuard guard(basis);
  const int KS = (D + 15) / 16, n_bins_pad = 8 * ((fftlen / 2 + 1 + 7) / 8);
  const size_t smem = sizeof(double) * ((size_t)order + 1 + fftlen);
  NNK_CUDA_CHECK(cudaFuncSetAttribute(postfilter_basis_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  postfilter_basis_kernel<<<16 * KS, 256, smem, (cudaStream_t)stream>>>(-alpha, D, order, fftlen, KS, n_bins_pad, basis);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

extern "C" int nnk_postfilter_apply(const void* mgc, int32_t dtype, int64_t N, int32_t D, int64_t ld, const double* weight,
                                    int32_t fftlen, const double* basis, int64_t basis_elems, void* out, int64_t out_ld,
                                    void* stream) {
  NNK_REQUIRE(mgc && weight && basis && out, NNK_ERR_ARG, "NULL pointer");
  NNK_REQUIRE(dtype == NNK_F32 || dtype == NNK_F64, NNK_ERR_ARG, "bad dtype");
  int rc = pf_check_geometry(D, 0, fftlen);
  if (rc) return rc;
  NNK_REQUIRE(N >= 0 && ld >= D && out_ld >= D, NNK_ERR_ARG, "bad size or row stride");
  NNK_REQUIRE(basis_elems == pf_basis_elems(D, fftlen), NNK_ERR_ARG, "basis_elems != nnk_postfilter_basis_elems(D, fftlen)");
  NNK_REQUIRE((N + PF_FRAMES - 1) / PF_FRAMES <= 0x7fffffff, NNK_ERR_ARG, "too many frames for one launch");
  if (N == 0) return NNK_OK;
  DeviceGuard guard(mgc);
  PfParams p;
  p.x = mgc; p.out = out; p.x_ld = ld; p.out_ld = out_ld; p.N = N; p.weight = weight; p.basis = basis;
  p.D = D; p.L = fftlen; p.n_tiles = (fftlen / 2 + 1 + 7) / 8;
  const int KS = (D + 15) / 16;
  cudaStream_t st = (cudaStream_t)stream;
  rc = dtype == NNK_F32 ? pf_dispatch<float>(p, KS, st) : pf_dispatch<double>(p, KS, st);
  if (rc) return rc;
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}
