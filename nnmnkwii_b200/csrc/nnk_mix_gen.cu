// nnk_mix_gen.cu -- parameter generation from mixture outputs (paramgen.mlpg_mixture_batch) on sm_90a, float64
// arithmetic (C ABI: nnk_mix_gen in include/nnk_b200.h, definition: DESIGN.md 3.19).
//
// The E-step of the EM of Tokuda et al. (ICASSP 2000) over explicit per-frame mixtures: for every frame t and
// component m the log-weight  l_{t,m} = lnorm_{t,m} - 1/2 |Y_t - mu_{t,m}|^2_{1 / s2_{t,m}}  over the columns
// that count at t, its softmax over m and the precision-weighted statistics the M-step (one MLPG solve) needs.
// One kernel family, mix_gen_kernel<EPL, MODE, T>: a CTA owns a tile of MIX_FT frames of one utterance; in the
// ESTEP / OBJECTIVE modes the tile's c rows plus the window halo (zero outside the utterance) are staged once.
// Each warp takes MIX_FPW frames one after the other, lanes along the input columns (EPL = columns per lane),
// forms Y_t from the window taps in registers, then streams the frame's M contiguous (mu, s2) rows: one warp
// reduction per component for the squared distance and an online log-sum-exp over m that rescales the two
// accumulators sum gamma / s2 and sum gamma mu / s2, so each row is read once per launch.  The c-independent
// log-normaliser is tabulated by the SELECT launch, so the E-step evaluates no log but the one per frame of the
// objective.  The per-frame log-sum-exp values of a tile are summed in frame order into one partial per tile:
// every result is a fixed function of the inputs.
//
// gmm_traj_em_kernel (csrc/nnk_gmm_traj.cu) runs the same EM for GMM voice conversion but forms Y_t by
// w * static_dim + s over one stream and recomputes its component means from x; this kernel reads Y_t's columns
// through the layout's column map (several streams, copied columns).  The two keep separate code, see DESIGN.md
// 3.19.
#include <math_constants.h>

#include "nnk_common.cuh"

namespace nnk {

constexpr int MIX_FT = NNK_MIX_GEN_TILE;  // frames per CTA
constexpr int MIX_WARPS = 8;
constexpr int MIX_FPW = MIX_FT / MIX_WARPS;  // frames per warp
constexpr double MIX_LOG_2PI = 1.83787706640934548356;
static_assert(MIX_WARPS * MIX_FPW == MIX_FT, "tile");

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void report_mix(unsigned long long* status, int64_t row, int kind) {
  atomicMax(status, ~(((unsigned long long)row << 2) | (unsigned long long)kind));
}

// shared memory (doubles): lse FT | c (FT + 2H) * c_cols   (ESTEP / OBJECTIVE only)
__host__ __device__ inline size_t mix_smem_doubles(int H, int c_cols) {
  return (size_t)MIX_FT + (size_t)(MIX_FT + 2 * H) * c_cols;
}

template <int EPL, int MODE, typename T>
__global__ void __launch_bounds__(MIX_WARPS * 32, 2) mix_gen_kernel(const nnk_mix_gen_args_t a) {
  extern __shared__ __align__(16) double msm[];
  const int M = a.M, D = a.D;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  // the tile: utterance u (last u with tile_off[u] <= blockIdx.x), frames t0 .. t0 + nf - 1
  const int tile = blockIdx.x;
  int lo = 0, hi = a.n_utt - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(a.tile_off + mid) <= tile) lo = mid; else hi = mid - 1;
  }
  const int ub = __ldg(a.utt_off + lo), ue = ub + __ldg(a.utt_len + lo);
  const int t0 = ub + (tile - __ldg(a.tile_off + lo)) * MIX_FT;
  const int nf = min(MIX_FT, ue - t0);
  int H = 0;
  for (int w = 0; w < a.win.nw; ++w) H = max(H, max(a.win.l[w], a.win.u[w]));

  int code[EPL];
#pragma unroll
  for (int k = 0; k < EPL; ++k) {
    const int i = lane + 32 * k;
    code[k] = (i < D) ? __ldg(a.col_map + i) : -1;
  }

  double* sm_lse = msm;
  double* sm_c = msm + MIX_FT;  // row r holds frame t0 - H + r
  if (MODE != NNK_MIX_GEN_SELECT) {
    const int C = a.c_cols, rows = MIX_FT + 2 * H;
    for (int e = threadIdx.x; e < rows * C; e += blockDim.x) {
      const int r = e / C, s = e - r * C;
      const int t = t0 - H + r;
      sm_c[e] = (t >= ub && t < ue) ? a.c[(int64_t)t * a.c_ld + s] : 0.0;
    }
    __syncthreads();
  }

  for (int f = 0; f < MIX_FPW; ++f) {
    const int fi = warp * MIX_FPW + f;
    if (fi >= nf) break;  // warp-uniform
    const int t = t0 + fi;
    const int64_t row = t;
    // mlpg gives the dynamic windows zero precision on the first and last H frames (every frame when H = 0)
    const bool edge = (H == 0) || (t - ub < H) || (ue - 1 - t < H);
    bool cnt[EPL];
#pragma unroll
    for (int k = 0; k < EPL; ++k) cnt[k] = code[k] >= 0 && ((code[k] & 7) <= 1 || !edge);
    const T* lw_row = static_cast<const T*>(a.log_weights) + row * M;
    const T* mu_row = static_cast<const T*>(a.means) + row * M * D;
    const T* s2_row = static_cast<const T*>(a.vars) + row * M * D;

    if constexpr (MODE == NNK_MIX_GEN_SELECT) {
      // arg-max of the log-weights, the lowest index on ties (np.argmax)
      double best = -CUDART_INF;
      int arg = -1;
      bool bad_lw = false;
      for (int m = 0; m < M; ++m) {
        const double v = (double)__ldg(lw_row + m);
        bad_lw |= isnan(v) || v == CUDART_INF;
        if (v > best) {
          best = v;
          arg = m;
        }
      }
      double n_cnt = 0.0;
#pragma unroll
      for (int k = 0; k < EPL; ++k) n_cnt += cnt[k] ? 1.0 : 0.0;
      n_cnt = warp_sum(n_cnt);
      bool bad_s2 = false;
      for (int m = 0; m < M; ++m) {
        double ls = 0.0;
#pragma unroll
        for (int k = 0; k < EPL; ++k) {
          if (code[k] >= 0) {
            const double v = (double)__ldg(s2_row + (size_t)m * D + lane + 32 * k);
            bad_s2 |= !(v > 0.0 && v < CUDART_INF);
            if (cnt[k]) ls += log(v);
          }
        }
        ls = warp_sum(ls);
        if (lane == 0) a.lnorm[row * M + m] = (double)__ldg(lw_row + m) - 0.5 * fma(n_cnt, MIX_LOG_2PI, ls);
      }
      bad_s2 = __any_sync(0xffffffffu, bad_s2);
      if (lane == 0) {
        const int kind = bad_lw ? 1 : (arg < 0 ? 2 : (bad_s2 ? 3 : 0));
        if (kind) report_mix(reinterpret_cast<unsigned long long*>(a.status_word), row, kind);
      }
      arg = max(arg, 0);
#pragma unroll
      for (int k = 0; k < EPL; ++k) {
        const int i = lane + 32 * k;
        if (i < D) {
          a.E[row * D + i] = (double)__ldg(mu_row + (size_t)arg * D + i);
          a.V[row * D + i] = (double)__ldg(s2_row + (size_t)arg * D + i);
        }
      }
    } else {
      // Y_t of the lane's columns
      double Y[EPL];
  #pragma unroll
      for (int k = 0; k < EPL; ++k) {
        double y = 0.0;
        if (code[k] >= 0) {
          const int oc = code[k] >> 3, kind = code[k] & 7;
          const double* cr = sm_c + (size_t)(fi + H) * a.c_cols + oc;
          if (kind == 0) {
            y = cr[0];
          } else {
            const int w = kind - 1, l = a.win.l[w], u = a.win.u[w];
            for (int j = -l; j <= u; ++j) y = fma(a.win.coef[w][l + j], cr[(ptrdiff_t)j * a.c_cols], y);
          }
        }
        Y[k] = y;
      }

      constexpr bool EM = MODE == NNK_MIX_GEN_ESTEP;
      double mx = -CUDART_INF, sum = 0.0;
      double accP[EM ? EPL : 1], accPE[EM ? EPL : 1];
  #pragma unroll
      for (int k = 0; k < (EM ? EPL : 1); ++k) accP[k] = accPE[k] = 0.0;
      const double* ln_row = a.lnorm + row * M;
      for (int m = 0; m < M; ++m) {
        const double ln = __ldg(ln_row + m);
        if (!(ln > -CUDART_INF)) continue;  // weight 0: gamma = 0 (warp-uniform)
        double mu[EPL], p[EPL];
        double q = 0.0;
  #pragma unroll
        for (int k = 0; k < EPL; ++k) {
          mu[k] = 0.0;
          p[k] = 0.0;
          if (code[k] >= 0) {
            const size_t e = (size_t)m * D + lane + 32 * k;
            mu[k] = (double)__ldg(mu_row + e);
            p[k] = 1.0 / (double)__ldg(s2_row + e);
            const double r = Y[k] - mu[k];
            if (cnt[k]) q = fma(r * r, p[k], q);
          }
        }
        q = warp_sum(q);
        const double lw = ln - 0.5 * q;
        if (!(lw > -CUDART_INF)) continue;
        // online log-sum-exp: the larger of (mx, lw) is the new reference
        double scale_old = 1.0, wgt = 1.0;
        if (lw > mx) {
          scale_old = exp(mx - lw);
          mx = lw;
        } else {
          wgt = exp(lw - mx);
        }
        sum = fma(sum, scale_old, wgt);
        if (EM) {
  #pragma unroll
          for (int k = 0; k < EPL; ++k) {
            const double wi = wgt * p[k];
            accP[k] = fma(accP[k], scale_old, wi);
            accPE[k] = fma(accPE[k], scale_old, wi * mu[k]);
          }
        }
      }
      if (lane == 0) sm_lse[fi] = mx + log(sum);
      if (EM) {
  #pragma unroll
        for (int k = 0; k < EPL; ++k) {
          const int i = lane + 32 * k;
          if (i < D) {
            a.E[row * D + i] = code[k] >= 0 ? accPE[k] / accP[k] : 0.0;
            a.V[row * D + i] = code[k] >= 0 ? sum / accP[k] : 1.0;
          }
        }
      }
    }
  }

  if (MODE != NNK_MIX_GEN_SELECT && a.ll_part) {
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int f = 0; f < nf; ++f) s += sm_lse[f];
      a.ll_part[tile] = s;
    }
  }
}

template <int EPL, int MODE, typename T>
static int mix_launch(const nnk_mix_gen_args_t& a, int H, cudaStream_t st) {
  const size_t smem = MODE == NNK_MIX_GEN_SELECT ? 0 : sizeof(double) * mix_smem_doubles(H, a.c_cols);
  NNK_CUDA_CHECK(cudaFuncSetAttribute(mix_gen_kernel<EPL, MODE, T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem));
  mix_gen_kernel<EPL, MODE, T><<<(unsigned)a.n_tiles, MIX_WARPS * 32, smem, st>>>(a);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

template <int MODE, typename T>
static int mix_dispatch(const nnk_mix_gen_args_t& a, int H, cudaStream_t st) {
  if (a.D <= 32) return mix_launch<1, MODE, T>(a, H, st);
  if (a.D <= 64) return mix_launch<2, MODE, T>(a, H, st);
  if (a.D <= 128) return mix_launch<4, MODE, T>(a, H, st);
  return mix_launch<8, MODE, T>(a, H, st);
}

template <typename T>
static int mix_mode(const nnk_mix_gen_args_t& a, int H, cudaStream_t st) {
  if (a.mode == NNK_MIX_GEN_SELECT) return mix_dispatch<NNK_MIX_GEN_SELECT, T>(a, H, st);
  if (a.mode == NNK_MIX_GEN_ESTEP) return mix_dispatch<NNK_MIX_GEN_ESTEP, T>(a, H, st);
  return mix_dispatch<NNK_MIX_GEN_OBJECTIVE, T>(a, H, st);
}

}  // namespace nnk

using namespace nnk;

extern "C" int nnk_mix_gen(const nnk_mix_gen_args_t* a, void* stream) {
  NNK_REQUIRE(a, NNK_ERR_ARG, "NULL pointer");
  NNK_REQUIRE(a->mode == NNK_MIX_GEN_SELECT || a->mode == NNK_MIX_GEN_ESTEP || a->mode == NNK_MIX_GEN_OBJECTIVE,
              NNK_ERR_ARG, "mode must be NNK_MIX_GEN_SELECT, NNK_MIX_GEN_ESTEP or NNK_MIX_GEN_OBJECTIVE");
  NNK_REQUIRE(a->dtype == NNK_F32 || a->dtype == NNK_F64, NNK_ERR_ARG, "dtype must be NNK_F32 or NNK_F64");
  NNK_REQUIRE(a->M >= 1 && a->D >= 1 && a->n_utt >= 1 && a->n_tiles >= 0, NNK_ERR_ARG, "bad size");
  NNK_REQUIRE(a->win.nw >= 1 && a->win.nw <= NNK_MAX_WIN, NNK_ERR_ARG, "bad window count");
  for (int w = 0; w < a->win.nw; ++w)
    NNK_REQUIRE(a->win.l[w] >= 0 && a->win.u[w] >= 0 && a->win.l[w] <= NNK_MAX_HALF && a->win.u[w] <= NNK_MAX_HALF,
                NNK_ERR_ARG, "window half-width out of range");
  NNK_REQUIRE(a->log_weights && a->means && a->vars && a->utt_off && a->utt_len && a->tile_off && a->col_map &&
                  a->lnorm, NNK_ERR_ARG, "NULL input");
  NNK_REQUIRE(a->mode == NNK_MIX_GEN_OBJECTIVE || (a->E && a->V), NNK_ERR_ARG, "NULL E / V");
  NNK_REQUIRE(a->mode != NNK_MIX_GEN_SELECT || a->status_word, NNK_ERR_ARG, "NULL status word");
  NNK_REQUIRE(a->mode != NNK_MIX_GEN_OBJECTIVE || a->ll_part, NNK_ERR_ARG, "NULL ll_part");
  NNK_REQUIRE(a->mode == NNK_MIX_GEN_SELECT || (a->c && a->c_cols >= 1 && a->c_ld >= a->c_cols), NNK_ERR_ARG,
              "bad c");
  NNK_REQUIRE(a->D <= NNK_MIX_GEN_MAX_D, NNK_ERR_UNSUPPORTED, "more than 256 input columns");
  NNK_REQUIRE(a->M <= NNK_MIX_GEN_MAX_M, NNK_ERR_UNSUPPORTED, "more than 64 mixture components");
  if (a->n_tiles == 0) return NNK_OK;
  int H = 0;
  for (int w = 0; w < a->win.nw; ++w) H = max(H, max(a->win.l[w], a->win.u[w]));
  DeviceGuard guard(a->means);
  cudaStream_t st = (cudaStream_t)stream;
  return a->dtype == NNK_F32 ? mix_mode<float>(*a, H, st) : mix_mode<double>(*a, H, st);
}
