// nnk_gmm_traj.cu -- trajectory EM of GMM-based voice conversion (baseline.gmm.MLPG.transform_em) on sm_90a,
// float64 (C ABI: include/nnk_b200.h).
//
// The E-step of the EM of Toda, Black & Tokuda 2007, Sec. III, with the diagonal Eq. 23 variances: for every
// frame t and mixture m the log-weight
//   lw_{t,m} = lp[t][m] + log_norm[m] - 1/2 |Y_t - E_{m,t}|^2_{1 / D_m},   E_{m,t} = nu_m + A_m (x_t - mu_m),
// (on an utterance's edge frames over the static columns only, see include/nnk_b200.h), its softmax over m, and the precision-weighted statistics the M-step (one MLPG solve) needs.  One kernel,
// gmm_traj_em_kernel<EPL, EM>: a CTA owns a tile of TRAJ_FT frames of one utterance; the tile's x rows and the
// c rows of the tile plus the window halo (zero outside the utterance) are staged once, Y_t is formed from the
// window taps into registers, then the mixtures stream through shared memory (A_m^T, mu_m, nu_m, 1 / D_m).
// E_{m,t} is recomputed (D^2 FMAs per frame and mixture: no (T, M, D) temporaries), and an online log-sum-exp
// over m rescales the two D-wide accumulators sum gamma / D_m and sum gamma E / D_m.  Lanes run along the
// output dimension (EPL = ceil(D / 32) per lane), each warp keeps TRAJ_FPW frames.  EM = false is the
// objective-only mode: no accumulators, no E_bar / V.  The per-frame log-sum-exp values of a tile are summed in
// frame order into one partial per tile, so every result is a fixed function of the inputs.
#include <math_constants.h>

#include "nnk_common.cuh"

namespace nnk {

constexpr int TRAJ_FT = NNK_GMM_TRAJ_TILE;    // frames per CTA
constexpr int TRAJ_FPW = 4;                   // frames per warp
constexpr int TRAJ_WARPS = TRAJ_FT / TRAJ_FPW;
constexpr int TRAJ_MAX_EPL = 3;               // D <= 96
constexpr int TRAJ_ROWS = TRAJ_FT + 2 * NNK_MAX_HALF;  // staged c rows: the tile and its halo
static_assert(TRAJ_WARPS * TRAJ_FPW == TRAJ_FT, "tile");

struct TrajParams {
  nnk_gmm_t g;
  nnk_gmm_traj_args_t a;
};

// shared memory (doubles): mat D*D | x FT*D | diff FT*D | c ROWS*S | nu D | invD D | lse FT
__host__ __device__ inline size_t traj_smem_doubles(int D, int S) {
  return (size_t)D * D + 2 * (size_t)TRAJ_FT * D + (size_t)TRAJ_ROWS * S + 2 * (size_t)D + TRAJ_FT;
}

template <int EPL, bool EM>
__global__ void __launch_bounds__(TRAJ_WARPS * 32) gmm_traj_em_kernel(const TrajParams p) {
  extern __shared__ __align__(16) double tsm[];
  const nnk_gmm_traj_args_t& a = p.a;
  const int D = p.g.D, M = p.g.M, S = a.static_dim;
  double* sm_mat = tsm;
  double* sm_x = sm_mat + (size_t)D * D;
  double* sm_diff = sm_x + (size_t)TRAJ_FT * D;
  double* sm_c = sm_diff + (size_t)TRAJ_FT * D;
  double* sm_nu = sm_c + (size_t)TRAJ_ROWS * S;
  double* sm_inv = sm_nu + D;
  double* sm_lse = sm_inv + D;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  // the tile: utterance u (last u with tile_off[u] <= blockIdx.x), frames t0 .. t1 - 1
  const int tile = blockIdx.x;
  int lo = 0, hi = a.n_utt - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(a.tile_off + mid) <= tile) lo = mid; else hi = mid - 1;
  }
  const int ub = __ldg(a.utt_off + lo), ue = __ldg(a.utt_off + lo + 1);
  const int t0 = ub + (tile - __ldg(a.tile_off + lo)) * TRAJ_FT;
  const int nf = min(TRAJ_FT, ue - t0);

  for (int e = threadIdx.x; e < TRAJ_FT * D; e += blockDim.x) {
    const int f = e / D, d = e - f * D;
    sm_x[e] = (f < nf) ? a.x[(int64_t)(t0 + f) * a.x_ld + d] : 0.0;
  }
  for (int e = threadIdx.x; e < TRAJ_ROWS * S; e += blockDim.x) {
    const int r = e / S, s = e - r * S;
    const int t = t0 - NNK_MAX_HALF + r;
    sm_c[e] = (t >= ub && t < ue) ? a.c[(int64_t)t * a.c_ld + s] : 0.0;
  }
  __syncthreads();

  // Y_t of the warp's frames, lane + 32 k = w * S + s
  double Y[TRAJ_FPW][EPL];
#pragma unroll
  for (int k = 0; k < EPL; ++k) {
    const int i = lane + 32 * k;
    const int w = (i < D) ? i / S : 0, s = (i < D) ? i - w * S : 0;
    const int l = a.win.l[w], u = a.win.u[w];
#pragma unroll
    for (int f = 0; f < TRAJ_FPW; ++f) {
      const int fi = warp * TRAJ_FPW + f;
      double y = 0.0;
      for (int j = -l; j <= u; ++j) y = fma(a.win.coef[w][l + j], sm_c[(fi + NNK_MAX_HALF + j) * S + s], y);
      Y[f][k] = y;
    }
  }

  // mlpg gives the dynamic windows (w >= 1) zero precision on the first and last H frames of an utterance
  // (H the widest half-width of the set), and on every frame when H = 0 (the reference's [-0:] slice is the
  // whole column, as m_edge == 0 in nnk_mlpg.cu); the model leaves those columns out there as well
  int H = 0;
  for (int w = 0; w < a.win.nw; ++w) H = max(H, max(a.win.l[w], a.win.u[w]));
  bool edge[TRAJ_FPW];
#pragma unroll
  for (int f = 0; f < TRAJ_FPW; ++f) {
    const int t = t0 + warp * TRAJ_FPW + f;
    edge[f] = (H == 0) || (t - ub < H) || (ue - 1 - t < H);
  }

  double mx[TRAJ_FPW], sum[TRAJ_FPW];
  double accP[EM ? TRAJ_FPW : 1][EPL], accPE[EM ? TRAJ_FPW : 1][EPL];
#pragma unroll
  for (int f = 0; f < TRAJ_FPW; ++f) {
    mx[f] = -CUDART_INF;
    sum[f] = 0.0;
  }
#pragma unroll
  for (int f = 0; f < (EM ? TRAJ_FPW : 1); ++f)
#pragma unroll
    for (int k = 0; k < EPL; ++k) accP[f][k] = accPE[f][k] = 0.0;

  for (int m = 0; m < M; ++m) {
    __syncthreads();
    const double* At = p.g.A_t + (size_t)m * D * D;
    const double* mu = p.g.src_means + (size_t)m * D;
    for (int e = threadIdx.x; e < D * D; e += blockDim.x) sm_mat[e] = At[e];
    for (int e = threadIdx.x; e < TRAJ_FT * D; e += blockDim.x) {
      const int f = e / D, d = e - f * D;
      sm_diff[e] = sm_x[e] - mu[d];
    }
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
      sm_nu[d] = p.g.tgt_means[(size_t)m * D + d];
      sm_inv[d] = a.inv_Dm[(size_t)m * D + d];
    }
    __syncthreads();

    // acc[f][k] = (A_m (x - mu_m))[lane + 32 k]
    double acc[TRAJ_FPW][EPL];
#pragma unroll
    for (int f = 0; f < TRAJ_FPW; ++f)
#pragma unroll
      for (int k = 0; k < EPL; ++k) acc[f][k] = 0.0;
    const double* df = sm_diff + (size_t)(warp * TRAJ_FPW) * D;
    for (int d = 0; d < D; ++d) {
      double mv[EPL];
#pragma unroll
      for (int k = 0; k < EPL; ++k) {
        const int i = lane + 32 * k;
        mv[k] = (i < D) ? sm_mat[(size_t)d * D + i] : 0.0;
      }
#pragma unroll
      for (int f = 0; f < TRAJ_FPW; ++f) {
        const double v = df[(size_t)f * D + d];
#pragma unroll
        for (int k = 0; k < EPL; ++k) acc[f][k] = fma(v, mv[k], acc[f][k]);
      }
    }

    const double lnorm_all = __ldg(a.log_norm + 2 * m), lnorm_static = __ldg(a.log_norm + 2 * m + 1);
#pragma unroll
    for (int f = 0; f < TRAJ_FPW; ++f) {
      double q = 0.0;
#pragma unroll
      for (int k = 0; k < EPL; ++k) {
        const int i = lane + 32 * k;
        if (i < D) {
          acc[f][k] += sm_nu[i];  // E_{m,t}
          const double r = Y[f][k] - acc[f][k];
          if (i < S || !edge[f]) q = fma(r * r, sm_inv[i], q);
        }
      }
      const double lnorm = edge[f] ? lnorm_static : lnorm_all;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      const int fi = warp * TRAJ_FPW + f;
      if (fi >= nf) continue;  // warp-uniform
      const double lw = __ldg(a.lp + (int64_t)(t0 + fi) * M + m) + lnorm - 0.5 * q;
      if (!(lw > -CUDART_INF)) continue;  // gamma = 0 (also skips NaN, which the caller has excluded)
      // online log-sum-exp: the larger of (mx, lw) is the new reference
      double scale_old = 1.0, wgt = 1.0;
      if (lw > mx[f]) {
        scale_old = exp(mx[f] - lw);
        mx[f] = lw;
      } else {
        wgt = exp(lw - mx[f]);
      }
      sum[f] = fma(sum[f], scale_old, wgt);
      if (EM) {
#pragma unroll
        for (int k = 0; k < EPL; ++k) {
          const int i = lane + 32 * k;
          const double wi = (i < D) ? wgt * sm_inv[i] : 0.0;
          accP[f][k] = fma(accP[f][k], scale_old, wi);
          accPE[f][k] = fma(accPE[f][k], scale_old, wi * acc[f][k]);
        }
      }
    }
  }

#pragma unroll
  for (int f = 0; f < TRAJ_FPW; ++f) {
    const int fi = warp * TRAJ_FPW + f;
    if (lane == 0) sm_lse[fi] = (fi < nf) ? mx[f] + log(sum[f]) : 0.0;
    if (EM && fi < nf) {
      const int64_t row = (int64_t)(t0 + fi) * D;
#pragma unroll
      for (int k = 0; k < EPL; ++k) {
        const int i = lane + 32 * k;
        if (i < D) {
          a.E_bar[row + i] = accPE[f][k] / accP[f][k];
          a.V[row + i] = sum[f] / accP[f][k];
        }
      }
    }
  }
  if (a.ll_part) {
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int f = 0; f < nf; ++f) s += sm_lse[f];
      a.ll_part[tile] = s;
    }
  }
}

template <int EPL, bool EM>
static int traj_launch(const TrajParams& p, cudaStream_t st) {
  const size_t smem = sizeof(double) * traj_smem_doubles(p.g.D, p.a.static_dim);
  NNK_CUDA_CHECK(cudaFuncSetAttribute(gmm_traj_em_kernel<EPL, EM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  gmm_traj_em_kernel<EPL, EM><<<(unsigned)p.a.n_tiles, TRAJ_WARPS * 32, smem, st>>>(p);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

template <bool EM>
static int traj_dispatch(const TrajParams& p, cudaStream_t st) {
  const int epl = (p.g.D + 31) / 32;
  if (epl == 1) return traj_launch<1, EM>(p, st);
  if (epl == 2) return traj_launch<2, EM>(p, st);
  return traj_launch<3, EM>(p, st);
}

}  // namespace nnk

using namespace nnk;

extern "C" int nnk_gmm_traj_em(const nnk_gmm_t* g, const nnk_gmm_traj_args_t* a, void* stream) {
  NNK_REQUIRE(g && a, NNK_ERR_ARG, "NULL pointer");
  NNK_REQUIRE(g->src_means && g->tgt_means && g->A_t, NNK_ERR_ARG, "NULL GMM table");
  NNK_REQUIRE(g->M >= 1 && g->D >= 1, NNK_ERR_ARG, "bad GMM size");
  NNK_REQUIRE(a->mode == NNK_GMM_TRAJ_EM || a->mode == NNK_GMM_TRAJ_OBJECTIVE, NNK_ERR_ARG,
              "mode must be NNK_GMM_TRAJ_EM or NNK_GMM_TRAJ_OBJECTIVE");
  NNK_REQUIRE(a->T >= 0 && a->n_utt >= 1 && a->n_tiles >= 0 && a->static_dim >= 1, NNK_ERR_ARG, "bad size");
  NNK_REQUIRE(a->win.nw >= 1 && a->win.nw <= NNK_MAX_WIN, NNK_ERR_ARG, "bad window count");
  for (int w = 0; w < a->win.nw; ++w)
    NNK_REQUIRE(a->win.l[w] >= 0 && a->win.u[w] >= 0 && a->win.l[w] <= NNK_MAX_HALF && a->win.u[w] <= NNK_MAX_HALF,
                NNK_ERR_ARG, "window half-width out of range");
  NNK_REQUIRE((int64_t)a->win.nw * a->static_dim == g->D, NNK_ERR_ARG, "D != nw * static_dim");
  NNK_REQUIRE(a->x_ld >= g->D && a->c_ld >= a->static_dim, NNK_ERR_ARG, "bad leading dimension");
  NNK_REQUIRE(a->x && a->lp && a->c && a->utt_off && a->tile_off && a->inv_Dm && a->log_norm, NNK_ERR_ARG, "NULL input");
  NNK_REQUIRE(a->mode == NNK_GMM_TRAJ_OBJECTIVE || (a->E_bar && a->V), NNK_ERR_ARG, "NULL E_bar / V");
  NNK_REQUIRE(a->mode == NNK_GMM_TRAJ_EM || a->ll_part, NNK_ERR_ARG, "NULL ll_part");
  NNK_REQUIRE(g->D <= 32 * TRAJ_MAX_EPL, NNK_ERR_UNSUPPORTED, "feature dimension > 96 is not supported by the GMM kernels");
  NNK_REQUIRE(g->M <= 65535, NNK_ERR_UNSUPPORTED, "more than 65535 mixtures");
  if (a->T == 0 || a->n_tiles == 0) return NNK_OK;
  DeviceGuard guard(a->x);
  TrajParams p{};
  p.g = *g;
  p.a = *a;
  cudaStream_t st = (cudaStream_t)stream;
  return a->mode == NNK_GMM_TRAJ_EM ? traj_dispatch<true>(p, st) : traj_dispatch<false>(p, st);
}
