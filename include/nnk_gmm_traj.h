/* nnk_gmm_traj.h -- C ABI of the trajectory EM of GMM-based voice conversion in libnnk_b200.so (sm_90a).
 *
 * Same conventions as nnk_b200.h (return codes, stream last, float64, no CPU fallback).  The symbol is
 * declared here, apart from nnk_b200.h, because every symbol of nnk_b200.h has a case in the buffers-and-
 * streams catalogue of the core library; tests/test_gmm_traj_em_gpu.py runs the same checks on this one.
 *
 * The model (Toda, Black & Tokuda 2007, Sec. III, with the diagonal Eq. 23 variances of baseline.gmm.MLPG):
 * source frames x_t (D = nw * static_dim columns), static trajectory c (static_dim columns) and its
 * static + dynamic sequence Y_t[w * static_dim + s] = sum_{k = -l_w}^{u_w} coef[w][l_w + k] c_{t+k}[s], where
 * frames outside the utterance of t are zero.  Per mixture m:
 *   E_{m,t} = nu_m + A_m (x_t - mu_m)                    (gmm->tgt_means, gmm->A_t, gmm->src_means; Eq. 22)
 *   lw_{t,m} = lp[t][m] + log_norm[m][e_t] - 1/2 sum_{d in K_t} (Y_t - E_{m,t})_d^2 inv_Dm[m][d]
 * with lp from nnk_gmm_logprob and inv_Dm = 1 / D_m.  Like nnk_mlpg_fwd, which gives the dynamic windows zero
 * precision on the first and last H frames of an utterance (H = max_w max(l_w, u_w)), the columns K_t of frame t
 * are all D columns (e_t = 0) except on those edge frames, where they are the static_dim columns of window 0
 * (e_t = 1); log_norm[m][e] = -1/2 (sum_{d in K} log D_m,d + |K| log 2 pi) over the same columns.
 *
 * nnk_gmm_traj_em, one CTA per tile of NNK_GMM_TRAJ_TILE frames of one utterance:
 *   mode NNK_GMM_TRAJ_EM (E-step): gamma_{t,m} = softmax_m lw_{t,m};
 *     V[t][d] = 1 / P_t,d with P_t,d = sum_m gamma_{t,m} inv_Dm[m][d];
 *     E_bar[t][d] = (sum_m gamma_{t,m} E_{m,t,d} inv_Dm[m][d]) / P_t,d;
 *     both (T, D) row-major, the layout nnk_mlpg_fwd reads as means / variances.
 *   mode NNK_GMM_TRAJ_OBJECTIVE: E_bar and V are not touched (may be NULL).
 *   Both modes: ll_part[tile] = sum over the tile's frames, in frame order, of log sum_m exp lw_{t,m}
 *     (ll_part may be NULL in mode EM).  Utterance u owns the tiles tile_off[u] .. tile_off[u+1] - 1, in frame
 *     order; the per-utterance objective is their sum.
 * Tables (device int32, n_utt + 1 entries each): utterance u is frames utt_off[u] .. utt_off[u+1] - 1 with
 * utt_off[0] = 0, utt_off[n_utt] = T; tile_off[0] = 0, tile_off[u+1] - tile_off[u] =
 * ceil(len_u / NNK_GMM_TRAJ_TILE), tile_off[n_utt] = n_tiles.
 * Errors: NNK_ERR_ARG for NULL pointers, bad sizes or strides, D != win.nw * static_dim, a bad window set or
 * mode; NNK_ERR_UNSUPPORTED for D > 96 or more than 65535 mixtures; all before anything touches the device. */
#ifndef NNK_GMM_TRAJ_H
#define NNK_GMM_TRAJ_H

#include <stdint.h>

#include "nnk_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define NNK_GMM_TRAJ_EM 0
#define NNK_GMM_TRAJ_OBJECTIVE 1
#define NNK_GMM_TRAJ_TILE 32

typedef struct nnk_gmm_traj_args {
  const double* x;            /* device (T, x_ld) source frames, D = gmm->D columns                         */
  int64_t x_ld;
  const double* lp;           /* device (T, M) from nnk_gmm_logprob                                         */
  const double* c;            /* device (T, c_ld) current static trajectory, static_dim columns              */
  int64_t c_ld;
  int32_t T;
  int32_t n_utt;
  const int32_t* utt_off;     /* device (n_utt + 1)                                                         */
  const int32_t* tile_off;    /* device (n_utt + 1)                                                         */
  int32_t n_tiles;
  int32_t static_dim;
  nnk_windows_t win;
  int32_t mode;               /* NNK_GMM_TRAJ_EM / NNK_GMM_TRAJ_OBJECTIVE                                    */
  const double* inv_Dm;       /* device (M, D) 1 / D_m                                                      */
  const double* log_norm;     /* device (M, 2): all columns, static columns only                            */
  double* E_bar;              /* device (T, D), mode EM                                                     */
  double* V;                  /* device (T, D), mode EM                                                     */
  double* ll_part;            /* device (n_tiles), or NULL in mode EM                                       */
} nnk_gmm_traj_args_t;

int nnk_gmm_traj_em(const nnk_gmm_t* gmm, const nnk_gmm_traj_args_t* args, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NNK_GMM_TRAJ_H */
