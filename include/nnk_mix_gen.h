/* nnk_mix_gen.h -- C ABI of parameter generation from mixture outputs in libnnk_b200.so (sm_90a).
 *
 * Same conventions as nnk_b200.h (return codes, dtype codes, windows, stream last, no CPU fallback).  The symbol
 * is declared here, apart from nnk_b200.h, because every symbol of nnk_b200.h has a case in the buffers-and-
 * streams catalogue of the core library; tests/test_mix_gen_gpu.py runs the same checks (poisoned allocations, a
 * side stream) on it.
 *
 * nnk_mix_gen: one launch of mix_gen_kernel (csrc/nnk_mix_gen.cu), the E-step side of the EM of
 * paramgen.mlpg_mixture_batch (DESIGN.md 3.19; Tokuda et al., ICASSP 2000).  Frame r (a row of the batch) has M
 * components: log-weights lw[r, m] (log_weights, (n_rows, M)), means mu[r, m, i] and variances s2[r, m, i]
 * (means / vars, (n_rows, M, D)), all of `dtype` and row-major; float32 inputs are widened in registers and every
 * operation is float64.  Utterance u has rows utt_off[u] .. utt_off[u] + utt_len[u] - 1 and the tiles
 * tile_off[u] .. tile_off[u + 1] - 1 of NNK_MIX_GEN_TILE frames (n_tiles = tile_off[n_utt]); rows outside every
 * utterance are never read or written.  col_map[i] describes input column i:
 *   -1                        the column takes no part (no chain reads it);
 *   (out_col << 3) | 0        a copied column: Y_t[i] = c[t, out_col];
 *   (out_col << 3) | (w + 1)  window w of a smoothed column: Y_t[i] = sum_j coef_w[j] c[t + j, out_col], with
 *                             c = 0 outside the utterance.
 * On the first and last H = max_w max(l_w, u_w) frames of an utterance, and on every frame when H = 0, only the
 * copied columns and those of window 0 count; elsewhere every column with col_map >= 0 counts.
 *   NNK_MIX_GEN_SELECT:    per frame the component a with the largest lw (the lowest index on ties) goes to
 *                          E[r, :] = mu[r, a, :], V[r, :] = s2[r, a, :]; every component's log-normaliser
 *                          lnorm[r, m] = lw[r, m] - 1/2 sum_{counted i} (log s2[r, m, i] + log 2 pi) goes to
 *                          lnorm.  Data errors set *status_word (below).
 *   NNK_MIX_GEN_ESTEP:     with l[r, m] = lnorm[r, m] - 1/2 sum_{counted i} (Y_r[i] - mu[r, m, i])^2 / s2[r, m, i]
 *                          and gamma its softmax over m: P = sum_m gamma / s2, E[r, i] = (sum_m gamma mu / s2) / P
 *                          and V[r, i] = 1 / P for every column with col_map >= 0 (0 and 1 for the others).
 *                          With ll_part, ll_part[tile] = sum over the tile's frames, in frame order, of
 *                          log sum_m exp(l[r, m]).
 *   NNK_MIX_GEN_OBJECTIVE: ll_part only (required).
 * c (rows of c_ld doubles, the first c_cols staged per tile) is read by ESTEP and OBJECTIVE only.
 * Status word (device, zeroed by the caller): 0, or ~((row << 2) | kind) of the first failing row, lowest kind
 * first: kind 1 = a NaN or +inf log-weight, 2 = every log-weight -inf, 3 = a variance of a column with
 * col_map >= 0 that is not positive and finite.  Results of a failing call are undefined but never fault.
 * Errors: NNK_ERR_ARG for NULL pointers, bad sizes, a bad mode, dtype or window set; NNK_ERR_UNSUPPORTED for
 * D > NNK_MIX_GEN_MAX_D or M > NNK_MIX_GEN_MAX_M; all before anything touches the device.  Every output element
 * is written by one thread in a fixed order: repeated calls give the same bits. */
#ifndef NNK_MIX_GEN_H
#define NNK_MIX_GEN_H

#include <stddef.h>
#include <stdint.h>

#include "nnk_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define NNK_MIX_GEN_SELECT 0
#define NNK_MIX_GEN_ESTEP 1
#define NNK_MIX_GEN_OBJECTIVE 2
#define NNK_MIX_GEN_TILE 32    /* frames per tile */
#define NNK_MIX_GEN_MAX_D 256  /* input columns   */
#define NNK_MIX_GEN_MAX_M 64   /* components      */

typedef struct nnk_mix_gen_args {
  const void* log_weights; /* device (n_rows, M) of dtype                                                   */
  const void* means;       /* device (n_rows, M, D) of dtype                                                */
  const void* vars;        /* device (n_rows, M, D) of dtype                                                */
  int32_t dtype;           /* NNK_F32 / NNK_F64                                                             */
  int32_t M;               /* components, 1 .. NNK_MIX_GEN_MAX_M                                            */
  int32_t D;               /* input columns, 1 .. NNK_MIX_GEN_MAX_D                                         */
  int32_t n_utt;           /* >= 1                                                                          */
  const int32_t* utt_off;  /* device (n_utt): first row of each utterance                                   */
  const int32_t* utt_len;  /* device (n_utt): frames of each utterance                                      */
  const int32_t* tile_off; /* device (n_utt + 1): first tile of each utterance                              */
  int32_t n_tiles;         /* tile_off[n_utt]                                                               */
  const int32_t* col_map;  /* device (D)                                                                    */
  nnk_windows_t win;
  int32_t mode;            /* NNK_MIX_GEN_SELECT / _ESTEP / _OBJECTIVE                                      */
  const double* c;         /* device, ESTEP / OBJECTIVE: current trajectories, row r at c + r * c_ld        */
  int64_t c_ld;
  int32_t c_cols;          /* columns of c the column map addresses (out_col < c_cols <= c_ld)             */
  double* lnorm;           /* device (n_rows, M): written by SELECT, read by ESTEP / OBJECTIVE              */
  double* E;               /* device (n_rows, D): written by SELECT / ESTEP                                 */
  double* V;               /* device (n_rows, D): written by SELECT / ESTEP                                 */
  double* ll_part;         /* device (n_tiles) or NULL (ESTEP); required for OBJECTIVE                      */
  uint64_t* status_word;   /* device, SELECT                                                                */
} nnk_mix_gen_args_t;

int nnk_mix_gen(const nnk_mix_gen_args_t* args, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NNK_MIX_GEN_H */
