/* nnk_ms_gen.h -- C ABI of parameter generation considering the modulation spectrum in libnnk_b200.so (sm_90a).
 *
 * Same conventions as nnk_b200.h (return codes, dtype codes, status word, stream last, no CPU fallback), whose
 * nnk_mlpg_args_t it takes.  The symbols are declared here, apart from nnk_b200.h, because every symbol of
 * nnk_b200.h has a case in the buffers-and-streams catalogue of the core library; tests/test_ms_gen_gpu.py runs
 * the same checks (poisoned allocations, a side stream) on these.
 *
 * nnk_mlpg_ms: per chain c (one smoothed output column s = c.out_col of one utterance of T <= n frames) and with
 * tau, P, b and c_m = P^-1 b exactly as nnk_mlpg_fwd builds them (edge rule included), Y = rfft(c, n) and
 * s_k(c) = log(max(|Y_k|^2, DBL_MIN)), maximises
 *   F(c) = omega (b^T c - c^T P c / 2) - 1/2 sum_{k=1}^{n/2} q_k (s_k(c) - nu_k)^2,
 *   nu_k = ms_mean[k * args->out_ld + s],  q_k = 1 / ms_var[k * args->out_ld + s]  (q_k = 0 when ms_var is inf)
 * from c0 = c_m by n_iter trials: g = grad of the MS term at c, h = P^-1 g, delta = (c_m - c) + h / omega,
 * c' = c + alpha delta is kept when F(c') >= F(c), otherwise alpha halves (alpha starts at `step`; a rejected
 * trial still counts).  Bin 0 has no term; a bin of power <= DBL_MIN adds a constant and no gradient.
 * omega = weight, or 1 / (nw T) when weight == 0.  Pass-through chains are copied.
 *
 * Everything is float64: args->dtype must be NNK_F64 (callers widen float32 inputs once) and args->out_off
 * NULL.  Every utterance must have T <= n frames (args->max_T <= n); longer ones are left unwritten.  One call
 * enqueues, on `stream` and without a host synchronisation, 2 + 2 n_iter launches: nnk_mlpg_fwd into the
 * workspace, one launch that copies c_m to out and forms the first gradient, then per trial one nnk_mlpg_solve
 * (float64 right-hand side) and one launch of ms_gen_kernel (csrc/nnk_ms_gen.cu).  Non-positive pivots set the
 * status word as for nnk_mlpg_fwd.  The workspace must hold nnk_mlpg_ms_workspace_bytes(): the MLPG factor
 * scratch of the whole batch, c_m and h ((n_rows, out_ld) each), g ((n_rows, n_chain)) and two numbers per
 * chain (F and alpha).  Per-chain sums run in a fixed order inside one CTA, so a chain's result does not depend
 * on the batch around it and repeated calls give the same bits. */
#ifndef NNK_MS_GEN_H
#define NNK_MS_GEN_H

#include <stddef.h>
#include <stdint.h>

#include "nnk_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nnk_mlpg_ms {
  const double* ms_mean; /* device (n / 2 + 1, args->out_ld): nu, finite where ms_var is finite          */
  const double* ms_var;  /* device (n / 2 + 1, args->out_ld): > 0, inf exempts the bin                    */
  int32_t n;             /* DFT length: 256, 512, 1024, 2048 or 4096                                      */
  int32_t n_iter;        /* >= 0 trials                                                                   */
  double step;           /* > 0 initial step alpha                                                        */
  double weight;         /* omega > 0, or 0 => 1 / (nw T) per utterance                                   */
  int64_t n_rows;        /* rows of means / vars / out (utt_off[n_utt] at most); sizes the workspace      */
} nnk_mlpg_ms_t;

int nnk_mlpg_ms(const nnk_mlpg_args_t* args, const nnk_mlpg_ms_t* ms, void* stream);
size_t nnk_mlpg_ms_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, int64_t n_rows, int64_t out_ld,
                                   const nnk_windows_t* win);

#ifdef __cplusplus
}
#endif
#endif /* NNK_MS_GEN_H */
