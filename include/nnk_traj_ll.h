/* nnk_traj_ll.h -- C ABI of the trajectory-model log-likelihood in libnnk_b200.so (sm_90a).
 *
 * Same conventions as nnk_b200.h (return codes, dtype codes, windows, stream last, no CPU fallback).  The symbols
 * are declared here, apart from nnk_b200.h, because every symbol of nnk_b200.h has a case in the buffers-and-
 * streams catalogue of the core library; tests/test_traj_ll_gpu.py runs the same checks (poisoned allocations, a
 * side stream) on them.
 *
 * nnk_mlpg_traj_ll: one launch of mlpg_kernel in MODE_TLL / MODE_TLL_GRAD (csrc/nnk_mlpg.cu, DESIGN.md 3.20) per
 * workspace wave.  Per chain c of utterance u (a static column, exactly as nnk_mlpg_fwd sees it: T frames,
 * tau_{t,w} = 1 / var with the edge rule of nnk_mlpg_fwd, mu_{t,w}, P = sum_w W_w^T diag(tau_w) W_w,
 * b = sum_w W_w^T (tau_w mu_w), cbar = P^-1 b, P = L D L^T with pivots d_t) and its target static trajectory x
 * (x_t at targets[(out_off or utt_off)[u] + t) * tgt_ld + chains[c].out_col]), the Gaussian trajectory model
 * N(x; cbar, P^-1) (Zen, Tokuda & Kitamura 2007) has the log-likelihood
 *
 *   l = 1/2 sum_t log d_t - 1/2 sum_{t,w} tau_{t,w} (u_{t,w} - ubar_{t,w})^2 - (T/2) log 2 pi,
 *   u_{t,w} = (W_w x)_t,  ubar_{t,w} = (W_w cbar)_t,
 *
 * written to ll[u * n_chain + c] (0 for copied chains, flags & 1).  With grad != 0 the gradients are written too,
 * with w_t row t of W_w and Sigma = P^-1:
 *
 *   dl/dmu_{t,w}   = tau_{t,w} (u_{t,w} - ubar_{t,w})                                         -> grad_means
 *   dl/dvar_{t,w}  = -tau_{t,w}^2 / 2 [w_t^T Sigma w_t - (u_{t,w} - mu_{t,w})^2 + (ubar_{t,w} - mu_{t,w})^2]
 *   dl/dx          = -P (x - cbar) = -sum_w W_w^T (dl/dmu_{.,w})                               -> grad_targets
 *
 * grad_means has the rows of means (utt_off[u] + t) and columns chains[c].in_col + w * win_stride with row stride
 * gm_ld; grad_targets has the rows and columns of the targets with row stride gx_ld; both are of `dtype`.  Per-frame
 * variances (var_ld > 0): grad_vars has the layout of grad_means with row stride gv_ld, of `dtype`.  Global (D,)
 * variances (var_ld == 0): grad_vars is a float64 (n_utt, gv_ld) array and grad_vars[u * gv_ld + column] is the
 * sum of the per-frame values over the utterance's frames.  Only the elements of solved chains at frames
 * 0 .. T - 1 are written: the caller zeroes the others.  Where the edge rule sets tau to zero, both gradients are 0.
 * Every sum runs in a fixed order in one thread, so a chain's results do not depend on the batch and repeated calls
 * give the same bits.  Arithmetic is float64; float32 inputs are widened exactly as nnk_mlpg_fwd widens them.
 * Targets and means are not checked: non-finite values give NaN.  A pivot d_t <= 0 sets the status word as
 * nnk_mlpg_fwd does.  Errors: NNK_ERR_ARG for NULL pointers or bad sizes, NNK_ERR_UNSUPPORTED for a window set no
 * instance serves, NNK_ERR_WORKSPACE for a workspace below one utterance's share of
 * nnk_mlpg_traj_ll_workspace_bytes; all before anything is launched.  args->out, grad_out, go_ld and go_f64 are
 * not used. */
#ifndef NNK_TRAJ_LL_H
#define NNK_TRAJ_LL_H

#include <stddef.h>
#include <stdint.h>

#include "nnk_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nnk_traj_ll {
  const void* targets; /* device, dtype: target static trajectories (rows and columns of the nnk_mlpg_fwd output) */
  int64_t tgt_ld;      /* row stride of targets, in elements                                                      */
  double* ll;          /* device (n_utt, n_chain) float64                                                         */
  int32_t grad;        /* 0: ll only; 1: ll and the three gradients                                               */
  void* grad_means;    /* device, dtype, rows and columns of means                                                */
  int64_t gm_ld;
  void* grad_vars;     /* device: per-frame, dtype, rows and columns of vars; global, float64 (n_utt, gv_ld)      */
  int64_t gv_ld;
  void* grad_targets;  /* device, dtype, rows and columns of targets                                              */
  int64_t gx_ld;
} nnk_traj_ll_t;

int nnk_mlpg_traj_ll(const nnk_mlpg_args_t* args, const nnk_traj_ll_t* tl, void* stream);
size_t nnk_mlpg_traj_ll_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, const nnk_windows_t* win);

#ifdef __cplusplus
}
#endif
#endif /* NNK_TRAJ_LL_H */
