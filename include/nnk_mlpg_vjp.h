/* nnk_mlpg_vjp.h -- C ABI of the gradient of MLPG in its means and variances in libnnk_b200.so (sm_90a).
 *
 * Same conventions as nnk_b200.h (return codes, dtype codes, windows, stream last, no CPU fallback).  The symbols
 * are declared here, apart from nnk_b200.h, because every symbol of nnk_b200.h has a case in the buffers-and-
 * streams catalogue of the core library; tests/test_mlpg_vjp_gpu.py runs the same checks (poisoned allocations, a
 * side stream) on them.
 *
 * nnk_mlpg_vjp: one launch of mlpg_kernel in MODE_VJP (csrc/nnk_mlpg.cu, DESIGN.md 3.22) per workspace wave.  Per
 * chain c of utterance u (a static column, exactly as nnk_mlpg_fwd sees it: T frames, tau_{t,w} = 1 / var with the
 * edge rule of nnk_mlpg_fwd, mu_{t,w}, P = sum_w W_w^T diag(tau_w) W_w, b = sum_w W_w^T (tau_w mu_w),
 * cbar = P^-1 b, the trajectory nnk_mlpg_fwd writes) and the gradient o = dL/dcbar of a loss L with respect to that
 * trajectory (o_t at grad_out[((out_off or utt_off)[u] + t) * go_ld + chains[c].out_col], of `dtype`), with
 * g = P^-1 o:
 *
 *   dL/dmu_{t,w}  = tau_{t,w} (W_w g)_t                                                      -> grad_means
 *   dL/dvar_{t,w} = -tau_{t,w}^2 (W_w g)_t (mu_{t,w} - (W_w cbar)_t)                          -> grad_vars
 *
 * (Wu & Wang 2006: minimum generation error training through MLPG in both).  Where the edge rule sets tau to zero,
 * both gradients are 0.  Copied chains (flags & 1) pass o through: dL/dmu = o, and their dL/dvar is not written.
 * grad_means has the rows of means (utt_off[u] + t) and columns chains[c].in_col + w * win_stride with row stride
 * gm_ld, of `dtype`.  Per-frame variances (var_ld > 0): grad_vars has the layout of grad_means with row stride
 * gv_ld, of `dtype`.  Global (D,) variances (var_ld == 0): grad_vars is a float64 (n_utt, gv_ld) array and
 * grad_vars[u * gv_ld + column] is the sum of the per-frame values over the utterance's frames.  Only the elements
 * of chains at frames 0 .. T - 1 are written: the caller zeroes the others.  Every sum runs in a fixed order in one
 * thread, so a chain's results do not depend on the batch and repeated calls give the same bits.  Arithmetic is
 * float64; float32 inputs are widened exactly as nnk_mlpg_fwd widens them, and the results are stored in `dtype`.
 * Means and grad_out are not checked: non-finite values give NaN.  A pivot d_t <= 0 sets the status word as
 * nnk_mlpg_fwd does.  Errors: NNK_ERR_ARG for NULL pointers or bad sizes, NNK_ERR_UNSUPPORTED for a window set no
 * instance serves, NNK_ERR_WORKSPACE for a workspace below one utterance's share of nnk_mlpg_vjp_workspace_bytes;
 * all before anything is launched.  args->out, args->grad_out, args->go_ld, args->out_ld and args->go_f64 are not
 * used. */
#ifndef NNK_MLPG_VJP_H
#define NNK_MLPG_VJP_H

#include <stddef.h>
#include <stdint.h>

#include "nnk_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nnk_mlpg_vjp {
  const void* grad_out; /* device, dtype: dL/dcbar (rows and columns of the nnk_mlpg_fwd output)                  */
  int64_t go_ld;        /* row stride of grad_out, in elements                                                     */
  void* grad_means;     /* device, dtype, rows and columns of means                                                */
  int64_t gm_ld;
  void* grad_vars;      /* device: per-frame, dtype, rows and columns of vars; global, float64 (n_utt, gv_ld)      */
  int64_t gv_ld;
} nnk_mlpg_vjp_t;

int nnk_mlpg_vjp(const nnk_mlpg_args_t* args, const nnk_mlpg_vjp_t* vj, void* stream);
size_t nnk_mlpg_vjp_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, const nnk_windows_t* win);

#ifdef __cplusplus
}
#endif
#endif /* NNK_MLPG_VJP_H */
