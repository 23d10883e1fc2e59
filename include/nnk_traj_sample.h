/* nnk_traj_sample.h -- C ABI of sampling from the trajectory model in libnnk_b200.so (sm_90a).
 *
 * Same conventions as nnk_b200.h (return codes, dtype codes, windows, stream last, no CPU fallback).  The symbols
 * are declared here, apart from nnk_b200.h, because every symbol of nnk_b200.h has a case in the buffers-and-
 * streams catalogue of the core library; tests/test_traj_sample_gpu.py runs the same checks (poisoned
 * allocations, a side stream) on them.
 *
 * nnk_mlpg_traj_sample: one launch of mlpg_kernel in MODE_SAMPLE (csrc/nnk_mlpg.cu, DESIGN.md 3.21) per workspace
 * wave.  Per chain c of utterance u (a static column, exactly as nnk_mlpg_fwd sees it: T frames, tau_{t,w} =
 * 1 / var with the edge rule of nnk_mlpg_fwd, P = sum_w W_w^T diag(tau_w) W_w, b = sum_w W_w^T (tau_w mu_w),
 * and the top-down factorisation P = L D L^T with unit lower L, pivots d_t, multipliers l_j[t] = L[t+j][t] and
 * zs_t = (L^-1 b)_t / d_t), sample s = 0 .. n_samples - 1 is
 *
 *   y_t = zs_t + scale * z_{s,t} / sqrt(d_t) - sum_{j=1..S} l_j[t] y_{t+j}      (t = T-1 .. 0, y_t = 0 for t >= T)
 *
 * that is y = L^-T (D^-1 L^-1 b + scale D^-1/2 z) ~ N(cbar, scale^2 P^-1), cbar = P^-1 b, for z ~ N(0, I).  It is
 * written in the dtype of the inputs to args->out + s * sample_stride at row (out_off or utt_off)[u] + t, column
 * chains[c].out_col, row stride out_ld.  With scale = 0 the recurrence is nnk_mlpg_fwd's backward sweep term for
 * term.  Copied chains (flags & 1) get the means column, unchanged and without noise, in every sample.  Elements
 * no chain writes are not touched.  Arithmetic is float64; float32 inputs are widened exactly as nnk_mlpg_fwd
 * widens them.
 *
 * The noise z_{s,t} of chain c of utterance u is a pure function of (seed, key_u, s, t, out_col = chains[c].out_col):
 * it does not depend on the batch around the utterance, the layout, the padding, the dtype, n_samples or the
 * workspace waves.  Normative definition:
 *
 *   Philox4x32-10 (Salmon, Moraes, Dror & Shaw, SC 2011) with multipliers M0 = 0xD2511F53, M1 = 0xCD9E8D57 and key
 *   increments W0 = 0x9E3779B9, W1 = 0xBB67AE85.  A round maps the counter (c0, c1, c2, c3) to
 *     (hi(M1 * c2) ^ c1 ^ k0, lo(M1 * c2), hi(M0 * c0) ^ c3 ^ k1, lo(M0 * c0))
 *   (hi / lo: upper / lower 32 bits of the 64-bit product); after each of the first nine rounds the key becomes
 *   (k0 + W0, k1 + W1) mod 2^32.  Ten rounds give the output words (r0, r1, r2, r3).
 *     key      (k0, k1)         = (seed mod 2^32, seed >> 32)
 *     counter  (c0, c1, c2, c3) = (t >> 1, out_col, s, key_u),   key_u = keys ? keys[u] : u
 *   u is the caller's utterance index (the index into utt_off), never a position in args->order.
 *     N_U = (r0 >> 6) * 2^26 + (r1 >> 6),   U = (N_U + 0.5) * 2^-52   in (0, 1)
 *     N_V = (r2 >> 6) * 2^26 + (r3 >> 6),   V = N_V * 2^-52           in [0, 1)
 *     R = sqrt(-2 log U),   z_{s,t} = R cos(2 pi V) for even t,  R sin(2 pi V) for odd t   (Box & Muller 1958)
 *   so one Philox call serves frames 2k and 2k + 1 of one chain and sample.  Known answers of the rounds
 *   (Random123's philox4x32-10 vectors): counter 0, key 0 -> 6627e8d5 e169c58d bc57ac4c 9b00dbd8; all ones ->
 *   408f276d 41c83b0e a20bc7c6 6d5451fd; counter 243f6a88 85a308d3 13198a2e 03707344, key a4093822 299f31d0 ->
 *   d16cfe09 94fdcceb 5001e420 24126ea1.
 *
 * A pivot d_t <= 0 sets the status word as nnk_mlpg_fwd does.  Errors: NNK_ERR_ARG for NULL pointers, bad sizes,
 * n_samples < 1, sample_stride < 0 or a scale that is negative or not finite; NNK_ERR_UNSUPPORTED for a window set
 * no instance serves; NNK_ERR_WORKSPACE for a workspace below one utterance's share of
 * nnk_mlpg_traj_sample_workspace_bytes; all before anything is launched.  args->grad_out, go_ld and go_f64 are
 * not used. */
#ifndef NNK_TRAJ_SAMPLE_H
#define NNK_TRAJ_SAMPLE_H

#include <stddef.h>
#include <stdint.h>

#include "nnk_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nnk_traj_sample {
  int64_t sample_stride; /* elements between samples in args->out                                        */
  int32_t n_samples;     /* >= 1                                                                           */
  uint64_t seed;
  const uint32_t* keys;  /* device (n_utt,), or NULL for key_u = u                                         */
  double scale;          /* >= 0, finite                                                                   */
} nnk_traj_sample_t;

int nnk_mlpg_traj_sample(const nnk_mlpg_args_t* args, const nnk_traj_sample_t* ts, void* stream);
size_t nnk_mlpg_traj_sample_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, const nnk_windows_t* win);

#ifdef __cplusplus
}
#endif
#endif /* NNK_TRAJ_SAMPLE_H */
