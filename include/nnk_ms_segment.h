/* nnk_ms_segment.h -- C ABI of the segment-level modulation-spectrum kernels in libnnk_b200.so (sm_90a).
 *
 * Same conventions as nnk_b200.h (return codes, dtype codes, stream last, no CPU fallback).  The symbols are
 * declared here, apart from nnk_b200.h, because every symbol of nnk_b200.h has a case in the buffers-and-
 * streams catalogue of the core library; tests/test_ms_segment_gpu.py and tests/test_ms_gen_segment_gpu.py run
 * the same checks (poisoned allocations, NaN padding, a side stream) on these.
 *
 * nnk_ms_segment: the segment-level MS of Takamichi et al. (ICASSP 2014) over a padded batch x (B, T, D),
 * row-major, in dtype (NNK_F32 / NNK_F64).  Utterance b has len_b = min(max(lengths[b], 0), T) frames
 * (lengths NULL: T); later frames are never read.  With the hop H = L / 2 and the periodic Hann window
 * w_m = 0.5 - 0.5 cos(2 pi m / L), utterance b has J_b = ceil(len_b / H) + 1 segments (0 when len_b = 0);
 * segment j starts at frame (j - 1) H, frames outside [0, len_b) are 0, and Y_j = rfft(w * x[seg j], n),
 * K = n / 2 + 1 bins, s_jk = log(max(|Y_jk|^2, tiny)).
 *   mode 0 (log power):   out (S, D, K) in dtype, S = sum_b J_b: row seg_off[b] + j, column d, bin k holds
 *                         s_jk of column d.  seg_off (B,) int64 on the device, the exclusive prefix sums of J_b
 *                         computed from the same lengths; table is unused (may be NULL).
 *   mode 1 (post-filter): table (K, D, 2) in dtype holds (a, c); every bin k >= 1 of non-zero power becomes
 *                         C_jk = Y_jk / |Y_jk| exp((a s_jk + c) / 2), bin 0 and zero-power bins as for
 *                         nnk_modspec's post-filter; out (B, T, D) = sum_j irfft(C_j, n)[t - (j - 1) H] over
 *                         the segments with 0 <= t - (j - 1) H < L for t < len_b, 0 for len_b <= t < T.
 *                         seg_off is unused (may be NULL).
 * n is 32, 64, 128, 256 or 512 and L even with 4 <= L <= n (else NNK_ERR_ARG).  Every output element is
 * written exactly once, without atomics: repeated calls give the same bits.
 *
 * nnk_mlpg_ms_segment: parameter generation considering the segment-level MS (paramgen.mlpg_ms_batch(segment=L),
 * DESIGN.md 3.18).  args, ms, tau, P, b, c_m = P^-1 b, omega, the start point c0 = c_m and the trials are exactly
 * those of nnk_mlpg_ms (include/nnk_ms_gen.h); only the MS term differs.  Per chain (one smoothed output column
 * s = c.out_col of one utterance of T >= 1 frames, any T), with the segments of nnk_ms_segment (H = L / 2,
 * J = ceil(T / H) + 1, segment j starts at frame (j - 1) H, frames outside [0, T) are 0, periodic Hann window w),
 * Y_j = rfft(w * c[seg j], n) and s_jk = log(max(|Y_jk|^2, DBL_MIN)), it maximises
 *   F(c) = omega (b^T c - c^T P c / 2) - 1/(2 J) sum_j sum_{k=1}^{n/2} q_k (s_jk - nu_k)^2
 * (nu_k, q_k from ms->ms_mean / ms->ms_var as for nnk_mlpg_ms): the mean of the utterance level's term over the J
 * segments, edge segments included.  Bin 0 has no term; a bin of power <= DBL_MIN adds a constant and no
 * gradient; ms_var = inf exempts a bin.  The gradient at frame t = (j - 1) H + m (0 <= m < L) is
 *   g_t = 1/J sum_{j containing t} w_m [n irfft(C_j, n)]_m,  C_jk = -q_k (s_jk - nu_k) / |Y_jk|^2 Y_jk
 * (C_j,n/2 doubled, C_j0 = 0): every frame lies in two segments, so g_t is one addition of two terms.
 * ms->n is 32, 64, 128, 256 or 512 and L even with 4 <= L <= n; there is no limit on args->max_T.  NNK_ERR_ARG:
 * args or ms NULL, dtype not NNK_F64, out_off not NULL, a negative size, a bad n or L, n_iter < 0, step <= 0,
 * weight < 0 or NaN, a NULL device pointer or NULL ms_mean / ms_var.  The workspace is
 * nnk_mlpg_ms_workspace_bytes() of the same arguments.  One call enqueues 2 + 2 n_iter launches on `stream`
 * without a host synchronisation, whatever the batch and T: nnk_mlpg_fwd, one launch that copies c_m to out and
 * forms the first gradient, then per trial one nnk_mlpg_solve and one launch of ms_gen_segment_kernel
 * (csrc/nnk_ms_gen.cu).  Non-positive pivots set the status word as for nnk_mlpg_ms.  Sums run in a fixed order
 * inside one CTA per chain, so a chain's bits do not depend on the batch and repeated calls give the same bits. */
#ifndef NNK_MS_SEGMENT_H
#define NNK_MS_SEGMENT_H

#include <stdint.h>

#include "nnk_ms_gen.h"

#ifdef __cplusplus
extern "C" {
#endif

#define NNK_MSSEG_LOGPOWER 0
#define NNK_MSSEG_POSTFILTER 1

int nnk_ms_segment(int32_t mode, int32_t dtype, int32_t n, int32_t L, const void* x, const void* table, void* out,
                   int32_t B, int32_t T, int32_t D, const int32_t* lengths, const int64_t* seg_off, void* stream);
int nnk_mlpg_ms_segment(const nnk_mlpg_args_t* args, const nnk_mlpg_ms_t* ms, int32_t L, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NNK_MS_SEGMENT_H */
