/* nnk_ms_segment.h -- C ABI of the segment-level modulation-spectrum kernels in libnnk_b200.so (sm_90a).
 *
 * Same conventions as nnk_b200.h (return codes, dtype codes, stream last, no CPU fallback).  The symbol is
 * declared here, apart from nnk_b200.h, because every symbol of nnk_b200.h has a case in the buffers-and-
 * streams catalogue of the core library; tests/test_ms_segment_gpu.py runs the same checks (poisoned
 * allocations, NaN padding, a side stream) on this one.
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
 * written exactly once, without atomics: repeated calls give the same bits. */
#ifndef NNK_MS_SEGMENT_H
#define NNK_MS_SEGMENT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NNK_MSSEG_LOGPOWER 0
#define NNK_MSSEG_POSTFILTER 1

int nnk_ms_segment(int32_t mode, int32_t dtype, int32_t n, int32_t L, const void* x, const void* table, void* out,
                   int32_t B, int32_t T, int32_t D, const int32_t* lengths, const int64_t* seg_off, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NNK_MS_SEGMENT_H */
