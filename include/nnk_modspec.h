/* nnk_modspec.h -- C ABI of the modulation-spectrum kernels in libnnk_b200.so (sm_90a).
 *
 * Same conventions as nnk_b200.h (return codes, dtype codes, stream last, no CPU fallback).  The symbol is
 * declared here, apart from nnk_b200.h, because every symbol of nnk_b200.h has a case in the buffers-and-
 * streams catalogue of the core library; tests/test_modspec_gpu.py runs the same checks (poisoned
 * allocations, NaN padding, a delayed side stream) on this one.
 *
 * nnk_modspec: one CTA per (utterance b, feature column d).  The column's first len_b frames (lengths[b], or
 * T_in when lengths is NULL; later frames are never read) are zero-padded to n and transformed with an n-point
 * real FFT in shared memory (n / 2-point complex FFT and split); Y = fwd_scale * X is the spectrum in the
 * norm's scaling.  K = n / 2 + 1 bins; all arrays are row-major (B, rows, D).
 *   mode 0 (power):   out  = |Y_k|^2, (B, K, D); out2 = Y_k / |Y_k| as interleaved (re, im), (B, K, D, 2),
 *                     or NULL.  A zero bin has phase (+1, 0), or (-1, 0) when its real part is -0.
 *   mode 1 (smooth):  bins k >= limit_bin become Y_k / |Y_k| (log_domain) or 0, then
 *                     out = inv_scale * irfft_unnormalised(Y)[:len_b], (B, T_out, D).
 *   mode 2 (inverse): in = |Y|^2 (B, K, D), in2 = phase (B, K, D, 2); Y = sqrt(in) * in2;
 *                     out = inv_scale * irfft_unnormalised(Y)[:len_b], (B, T_out, D).  The imaginary parts of
 *                     bins 0 and n / 2 are ignored, as numpy.fft.irfft does.
 *   mode 3 (grad):    in2 = dL/d|Y|^2 (B, K, D); out = dL/dx = 2 fwd_scale Re(sum_k G_k conj(Y_k) e^{-2 pi i k t / n})
 *                     for t < len_b, (B, T_out, D).
 *   mode 4 (log power): out = log(max(|Y_k|^2, tiny)), (B, K, D), tiny the smallest normal number of the dtype
 *                     (FLT_MIN, DBL_MIN); out2 must be NULL.  No inverse FFT, like mode 0.
 *   mode 5 (post-filter): in2 = (a, c) interleaved, (K, D, 2), shared by every utterance.  Bin 0 is kept; a bin
 *                     k >= 1 of zero power stays 0, any other becomes Y_k / |Y_k| exp(s' / 2) with
 *                     s' = a s + c, s = log(max(|Y_k|^2, tiny)); then, as mode 1,
 *                     out = inv_scale * irfft_unnormalised(Y)[:len_b], (B, T_out, D).  out2 must be NULL.
 * Frames len_b <= t < T_out of out are written as 0.  n is 256, 512, 1024, 2048 or 4096 (else NNK_ERR_ARG);
 * every len_b must be <= n and <= T_out (<= T_in for the modes that read x). */
#ifndef NNK_MODSPEC_H
#define NNK_MODSPEC_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NNK_MS_POWER 0
#define NNK_MS_SMOOTH 1
#define NNK_MS_INVERSE 2
#define NNK_MS_GRAD 3
#define NNK_MS_LOGPOWER 4
#define NNK_MS_POSTFILTER 5

int nnk_modspec(int32_t mode, int32_t dtype, int32_t n, const void* in, const void* in2, void* out, void* out2,
                int32_t B, int32_t T_in, int32_t T_out, int32_t D, const int32_t* lengths, double fwd_scale,
                double inv_scale, int32_t limit_bin, int32_t log_domain, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NNK_MODSPEC_H */
