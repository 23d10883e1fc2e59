"""Float64 NumPy restatement of the utterance-level modulation-spectrum (MS) post-filter and its statistics.  TEST
INFRASTRUCTURE, NOT PRODUCT.

Written from Takamichi et al., "A postfilter to modify the modulation spectrum in HMM-based speech synthesis",
ICASSP 2014, with this project's choices (postfilters.modspec_post_filter, DESIGN.md 3.16).  One utterance x of
T <= n frames, one column: Y = rfft(x, n), s = log(max(|Y|^2, tiny)), tiny the smallest normal number of x's dtype.

    statistics   mean and population variance of s over utterances, (n // 2 + 1, D) each
    post-filter  g = sqrt(v_N / v_G) (1 where v_G == 0), s' = (1 - k) s + k (g (s - mu_G) + mu_N),
                 C = Y / |Y| exp(s' / 2) on bins >= 1 of non-zero power, C_0 = Y_0, 0 elsewhere;
                 irfft(C, n)[:T]
"""
import numpy as np


def log_ms(x, n):
    """``(s, Y, P)`` of a ``(T, D)`` utterance: log power, spectrum and power, float64, ``(n // 2 + 1, D)``."""
    x = np.asarray(x)
    tiny = np.finfo(x.dtype if x.dtype.kind == "f" else np.float64).tiny
    Y = np.fft.rfft(x.astype(np.float64), n, axis=0)
    P = Y.real ** 2 + Y.imag ** 2
    return np.log(np.maximum(P, tiny)), Y, P


def statistics(utts, n):
    """``(mean, var)`` of the log MS over a list of ``(T, D)`` utterances."""
    s = np.stack([log_ms(u, n)[0] for u in utts])
    return s.mean(axis=0), s.var(axis=0)


def post_filter(x, natural, generated, k, n):
    """The filtered ``(T, D)`` utterance, float64."""
    (mu_n, v_n), (mu_g, v_g) = [(np.asarray(m, np.float64), np.asarray(v, np.float64)) for m, v in (natural, generated)]
    s, Y, P = log_ms(x, n)
    g = np.sqrt(np.divide(v_n, v_g, out=np.ones_like(v_n), where=v_g > 0))
    s2 = (1.0 - k) * s + k * (g * (s - mu_g) + mu_n)
    live = P > 0
    C = np.where(live, Y / np.where(live, np.abs(Y), 1.0) * np.exp(s2 / 2), 0)
    C[0] = Y[0]
    return np.fft.irfft(C, n, axis=0)[:len(x)]
