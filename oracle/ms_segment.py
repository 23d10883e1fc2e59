"""Float64 NumPy restatement of the segment-level modulation-spectrum (MS) post-filter and its statistics.  TEST
INFRASTRUCTURE, NOT PRODUCT.

Written from Takamichi et al., "A postfilter to modify the modulation spectrum in HMM-based speech synthesis",
ICASSP 2014, with this project's choices (postfilters.modspec_post_filter(segment=L), DESIGN.md 3.16).  One
utterance x of T frames, one column; hop H = L / 2, periodic Hann window w_m = 0.5 - 0.5 cos(2 pi m / L):

    segments     j = 0 .. J - 1, J = ceil(T / H) + 1 (0 for T = 0), segment j = x[(j - 1) H : (j - 1) H + L]
                 with frames outside [0, T) taken as 0
    per segment  Y_j = rfft(w * segment j, n), s_j = log(max(|Y_j|^2, tiny)), tiny of x's dtype
    statistics   mean and population variance of s_j over all segments of all utterances, (n // 2 + 1, D)
    post-filter  C_j as in oracle/ms_postfilter.py, y_t = sum_j irfft(C_j, n)[t - (j - 1) H] over the j with
                 0 <= t - (j - 1) H < L
Explicit loops over the segments, on purpose: it restates the definition, not the kernel.
"""
import numpy as np


def window(L):
    m = np.arange(L)
    return 0.5 - 0.5 * np.cos(2 * np.pi * m / L)


def count(T, L):
    """Segments of an utterance of ``T`` frames."""
    return 0 if T == 0 else -(-T // (L // 2)) + 1


def segments(x, L):
    """``(J, L, D)`` float64 windowed segments of a ``(T, D)`` utterance."""
    x = np.asarray(x)
    T, D = x.shape
    H = L // 2
    w = window(L)[:, None]
    out = np.zeros((count(T, L), L, D))
    for j in range(len(out)):
        s = (j - 1) * H
        for m in range(L):
            if 0 <= s + m < T:
                out[j, m] = x[s + m]
        out[j] *= w
    return out


def _tiny(x):
    x = np.asarray(x)
    return np.finfo(x.dtype if x.dtype.kind == "f" else np.float64).tiny


def log_ms(x, n, L):
    """``(s, Y, P)`` of every segment of a ``(T, D)`` utterance, float64, ``(J, n // 2 + 1, D)`` each."""
    Y = np.fft.rfft(segments(x, L), n, axis=1)
    P = Y.real ** 2 + Y.imag ** 2
    return np.log(np.maximum(P, _tiny(x))), Y, P


def statistics(utts, n, L):
    """``(mean, var)`` of the log MS over every segment of a list of ``(T, D)`` utterances."""
    s = np.concatenate([log_ms(u, n, L)[0] for u in utts])
    return s.mean(axis=0), s.var(axis=0)


def post_filter(x, natural, generated, k, n, L):
    """The filtered ``(T, D)`` utterance, float64."""
    (mu_n, v_n), (mu_g, v_g) = [(np.asarray(m, np.float64), np.asarray(v, np.float64)) for m, v in (natural, generated)]
    x = np.asarray(x)
    T = len(x)
    H = L // 2
    s, Y, P = log_ms(x, n, L)
    g = np.sqrt(np.divide(v_n, v_g, out=np.ones_like(v_n), where=v_g > 0))
    y = np.zeros((T, x.shape[1]))
    for j in range(len(s)):
        s2 = (1.0 - k) * s[j] + k * (g * (s[j] - mu_g) + mu_n)
        live = P[j] > 0
        C = np.where(live, Y[j] / np.where(live, np.abs(Y[j]), 1.0) * np.exp(s2 / 2), 0)
        C[0] = Y[j][0]
        seg = np.fft.irfft(C, n, axis=0)
        for m in range(L):
            t = (j - 1) * H + m
            if 0 <= t < T:
                y[t] += seg[m]
    return y
