"""Merlin post-filter oracle: restated SPTK, not pysptk.  TEST INFRASTRUCTURE, NOT PRODUCT.

pysptk is not available to the tests, so the reference's ``merlin_post_filter``
(nnmnkwii/postfilters/__init__.py:7-62) cannot run.  This module restates, literally and in float64, the
four SPTK routines it calls -- ``freqt`` (SPTK freqt.c), ``c2acr`` (c2acr.c, with numpy's FFT for
``fftr``), ``mc2b`` (mc2b.c), ``b2mc`` (b2mc.c) -- and the reference's five-step chain over them.  It
deliberately does not use the collapsed basis form of csrc/nnk_postfilter.cu, so the kernel is checked
against an independent computation.  tests/golden/merlin_post_filter_golden.npz holds Merlin's own SPTK
command-line output for the same chain.
"""
import numpy as np

__all__ = ["freqt", "c2acr", "mc2b", "b2mc", "merlin_post_filter_steps", "merlin_post_filter"]


def freqt(c1, m2, a):
    """Frequency transform of the cepstra c1 (..., m1 + 1) to order m2 with all-pass constant a.

    SPTK's loop, run on every frame at once (leading axes are frames; no arithmetic mixes them)."""
    c1 = np.asarray(c1, dtype=np.float64)
    m1 = c1.shape[-1] - 1
    g = np.zeros(c1.shape[:-1] + (m2 + 1,))
    d = np.zeros_like(g)
    b = 1 - a * a
    for i in range(-m1, 1):
        if 0 <= m2:
            d[..., 0] = g[..., 0]
            g[..., 0] = c1[..., -i] + a * d[..., 0]
        if 1 <= m2:
            d[..., 1] = g[..., 1]
            g[..., 1] = b * d[..., 0] + a * d[..., 1]
        for j in range(2, m2 + 1):
            d[..., j] = g[..., j]
            g[..., j] = d[..., j - 1] + a * (d[..., j] - g[..., j - 1])
    return g


def c2acr(c, m2, flng):
    """Autocorrelation r[0..m2] of the cepstra c (..., m1 + 1) through an flng-point FFT: zero-padded buffer,
    real part of its DFT (fftr), exp of twice that, DFT again, divided by flng."""
    c = np.asarray(c, dtype=np.float64)
    x = np.zeros(c.shape[:-1] + (flng,))
    x[..., :c.shape[-1]] = c
    x = np.fft.fft(x, axis=-1).real
    x = np.exp(2.0 * x)
    x = np.fft.fft(x, axis=-1).real
    return x[..., :m2 + 1] / flng


def mc2b(mc, a):
    """Mel-cepstrum to MLSA filter coefficients (last axis)."""
    mc = np.asarray(mc, dtype=np.float64)
    m = mc.shape[-1] - 1
    b = np.empty_like(mc)
    b[..., m] = mc[..., m]
    for k in range(m - 1, -1, -1):
        b[..., k] = mc[..., k] - a * b[..., k + 1]
    return b


def b2mc(b, a):
    """MLSA filter coefficients to mel-cepstrum (last axis; inverse of mc2b)."""
    b = np.asarray(b, dtype=np.float64)
    m = b.shape[-1] - 1
    mc = np.empty_like(b)
    d = mc[..., m] = b[..., m]
    for k in range(m - 1, -1, -1):
        o = b[..., k] + a * d
        d = b[..., k]
        mc[..., k] = o
    return mc


def _weight(D, coef, weight):
    if weight is None:
        weight = np.ones(D) * coef
        weight[:2] = 1
    return np.asarray(weight, dtype=np.float64)


def merlin_post_filter_steps(mgc, alpha, minimum_phase_order=511, fftlen=1024, coef=1.4, weight=None):
    """The reference's chain in float64 (postfilters/__init__.py:48-62):
    (mgc_r0, mgc_p_r0, mgc_b0, mgc_p_b0, mgc_p_mgc)."""
    mgc = np.asarray(mgc, dtype=np.float64)
    _, D = mgc.shape
    w = _weight(D, coef, weight)
    assert len(w) == D
    r0 = c2acr(freqt(mgc, minimum_phase_order, -alpha), 0, fftlen)[:, 0]
    p_r0 = c2acr(freqt(mgc * w, minimum_phase_order, -alpha), 0, fftlen)[:, 0]
    bw = mc2b(w * mgc, alpha)
    b0 = bw[:, 0]
    p_b0 = np.log(r0 / p_r0) / 2 + b0
    out = b2mc(np.hstack((p_b0[:, None], bw[:, 1:])), alpha)
    return r0, p_r0, b0, p_b0, out


def merlin_post_filter(mgc, alpha, minimum_phase_order=511, fftlen=1024, coef=1.4, weight=None):
    """Post-filtered mel-cepstrum (float64) by the restated SPTK chain."""
    return merlin_post_filter_steps(mgc, alpha, minimum_phase_order, fftlen, coef, weight)[4]
