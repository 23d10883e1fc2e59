"""Restatement of the reference's waveform and F0 preprocessing on scipy and NumPy.  TEST INFRASTRUCTURE.

interp1d, preemphasis / inv_preemphasis and the mu-law family as nnmnkwii.preprocessing computes them
(generic.py:56-226, f0.py): the same scipy calls and the same NumPy / torch promotion chains, written
from their documented behaviour.  tests/test_wave_cpu.py checks it against the reference's own outputs
(tests/golden/wave_reference_golden.npz); the GPU tests compare the device functions against it.
"""
import numpy as np
from scipy import interpolate, signal


def interp1d(f0, kind="slinear"):
    if len(f0) != f0.size:
        raise RuntimeError("1d array is only supported")
    y = f0.flatten()
    voiced = np.flatnonzero(y > 0)
    if voiced.size == 0:
        return f0
    y[0], y[-1] = y[voiced[0]], y[voiced[-1]]
    voiced = np.flatnonzero(y > 0)
    fill = np.flatnonzero(y <= 0)  # NaN is neither voiced nor filled
    y[fill] = interpolate.interp1d(voiced, y[voiced], kind=kind)(fill)
    return y[:, None] if f0.ndim == 2 else y


def preemphasis(x, coef=0.97):
    return signal.lfilter(np.array([1.0, -coef], x.dtype), np.array([1.0], x.dtype), x)


def inv_preemphasis(x, coef=0.97):
    return signal.lfilter(np.array([1.0], x.dtype), np.array([1.0, -coef], x.dtype), x)


def _is_np(x):
    return isinstance(x, np.ndarray) or np.isscalar(x)


def mulaw(x, mu=256):
    if _is_np(x):
        return np.sign(x) * np.log1p(mu * np.abs(x)) / np.log1p(mu)
    return x.sign() * (mu * x.abs()).log1p() / np.log1p(mu)


def inv_mulaw(y, mu=256):
    if _is_np(y):
        return np.sign(y) * (1.0 / mu) * ((1.0 + mu) ** np.abs(y) - 1.0)
    return y.sign() * (1.0 / mu) * ((1.0 + mu) ** y.abs() - 1.0)


def mulaw_quantize(x, mu=256):
    y = (mulaw(x, mu) + 1) / 2 * mu
    if isinstance(y, np.ndarray):
        return y.astype(int)
    return int(y) if np.isscalar(y) else y.long()


def mulaw_quantize_unrounded(x, mu=256):
    """The value mulaw_quantize truncates."""
    return (mulaw(x, mu) + 1) / 2 * mu


def inv_mulaw_quantize(y, mu=256):
    if isinstance(y, np.ndarray):
        f = y.astype(np.float32)
    elif np.isscalar(y):
        f = float(y)
    else:
        f = y.float()
    return inv_mulaw(2 * f / mu - 1, mu)
