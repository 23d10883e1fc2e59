"""CPU: the waveform / F0 restatement (oracle/wave.py) against the reference's own outputs, the host-side
frame-length helpers, and every argument error and dtype rule of interp1d, preemphasis /
inv_preemphasis and the mu-law family, raised before any launch (so without a GPU)."""
import hashlib
import os

import numpy as np
import pytest

import oracle.wave as R
from conftest import ROOT
from nnmnkwii_b200 import preprocessing as P

KINDS = ("linear", "slinear", "zero", "nearest", "nearest-up", "previous", "next")
COEFS = (0.97, 0.86, 0.0)


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(ROOT, "tests", "golden", "wave_reference_golden.npz"))


def _digest(a):
    a = np.ascontiguousarray(a)
    return "%s %s %s" % (a.dtype.str, "x".join(map(str, a.shape)), hashlib.sha256(a.tobytes()).hexdigest())


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_interp1d_restatement(g, dt):
    for i in range(3):
        lf0 = g["lf0_%d" % i].astype(dt)
        for kind in KINDS:
            key = "interp_%d_%s_%s" % (i, np.dtype(dt).name, kind)
            assert _same(R.interp1d(lf0, kind), g[key]), key
            assert _digest(R.interp1d(lf0[:, None], kind)) == str(g[key + "_col"]), key


def test_golden_f0_has_unvoiced_runs(g):
    for i in range(3):
        lf0 = g["lf0_%d" % i]
        assert (lf0 <= 0).sum() > 20 and (lf0 > 0).sum() > 20 and lf0[0] <= 0


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_preemphasis_restatement(g, dt):
    x = (g["audio"] / 32768.0).astype(dt)
    for c in COEFS:
        assert _digest(R.preemphasis(x, c)) == str(g["pre_%s_%g" % (np.dtype(dt).name, c)])
        assert _digest(R.inv_preemphasis(x, c)) == str(g["inv_%s_%g" % (np.dtype(dt).name, c)])


@pytest.mark.parametrize("mu", [256, 2])
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_mulaw_restatement_and_dtypes(g, mu, dt):
    x = (g["audio"][:1024] / 32768.0).astype(dt)
    tag = "%d_%s" % (mu, np.dtype(dt).name)
    y = R.mulaw(x, mu)
    q = R.mulaw_quantize(x, mu)
    got = {"mulaw": y, "quant": q, "inv": R.inv_mulaw(y.astype(dt), mu), "invq": R.inv_mulaw_quantize(q, mu)}
    for name, v in got.items():
        ref = g["mu_%s_%s" % (name, tag)]
        assert str(g["mu_%s_%s_dtype" % (name, tag)]) == ref.dtype.str == v.dtype.str
        assert _same(v, ref), name
    # the reference's dtype rules under NumPy 2: float32 companding divides by a float64 scalar
    assert y.dtype == np.float64 and q.dtype == np.int64 and got["invq"].dtype == np.float32


def _golden_maker():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_wave_golden",
                                                  os.path.join(ROOT, "tests", "golden", "make_wave_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_adjust_frame_lengths_against_reference(g):
    for name, x, y, kw in _golden_maker().adjust_cases():
        if y is None:
            assert _same(P.adjust_frame_length(x, **kw), g["adj_" + name]), name
            assert _same(P.adjast_frame_length(x, **kw), g["adj_" + name]), name
        else:
            a, b = P.adjust_frame_lengths(x, y, **kw)
            assert _same(a, g["adj_%s_x" % name]) and _same(b, g["adj_%s_y" % name]), name
            a, b = P.adjast_frame_lengths(x, y, **kw)
            assert _same(a, g["adj_%s_x" % name]) and _same(b, g["adj_%s_y" % name]), name


def test_adjust_frame_length_returns_input_when_divisible():
    x = np.zeros((12, 2))
    assert P.adjust_frame_length(x, divisible_by=3) is x
    with pytest.raises(AssertionError):
        P.adjust_frame_length(np.zeros((2, 2, 2)))
    with pytest.raises(AssertionError):
        P.adjust_frame_lengths(np.zeros((4, 2)), np.zeros((4, 3)))


def test_exports():
    from nnmnkwii_b200.preprocessing import (adjast_frame_length, adjast_frame_lengths,  # noqa: F401
                                             adjust_frame_length, adjust_frame_lengths, interp1d,
                                             inv_mulaw, inv_mulaw_quantize, inv_preemphasis, mulaw,
                                             mulaw_quantize, preemphasis)
    for name in ("interp1d", "preemphasis", "inv_preemphasis", "mulaw", "inv_mulaw", "mulaw_quantize",
                 "inv_mulaw_quantize", "adjust_frame_length", "adjust_frame_lengths", "adjast_frame_length",
                 "adjast_frame_lengths"):
        assert name in P.__all__


# ---- argument errors: raised before any launch --------------------------------------------------------
@pytest.mark.parametrize("kind", ["quadratic", "cubic", 2, 3])
def test_interp1d_spline_kinds_rejected(kind):
    with pytest.raises(ValueError, match="supported kinds"):
        P.interp1d(np.array([0.0, 1.0, 0.0, 2.0]), kind=kind)


def test_interp1d_argument_errors():
    with pytest.raises(NotImplementedError):
        P.interp1d(np.array([0.0, 1.0, 2.0]), kind="foo")
    with pytest.raises(RuntimeError, match="1d array"):
        P.interp1d(np.zeros((4, 2)))
    with pytest.raises(TypeError):
        P.interp1d(np.array([0, 1, 2], dtype=np.int64))
    with pytest.raises(ValueError):
        P.interp1d(np.zeros((2, 5)), lengths=[5])
    with pytest.raises(ValueError):
        P.interp1d(np.zeros((2, 5)), lengths=[5, -1])
    with pytest.raises(ValueError):
        P.interp1d(np.zeros((2, 5, 2)), lengths=[5, 5])
    with pytest.raises(ValueError):
        P.interp1d(np.zeros(5), lengths=[5])


def test_preemphasis_argument_errors():
    for f in (P.preemphasis, P.inv_preemphasis):
        for dt in (np.int16, np.int32, np.float16):
            with pytest.raises(NotImplementedError):
                f(np.arange(10).astype(dt))
        with pytest.raises(ValueError):
            f(np.zeros((2, 3, 4), np.float32), lengths=[1, 2])
        with pytest.raises(ValueError):
            f(np.zeros((2, 4), np.float32), lengths=[1])
        with pytest.raises(ValueError):
            f(np.zeros((2, 4), np.float32), lengths=[1, -2])


def test_reference_errors_match_for_integer_inputs():
    """The reference raises NotImplementedError (from scipy.signal.lfilter) for integer and float16 x."""
    for f in (R.preemphasis, R.inv_preemphasis):
        for dt in (np.int16, np.int32, np.float16):
            with pytest.raises(NotImplementedError):
                f(np.arange(10).astype(dt))


def test_mulaw_argument_errors():
    for f in (P.mulaw, P.inv_mulaw, P.mulaw_quantize):
        with pytest.raises(TypeError):
            f(np.arange(4, dtype=np.int16))
        with pytest.raises(TypeError):
            f([0.1, 0.2])
    with pytest.raises(TypeError):
        P.inv_mulaw_quantize(np.array(["a"]))


def test_no_gpu_fails_loudly(monkeypatch):
    import torch
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    x = np.array([0.0, 1.0, 0.0, 2.0, 0.0])
    for call in (lambda: P.interp1d(x), lambda: P.preemphasis(x), lambda: P.inv_preemphasis(x),
                 lambda: P.mulaw(x), lambda: P.inv_mulaw(x), lambda: P.mulaw_quantize(x),
                 lambda: P.inv_mulaw_quantize(np.array([3, 4])), lambda: P.mulaw(0.5)):
        with pytest.raises(RuntimeError, match="CUDA device"):
            call()
    assert P.adjust_frame_length(np.zeros((5, 2)), divisible_by=2).shape == (6, 2)
