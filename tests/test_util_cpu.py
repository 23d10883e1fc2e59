"""CPU: nnmnkwii_b200.util -- imports and re-exports, apply_each2d_trim / apply_each2d_padded on NumPy
input against the reference's definitions (restated here), every argument error of util.linalg raised
before any launch, and the float64 restatement of the dense kernel's order against LAPACK's dpotri,
which sets the tolerance tests/test_util_gpu.py holds the GPU to."""
import os
import re

import numpy as np
import pytest

import linalg_mirror as M
from conftest import ROOT
from nnmnkwii_b200 import _lib
from nnmnkwii_b200 import preprocessing as Pp
from nnmnkwii_b200 import util
from nnmnkwii_b200.util import linalg


def test_imports_and_reexports():
    for name in ("adjust_frame_length", "delta_features", "meanstd", "meanvar", "minmax", "minmax_scale",
                 "remove_zeros_frames", "scale", "trim_zeros_frames"):
        assert getattr(util, name) is getattr(Pp, name), name
    assert util.apply_delta_windows is Pp.delta_features
    assert util.linalg is linalg
    assert callable(util.apply_each2d_trim) and callable(util.apply_each2d_padded)
    assert callable(linalg.cholesky_inv) and callable(linalg.cholesky_inv_banded)
    assert "nnk_cholesky_inv" in _lib.EXPORTS and "nnk_cholesky_inv_banded" in _lib.EXPORTS


# ---- the reference's definitions (nnmnkwii/util/__init__.py:19-66), restated ----------------------------
def ref_apply_each2d_trim(func2d, X, *args, **kwargs):
    assert X.ndim == 3
    N, T, _ = X.shape
    x = Pp.trim_zeros_frames(X[0])
    y = func2d(x, *args, **kwargs)
    assert y.ndim == 2
    _, D = y.shape
    Y = np.zeros((N, T, D))
    for idx in range(N):
        x = Pp.trim_zeros_frames(X[idx])
        y = func2d(x, *args, **kwargs)
        Y[idx][: len(y)] = y
    return Y


def ref_apply_each2d_padded(func2d, X, lengths, *args, **kwargs):
    assert X.ndim == 3
    N, T, _ = X.shape
    y = func2d(X[0][: lengths[0]], *args, **kwargs)
    assert y.ndim == 2
    _, D = y.shape
    Y = np.zeros((N, T, D))
    Y[0][: len(y)] = y
    for idx in range(1, N):
        y = func2d(X[idx][: lengths[idx]], *args, **kwargs)
        Y[idx][: len(y)] = y
    return Y


def _widen(x, windows):
    """A func2d that changes the width like delta_features with three windows, on the host."""
    if len(x) == 0:
        return np.zeros((0, x.shape[1] * len(windows)))
    return np.concatenate([np.apply_along_axis(np.correlate, 0, x, np.asarray(w[2]), mode="same")
                           for w in windows], axis=1)


def _batch(rng, dtype=np.float64):
    X = rng.standard_normal((4, 30, 5)).astype(dtype)
    X[0, 22:] = 0.0          # zero tail
    X[1] = 0.0               # all-zero slice
    X[2, 17:] = 0.0
    X[2, 16] = [1e-8, 0, 0, 0, 0]  # below eps: trimmed
    return X


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_apply_each2d_numpy_matches_reference(dtype):
    from conftest import windows_set
    windows = windows_set()[2]
    X = _batch(np.random.default_rng(0), dtype)
    calls = []

    def f(x, *a, **k):
        calls.append(len(x))
        return _widen(x, *a, **k)

    Y = util.apply_each2d_trim(f, X, windows)
    assert Y.dtype == np.float64 and Y.shape == (4, 30, 15)
    assert np.array_equal(Y, ref_apply_each2d_trim(_widen, X, windows))
    assert calls == [22, 0, 16, 30]  # once per slice (the reference calls slice 0 twice)
    lengths = [30, 3, 0, 12]
    Y = util.apply_each2d_padded(_widen, X, lengths, windows=windows)
    assert np.array_equal(Y, ref_apply_each2d_padded(_widen, X, lengths, windows=windows))


def test_apply_each2d_reference_function_utils():
    """The reference's tests/test_util.py:28-49."""
    T, D = 10, 24
    np.random.seed(1234)
    X = np.random.rand(2, T, D)
    lengths = [60, 100]
    Y = util.apply_each2d_padded(lambda x: x + 1, X, lengths)
    for i, n in enumerate(lengths):
        assert np.allclose(X[i][:n] + 1, Y[i][:n]) and np.all(Y[i][n:] == 0)
    for i, n in enumerate(lengths):
        X[i][n:] = 0
    Y = util.apply_each2d_trim(lambda x: x + 1, X)
    for i, n in enumerate(lengths):
        assert np.allclose(X[i][:n] + 1, Y[i][:n]) and np.all(Y[i][n:] == 0)


# ---- argument errors: raised before anything reaches the device ------------------------------------------
@pytest.mark.parametrize("call, exc", [
    (lambda: linalg.cholesky_inv(np.eye(3)[:2]), AssertionError),
    (lambda: linalg.cholesky_inv(np.zeros((2, 3, 4))), AssertionError),
    (lambda: linalg.cholesky_inv(np.eye(3)[0]), ValueError),
    (lambda: linalg.cholesky_inv(np.zeros((1, 2, 3, 3))), ValueError),
    (lambda: linalg.cholesky_inv(np.eye(3, dtype=np.float32)), AssertionError),
    (lambda: linalg.cholesky_inv(np.eye(3, dtype=np.float32), lower=True), AssertionError),
    (lambda: linalg.cholesky_inv_banded(np.eye(3)[:2]), AssertionError),
    (lambda: linalg.cholesky_inv_banded(np.eye(3)[0]), ValueError),
    (lambda: linalg.cholesky_inv_banded(np.eye(3), 0), ValueError),
    (lambda: linalg.cholesky_inv_banded(np.eye(3), -2), ValueError),
    (lambda: linalg.cholesky_inv_banded(np.eye(3), 2.5), ValueError),
])
def test_argument_errors_before_launch(call, exc):
    n0 = _lib.launch_count()
    with pytest.raises(exc):
        call()
    assert _lib.launch_count() == n0


def test_tensor_dtype_error_before_launch():
    torch = pytest.importorskip("torch")
    n0 = _lib.launch_count()
    with pytest.raises(TypeError):
        linalg.cholesky_inv(torch.eye(3, dtype=torch.int64))
    with pytest.raises(TypeError):
        linalg.cholesky_inv_banded(torch.eye(3, dtype=torch.float16))
    assert _lib.launch_count() == n0


def test_apply_each2d_rejects_2d():
    with pytest.raises(AssertionError):
        util.apply_each2d_trim(lambda x: x, np.zeros((3, 4)))
    with pytest.raises(AssertionError):
        util.apply_each2d_padded(lambda x: x, np.zeros((3, 4)), [3])


# ---- the dense kernel's order against dpotri: the GPU tolerance ------------------------------------------
@pytest.mark.parametrize("lower", [True, False])
def test_dense_restatement_sets_the_gpu_bar(lower):
    rng = np.random.default_rng(0)
    worst = 0.0
    for N in (1, 2, 31, 32, 33, 64, 65, 130, 256, 512):
        F, ref = M.spd_factor(rng, N, lower)
        P = M.dense_restatement(F, lower)
        assert np.array_equal(P, P.T)
        worst = max(worst, M.rel_to_scale(P, ref) / (np.sqrt(N) * M.EPS))
    assert worst <= M.DENSE_BAR / 2, worst


def test_dense_restatement_reads_one_triangle():
    rng = np.random.default_rng(1)
    F, _ = M.spd_factor(rng, 40, True, garbage=False)
    G, _ = M.spd_factor(np.random.default_rng(1), 40, True, garbage=True)
    assert np.array_equal(M.dense_restatement(F, True), M.dense_restatement(G, True))
    assert np.array_equal(M.dense_restatement(F, True), M.dense_restatement(F.T.copy(), False))


def test_mirror_constants_match_the_source():
    with open(os.path.join(ROOT, "nnmnkwii_b200", "csrc", "nnk_linalg.cu")) as f:
        src = f.read()
    for name, val in (("kDenseBlock", M.BLOCK), ("kDenseRows", M.ROWS)):
        assert int(re.search(r"constexpr int %s = (\d+);" % name, src).group(1)) == val, name


def test_banded_oracle_on_golden(golden):
    """The float64 restatement of the banded recurrence the GPU is held to, bit for bit, on the reference's
    own output (zeros compared by value)."""
    import oracle
    assert np.array_equal(oracle.cholesky_inv_banded(golden["cib_L"], 3), golden["cib_Pinv"])
