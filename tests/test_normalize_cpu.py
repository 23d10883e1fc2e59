"""CPU: the normalisation restatement against the reference's own outputs, the host-side helpers, and
every argument error of preprocessing.meanvar / meanstd / minmax / the scale family, raised before any
launch (so without a GPU)."""
import hashlib
import os

import numpy as np
import pytest

import oracle.normalize as R
from conftest import ROOT
from nnmnkwii_b200 import preprocessing as P


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(ROOT, "tests", "golden", "normalize_reference_golden.npz"))


def _digest(a):
    """The golden file stores the scaling outputs as 'dtype shape sha256' of their C-order bytes."""
    a = np.ascontiguousarray(a)
    return "%s %s %s" % (a.dtype.str, "x".join(map(str, a.shape)), hashlib.sha256(a.tobytes()).hexdigest())


def _inc_input():
    """The input of the reference's test_meanvar_incremental (np.random.seed(1234); randn(32, 100, 24))."""
    return np.random.RandomState(1234).randn(32, 100, 24)


def _utts(g, name):
    return [g["%s_%d" % (name, i)] for i in range(3)]


def _padded(g, name):
    u = _utts(g, name)
    pad = np.zeros((3, 1000, u[0].shape[1]), dtype=u[0].dtype)
    for i, x in enumerate(u):
        pad[i, :len(x)] = x
    return pad


@pytest.mark.parametrize("name", ["X", "Y"])
def test_restatement_reproduces_reference(g, name):
    u, pad, lens = _utts(g, name), _padded(g, name), g[name + "_lengths"]
    for got, key in ((R.meanvar(u), "%s_mean %s_var"), (R.meanvar(pad, lens), "%s_pad_mean %s_pad_var"),
                     (R.meanstd(u), "%s_mean %s_std"), (R.minmax(u), "%s_min %s_max"),
                     (R.minmax(pad, lens), "%s_pad_min %s_pad_max")):
        for a, k in zip(got, key.split()):
            ref = g[k % name]
            assert a.dtype == ref.dtype and np.array_equal(a, ref), k % name


def test_restatement_incremental_and_scaling(g):
    inc = _inc_input()
    ma, va, n = R.meanvar(inc[:16], return_last_sample_count=True)
    assert n == int(g["inc_count_a"]) == 1600
    assert np.array_equal(ma, g["inc_mean_a"]) and np.array_equal(va, g["inc_var_a"])
    mb, vb = R.meanvar(inc[16:], mean_=ma, var_=va, last_sample_count=n)
    assert np.array_equal(mb, g["inc_mean_b"]) and np.array_equal(vb, g["inc_var_b"])
    y0, x0 = g["Y_0"], g["X_0"]
    sy = R.scale(y0, g["Y_mean"], g["Y_std"])
    assert _digest(sy) == str(g["scale_Y0"])
    assert _digest(R.inv_scale(sy, g["Y_mean"], g["Y_std"])) == str(g["inv_scale_Y0"])
    fr = (0.01, 0.99)
    sx = R.minmax_scale(x0, g["X_min"], g["X_max"], feature_range=fr)
    assert _digest(sx) == str(g["minmax_scale_X0"])
    assert _digest(R.inv_minmax_scale(sx, g["X_min"], g["X_max"], feature_range=fr)) == str(g["inv_minmax_scale_X0"])


def test_host_helpers_equal_reference(g):
    m, s = P.minmax_scale_params(g["X_min"], g["X_max"], feature_range=(0.01, 0.99))
    assert m.dtype == g["params_min_"].dtype and np.array_equal(m, g["params_min_"])
    assert s.dtype == g["params_scale_"].dtype and np.array_equal(s, g["params_scale_"])
    out = P.remove_zeros_frames(g["rz_in"])
    assert np.array_equal(out, g["rz_out"])


def test_package_reexports_reference_names():
    for name in ("meanvar", "meanstd", "minmax", "scale", "inv_scale", "minmax_scale_params", "minmax_scale",
                 "inv_minmax_scale", "remove_zeros_frames", "trim_zeros_frames"):
        assert callable(getattr(P, name)) and name in P.__all__


_X3 = np.ones((2, 4, 3), np.float32)


@pytest.mark.parametrize("fn", [P.meanvar, P.meanstd, P.minmax])
@pytest.mark.parametrize("args,match", [
    ((np.ones((4, 3), np.float32),), "2-D"),
    ((_X3, [4]), "entries"),
    ((_X3, [4, 2, 1]), "entries"),
    ((_X3, [4, -1]), ">= 0"),
    ((_X3, [0, 0]), "no frames"),
    ((np.ones((2, 0, 3)),), "no frames"),
    (([],), "empty"),
    (([np.ones((4, 3))], [1.5]), "integers"),
    ((iter([np.ones((4, 3))]), [4]), "sized"),
])
def test_argument_errors_before_any_launch(fn, args, match):
    with pytest.raises(ValueError, match=match):
        fn(*args)


def test_incoming_count_allows_no_frames_for_meanvar_only():
    import torch
    if torch.cuda.is_available():
        pytest.skip("checks the argument path without a GPU")
    with pytest.raises(RuntimeError, match="CUDA"):  # passes validation, then needs the device
        P.meanvar(_X3, [0, 0], mean_=np.zeros(3), var_=np.ones(3), last_sample_count=5)
    with pytest.raises(ValueError):
        P.minmax(_X3, [0, 0])
    with pytest.raises(ValueError, match=">= 0"):
        P.meanvar(_X3, last_sample_count=-1)


@pytest.mark.parametrize("fn", [P.minmax_scale, P.inv_minmax_scale])
def test_minmax_scale_needs_range_or_params(fn):
    x = np.ones((4, 3), np.float32)
    with pytest.raises(ValueError):
        fn(x)
    with pytest.raises(ValueError):
        fn(x, data_min=np.zeros(3))
    with pytest.raises(ValueError):
        fn(x, scale_=np.ones(3))


def test_no_gpu_means_loud_failure():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    for call in (lambda: P.meanvar(_X3), lambda: P.minmax([np.ones((4, 3))]),
                 lambda: P.scale(np.ones((4, 3)), np.zeros(3), np.ones(3)),
                 lambda: P.inv_scale(np.ones((4, 3)), np.zeros(3), np.ones(3))):
        with pytest.raises(RuntimeError, match="CUDA"):
            call()
