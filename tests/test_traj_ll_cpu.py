"""The trajectory-model log-likelihood without a GPU: the float64 restatement (tests/traj_ll_oracle.py) against
scipy's multivariate normal, a dense torch autograd formulation, central differences and its own banded path; the
argument errors of paramgen.trajectory_log_likelihood_batch, raised before any launch, and those of the C entry
point."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
from scipy.stats import multivariate_normal

import traj_ll_oracle as O
from conftest import ROOT

_spec = importlib.util.spec_from_file_location("make_gmm_traj_golden",
                                               os.path.join(ROOT, "tests", "golden", "make_gmm_traj_golden.py"))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
SETS = MG.em_window_sets()


def _chain_data(rng, T, nw, ratio=1.0):
    mean = rng.standard_normal((T, nw)) * 0.5
    var = rng.random((T, nw)) + 0.5
    var[:, 1:] /= ratio
    x = np.cumsum(rng.standard_normal(T)) * 0.1
    return x, mean, var


@pytest.mark.parametrize("name", list(SETS))
def test_ll_is_the_gaussian_log_density(name):
    w = SETS[name]
    rng = np.random.default_rng(len(name))
    for T in (1, 2, 5, 13, 40):
        x, mean, var = _chain_data(rng, T, len(w))
        r = O.chain(x, mean, var, w)
        want = multivariate_normal.logpdf(x, r["cbar"], np.linalg.inv(r["P"]))
        assert abs(r["ll"] - want) <= 1e-10 * max(1.0, abs(want)), (T, r["ll"], want)


@pytest.mark.parametrize("name", list(SETS))
def test_banded_path_equals_the_dense_one(name):
    w = SETS[name]
    rng = np.random.default_rng(7 + len(name))
    for T in (1, 3, 9, 60):
        x, mean, var = _chain_data(rng, T, len(w), ratio=1e4 if T == 60 else 1.0)
        d, b = O.chain(x, mean, var, w), O.chain(x, mean, var, w, banded=True)
        assert abs(d["ll"] - b["ll"]) <= 1e-11 * max(1.0, abs(d["ll"]))
        for k in ("cbar", "g_mean", "g_var", "g_x"):
            assert np.abs(d[k] - b[k]).max() <= 1e-10 * max(1e-300, np.abs(d[k]).max()), (T, k)


@pytest.mark.parametrize("name", ["nw3", "hw2", "hw4", "asym"])
def test_sigma_band_is_the_band_of_the_inverse(name):
    w = SETS[name]
    S = max(l for l, _, _ in w) + max(u for _, u, _ in w)
    x, mean, var = _chain_data(np.random.default_rng(3), 50, len(w))
    P = O.chain(x, mean, var, w)["P"]
    sig, _ = O.sigma_band(O._band(P, S))
    inv = np.linalg.inv(P)
    for j in range(S + 1):
        want = np.concatenate([np.diagonal(inv, j), np.zeros(j)])
        assert np.abs(sig[:, j] - want).max() <= 1e-12 * np.abs(inv).max(), j


def _torch_ll(x, mean, var, w):
    """Dense float64 CPU torch formulation: logdet and solve, differentiable in x, mean and var."""
    import torch
    T = x.shape[0]
    st = O._Stream(w, False)
    mats = [torch.from_numpy(W) for W in st.window_matrices(T)]
    keep = torch.from_numpy(st.kept(T))
    tau = torch.where(keep, 1.0 / var, torch.zeros_like(var))
    P = sum(W.T @ (tau[:, i:i + 1] * W) for i, W in enumerate(mats))
    b = sum(W.T @ (tau[:, i] * mean[:, i]) for i, W in enumerate(mats))
    cbar = torch.linalg.solve(P, b)
    e = x - cbar
    return 0.5 * torch.logdet(P) - 0.5 * e @ (P @ e) - 0.5 * T * O.LOG_2PI


@pytest.mark.parametrize("name", ["nw2", "nw3", "hw2", "asym", "hw3", "h0"])
def test_gradients_equal_torch_autograd_and_central_differences(name):
    import torch
    w = SETS[name]
    rng = np.random.default_rng(11 + len(name))
    for T in (1, 4, 17):
        x, mean, var = _chain_data(rng, T, len(w))
        r = O.chain(x, mean, var, w)
        tx, tm, tv = (torch.tensor(a, requires_grad=True) for a in (x, mean, var))
        ll = _torch_ll(tx, tm, tv, w)
        ll.backward()
        assert abs(ll.item() - r["ll"]) <= 1e-10 * max(1.0, abs(r["ll"]))
        for got, t in ((r["g_x"], tx), (r["g_mean"], tm), (r["g_var"], tv)):
            want = t.grad.numpy()
            assert np.abs(got - want).max() <= 1e-10 * max(1e-300, np.abs(want).max()), (T, name)
        # central differences on a few entries of each input
        h = 1e-6
        for arr, g in ((x, r["g_x"]), (mean, r["g_mean"]), (var, r["g_var"])):
            for idx in list(np.ndindex(arr.shape))[:: max(1, arr.size // 5)]:
                a1, a2 = arr.copy(), arr.copy()
                a1[idx] += h
                a2[idx] -= h
                args1 = [a1 if arr is a else a for a in (x, mean, var)]
                args2 = [a2 if arr is a else a for a in (x, mean, var)]
                fd = (O.chain(*args1, w)["ll"] - O.chain(*args2, w)["ll"]) / (2 * h)
                assert abs(fd - g[idx]) <= 1e-6 * max(1.0, abs(g[idx])), (idx, fd, g[idx])


def test_edge_frames_have_zero_gradients():
    w = SETS["hw2"]
    x, mean, var = _chain_data(np.random.default_rng(5), 30, len(w))
    r = O.chain(x, mean, var, w)
    H = 2
    assert np.all(r["g_mean"][:H, 1:] == 0) and np.all(r["g_mean"][-H:, 1:] == 0)
    assert np.all(r["g_var"][:H, 1:] == 0) and np.all(r["g_var"][-H:, 1:] == 0)


def test_static_window_alone_is_the_per_frame_gaussian():
    w = [(0, 0, np.array([1.0]))]
    rng = np.random.default_rng(9)
    x, mean, var = _chain_data(rng, 25, 1)
    r = O.chain(x, mean, var, w)
    want = np.sum(-0.5 * np.log(2 * np.pi * var[:, 0]) - 0.5 * (x - mean[:, 0]) ** 2 / var[:, 0])
    assert abs(r["ll"] - want) <= 1e-12 * abs(want)


@pytest.mark.parametrize("name", list(SETS))
def test_the_mlpg_trajectory_is_the_mode(name):
    w = SETS[name]
    rng = np.random.default_rng(13 + len(name))
    x, mean, var = _chain_data(rng, 40, len(w))
    r = O.chain(x, mean, var, w)
    at_mode = O.chain(r["cbar"], mean, var, w)
    assert at_mode["ll"] >= r["ll"]
    assert np.abs(at_mode["g_x"]).max() <= 1e-9 * np.abs(r["g_x"]).max()
    assert np.abs(at_mode["g_mean"]).max() <= 1e-9 * np.abs(r["g_mean"]).max()


def test_layout_oracle_zeroes_copied_columns():
    import nnmnkwii_b200.paramgen as G  # noqa: F401  (the layout below is merlin_layout's)
    w = MG.WINDOWS
    streams = [(0, 60), (180, 1), (183, 1, "copy"), (184, 1)]
    rng = np.random.default_rng(2)
    T = 12
    m, v = rng.standard_normal((T, 187)), rng.random((T, 187)) + 0.5
    x = rng.standard_normal((T, 63))
    ll, gm, gv, gx = O.log_likelihood(x, m, v, w, streams)
    assert ll[61] == 0 and not gm[:, 183].any() and not gv[:, 183].any() and not gx[:, 61].any()
    ll1, gm1, gv1, gx1 = O.log_likelihood(x, m, v[0], w, streams)
    assert gv1.shape == (187,) and gv1[183] == 0


# ---- argument errors -------------------------------------------------------------------------------------------
def _args():
    rng = np.random.default_rng(0)
    w = MG.WINDOWS
    m = rng.standard_normal((30, 9))
    v = rng.random((30, 9)) + 0.5
    x = rng.standard_normal((30, 3))
    return x, m, v, w


def test_argument_errors_raise_before_any_launch(monkeypatch):
    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200 import paramgen as G

    def no_launch(*a, **k):
        raise AssertionError("launched")
    monkeypatch.setattr(G, "_traj_ll_device", no_launch)
    x, m, v, w = _args()
    f = G.trajectory_log_likelihood_batch
    bad = [
        lambda: f(x.astype(np.float32), m, v, w, lengths=[30]),
        lambda: f(x, m.astype(np.float32), v, w, lengths=[30]),
        lambda: f(x, m.astype(np.int64), v.astype(np.int64), w, lengths=[30]),
        lambda: f(x[:, :2], m, v, w, lengths=[30]),
        lambda: f(x[:29], m, v, w, lengths=[30]),
        lambda: f(x, m, v[:, :8], w, lengths=[30]),
        lambda: f(x, m, v[0, :8], w, lengths=[30]),
        lambda: f(x, m, v, w, lengths=[20]),
        lambda: f(x, m, v, w, lengths=[20, 20]),
        lambda: f(x, m, v, w, layout=G.merlin_layout()),
        lambda: f(x, m, v, [], lengths=[30]),
        lambda: f(x, m, v, [(0, 0, np.array([1.0]))] * (_lib.NNK_MAX_WIN + 1), lengths=[30]),
        lambda: f(x, m, v, [(0, _lib.NNK_MAX_HALF + 1, np.ones(_lib.NNK_MAX_HALF + 2))], lengths=[30]),
        lambda: f(x, m[None], v[None], w),
        lambda: f(x, m[None], v[None], w, lengths=[30]),
        lambda: f(x[None], m[None], v[None], w, lengths=[31]),
        lambda: f(x, m[None, None], v, w, lengths=[30]),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(ValueError):
            call()
    import torch
    with pytest.raises(ValueError):  # mixed arrays and tensors
        f(torch.from_numpy(x), m, v, w, lengths=[30])
    with pytest.raises(ValueError):  # CPU tensors
        f(*(torch.from_numpy(a) for a in (x, m, v)), w, lengths=[30])


# ---- the C entry point ------------------------------------------------------------------------------------
def test_c_argument_checks():
    from nnmnkwii_b200 import _lib
    fn = _lib.lib.nnk_mlpg_traj_ll
    a, t = _lib.NnkMlpgArgs(), _lib.NnkTrajLl()
    assert fn(None, ctypes.byref(t), None) == _lib.NNK_ERR_ARG
    assert fn(ctypes.byref(a), None, None) == _lib.NNK_ERR_ARG
    a.dtype = _lib.NNK_F64
    assert fn(ctypes.byref(a), ctypes.byref(t), None) == _lib.NNK_OK  # empty batch
    t.grad = 2
    assert fn(ctypes.byref(a), ctypes.byref(t), None) == _lib.NNK_ERR_ARG
    t.grad = 1
    a.n_utt, a.n_chain, a.max_T = 1, 1, 5
    assert fn(ctypes.byref(a), ctypes.byref(t), None) == _lib.NNK_ERR_ARG  # NULL pointers
    w = _lib.make_windows(MG.WINDOWS)
    S = 2
    assert _lib.lib.nnk_mlpg_traj_ll_workspace_bytes(3, 33, 10, ctypes.byref(w)) == 3 * 2 * 10 * (S + 2) * 32 * 8
