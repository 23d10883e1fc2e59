"""The gradient of MLPG in its means and variances without a GPU: the float64 restatement (tests/mlpg_vjp_oracle.py)
against a dense torch autograd formulation, central differences, the reference's own paramgen.mlpg (central
differences stored in tests/golden/mlpg_vjp_reference_golden.npz) and its own banded path; the argument errors of
paramgen.mlpg_vjp_batch, raised before any launch, and those of the C entry point."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest

import mlpg_vjp_oracle as O
from conftest import ROOT

_spec = importlib.util.spec_from_file_location("make_gmm_traj_golden",
                                               os.path.join(ROOT, "tests", "golden", "make_gmm_traj_golden.py"))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
SETS = MG.em_window_sets()
_spec = importlib.util.spec_from_file_location("make_mlpg_vjp_golden",
                                               os.path.join(ROOT, "tests", "golden", "make_mlpg_vjp_golden.py"))
MV = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MV)


def _chain_data(rng, T, nw, ratio=1.0):
    mean = rng.standard_normal((T, nw)) * 0.5
    var = rng.random((T, nw)) + 0.5
    var[:, 1:] /= ratio
    o = rng.standard_normal(T)
    return o, mean, var


def _torch_grads(o, mean, var, w):
    """Dense float64 CPU torch formulation of L = o . P^-1 b, differentiated by autograd in mean and var."""
    import torch
    T = o.shape[0]
    st = O.O._Stream(w, False)
    mats = [torch.from_numpy(W) for W in st.window_matrices(T)]
    keep = torch.from_numpy(st.kept(T))
    tm, tv = (torch.tensor(a, requires_grad=True) for a in (mean, var))
    tau = torch.where(keep, 1.0 / tv, torch.zeros_like(tv))
    P = sum(W.T @ (tau[:, i:i + 1] * W) for i, W in enumerate(mats))
    b = sum(W.T @ (tau[:, i] * tm[:, i]) for i, W in enumerate(mats))
    (torch.from_numpy(o) @ torch.linalg.solve(P, b)).backward()
    return tm.grad.numpy(), tv.grad.numpy()


def _loss(o, mean, var, w):
    return float(o @ O.chain(o, mean, var, w)["cbar"])


@pytest.mark.parametrize("name", list(SETS))
def test_gradients_equal_torch_autograd_and_central_differences(name):
    w = SETS[name]
    rng = np.random.default_rng(21 + len(name))
    for T in (1, 4, 17):
        o, mean, var = _chain_data(rng, T, len(w))
        r = O.chain(o, mean, var, w)
        tgm, tgv = _torch_grads(o, mean, var, w)
        # the scale floor |o|: with T <= 2 H only the static window is left and dL/dvar is 0 up to rounding
        for got, want in ((r["g_mean"], tgm), (r["g_var"], tgv)):
            assert np.abs(got - want).max() <= 1e-10 * max(np.abs(o).max(), np.abs(want).max()), (T, name)
        h = 1e-6
        for arr, g in ((mean, r["g_mean"]), (var, r["g_var"])):
            for idx in list(np.ndindex(arr.shape))[:: max(1, arr.size // 5)]:
                a1, a2 = arr.copy(), arr.copy()
                a1[idx] += h
                a2[idx] -= h
                args1 = [a1 if arr is a else a for a in (mean, var)]
                args2 = [a2 if arr is a else a for a in (mean, var)]
                fd = (_loss(o, *args1, w) - _loss(o, *args2, w)) / (2 * h)
                assert abs(fd - g[idx]) <= 1e-6 * max(1.0, abs(g[idx])), (idx, fd, g[idx])


@pytest.mark.parametrize("i", range(len(MV.cases())))
def test_oracle_matches_central_differences_of_the_reference(i):
    """The stored differences come from the reference's float64 paramgen.mlpg (oracle/_ref), not the restatement."""
    gold = np.load(os.path.join(ROOT, "tests", "golden", "mlpg_vjp_reference_golden.npz"))
    name, T, sd, var_global = MV.cases()[i]
    m, v, go = (gold["%s_%d" % (k, i)] for k in ("means", "variances", "go"))
    for a, b in zip((m, v, go), MV.inputs(i)):
        assert np.array_equal(a, b)
    gm, gv = O.vjp(m, v, MV.WINDOW_SETS[name], go)
    assert gv.shape == v.shape
    # scale floored by the mean gradient's: at T <= 2 H dL/dvar is 0 and the differences are rounding
    scale = np.abs(gold["g_means_%d" % i]).max()
    for got, want in ((gm, gold["g_means_%d" % i]), (gv, gold["g_variances_%d" % i])):
        assert np.abs(got - want).max() <= 1e-6 * max(scale, np.abs(want).max()), (i, np.abs(got - want).max())


@pytest.mark.parametrize("name", list(SETS))
def test_banded_path_equals_the_dense_one(name):
    w = SETS[name]
    rng = np.random.default_rng(27 + len(name))
    for T in (1, 3, 9, 60):
        o, mean, var = _chain_data(rng, T, len(w), ratio=1e4 if T == 60 else 1.0)
        d, b = O.chain(o, mean, var, w), O.chain(o, mean, var, w, banded=True)
        for k in ("cbar", "g", "g_mean", "g_var"):
            assert np.abs(d[k] - b[k]).max() <= 1e-10 * max(np.abs(o).max(), np.abs(d[k]).max()), (T, k)


@pytest.mark.parametrize("name", list(SETS))
def test_trajectory_is_homogeneous_of_degree_zero_in_the_precisions(name):
    """Scaling every variance of a chain leaves cbar unchanged, so sum_{t,w} var dL/dvar = 0."""
    w = SETS[name]
    rng = np.random.default_rng(31 + len(name))
    for T in (2, 17, 40):
        o, mean, var = _chain_data(rng, T, len(w))
        r = O.chain(o, mean, var, w)
        # at T <= 2 H every term is rounding: the mean gradient's size floors the scale
        scale = np.abs(var * r["g_var"]).sum() + np.abs(r["g_mean"]).sum()
        assert abs(np.sum(var * r["g_var"])) <= 1e-12 * scale, (T, name)


def test_static_window_alone_passes_the_gradient_through():
    w = [(0, 0, np.array([1.0]))]
    o, mean, var = _chain_data(np.random.default_rng(9), 25, 1)
    r = O.chain(o, mean, var, w)
    assert np.abs(r["g_mean"][:, 0] - o).max() <= 1e-15 * np.abs(o).max()
    assert np.abs(r["g_var"]).max() <= 1e-15 * np.abs(o).max()


def test_edge_frames_have_zero_gradients():
    w = SETS["hw2"]
    o, mean, var = _chain_data(np.random.default_rng(5), 30, len(w))
    r = O.chain(o, mean, var, w)
    assert np.all(r["g_mean"][:2, 1:] == 0) and np.all(r["g_mean"][-2:, 1:] == 0)
    assert np.all(r["g_var"][:2, 1:] == 0) and np.all(r["g_var"][-2:, 1:] == 0)


def test_layout_oracle_passes_copied_columns_through():
    w = MG.WINDOWS
    streams = [(0, 60), (180, 1), (183, 1, "copy"), (184, 1)]
    rng = np.random.default_rng(2)
    T = 12
    m, v, go = rng.standard_normal((T, 187)), rng.random((T, 187)) + 0.5, rng.standard_normal((T, 63))
    gm, gv = O.vjp(m, v, w, go, streams)
    assert np.array_equal(gm[:, 183], go[:, 61]) and not gv[:, 183].any()
    gm1, gv1 = O.vjp(m, v[0], w, go, streams)
    assert gv1.shape == (187,) and gv1[183] == 0


# ---- argument errors -------------------------------------------------------------------------------------------
def test_argument_errors_raise_before_any_launch(monkeypatch):
    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200 import paramgen as G

    def no_launch(*a, **k):
        raise AssertionError("launched")
    monkeypatch.setattr(G, "_mlpg_vjp_device", no_launch)
    rng = np.random.default_rng(0)
    w = MG.WINDOWS
    m, v, go = rng.standard_normal((30, 9)), rng.random((30, 9)) + 0.5, rng.standard_normal((30, 3))
    f = G.mlpg_vjp_batch
    bad = [
        lambda: f(m, v, w, go.astype(np.float32), lengths=[30]),
        lambda: f(m.astype(np.float32), v, w, go, lengths=[30]),
        lambda: f(m.astype(np.int64), v.astype(np.int64), w, go.astype(np.int64), lengths=[30]),
        lambda: f(m, v, w, go[:, :2], lengths=[30]),
        lambda: f(m, v, w, go[:29], lengths=[30]),
        lambda: f(m, v[:, :8], w, go, lengths=[30]),
        lambda: f(m, v[0, :8], w, go, lengths=[30]),
        lambda: f(m, v, w, go, lengths=[20]),
        lambda: f(m, v, w, go, lengths=[20, 20]),
        lambda: f(m, v, w, go, layout=G.merlin_layout()),
        lambda: f(m, v, [], go, lengths=[30]),
        lambda: f(m, v, [(0, 0, np.array([1.0]))] * (_lib.NNK_MAX_WIN + 1), go, lengths=[30]),
        lambda: f(m, v, [(0, _lib.NNK_MAX_HALF + 1, np.ones(_lib.NNK_MAX_HALF + 2))], go, lengths=[30]),
        lambda: f(m[None], v[None], w, go),
        lambda: f(m[None], v[None], w, go, lengths=[30]),
        lambda: f(m[None], v[None], w, go[None], lengths=[31]),
        lambda: f(m[None, None], v, w, go, lengths=[30]),
    ]
    for call in bad:
        with pytest.raises(ValueError):
            call()
    import torch

    from nnmnkwii_b200 import autograd as A
    with pytest.raises(ValueError):  # mixed arrays and tensors
        f(torch.from_numpy(m), v, w, go, lengths=[30])
    with pytest.raises(ValueError):  # CPU tensors
        f(*(torch.from_numpy(a) for a in (m, v)), w, torch.from_numpy(go), lengths=[30])
    with pytest.raises(ValueError):  # the autograd function takes CUDA tensors only
        A.mlpg_with_variances(torch.from_numpy(m).requires_grad_(), torch.from_numpy(v), w)


# ---- the C entry point ------------------------------------------------------------------------------------
def test_c_argument_checks():
    from nnmnkwii_b200 import _lib
    fn = _lib.lib.nnk_mlpg_vjp
    a, t = _lib.NnkMlpgArgs(), _lib.NnkMlpgVjp()
    assert fn(None, ctypes.byref(t), None) == _lib.NNK_ERR_ARG
    assert fn(ctypes.byref(a), None, None) == _lib.NNK_ERR_ARG
    a.dtype = 7
    assert fn(ctypes.byref(a), ctypes.byref(t), None) == _lib.NNK_ERR_ARG
    a.dtype = _lib.NNK_F64
    assert fn(ctypes.byref(a), ctypes.byref(t), None) == _lib.NNK_OK  # empty batch
    t.gm_ld = -1
    assert fn(ctypes.byref(a), ctypes.byref(t), None) == _lib.NNK_ERR_ARG
    t.gm_ld = 0
    a.n_utt, a.n_chain, a.max_T = 1, 1, 5
    assert fn(ctypes.byref(a), ctypes.byref(t), None) == _lib.NNK_ERR_ARG  # NULL pointers
    a.n_chain = 1 << 21
    assert fn(ctypes.byref(a), ctypes.byref(t), None) == _lib.NNK_ERR_ARG
    w = _lib.make_windows(MG.WINDOWS)
    S = 2
    assert _lib.lib.nnk_mlpg_vjp_workspace_bytes(3, 33, 10, ctypes.byref(w)) == 3 * 2 * 10 * (S + 2) * 32 * 8
