"""paramgen.trajectory_log_likelihood_batch and autograd.TrajectoryLogLikelihood on the GPU (mlpg_kernel in MODE_TLL /
MODE_TLL_GRAD, csrc/nnk_mlpg.cu) against the float64 restatement tests/traj_ll_oracle.py.

Bars: l within 1e-11 relative, each gradient within 1e-9 of the max-abs of its oracle column (DESIGN.md 3.20)."""
import importlib.util
import os

import numpy as np
import pytest

import traj_ll_oracle as O
import variant_mirror as M
from conftest import ROOT

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location("make_gmm_traj_golden",
                                               os.path.join(ROOT, "tests", "golden", "make_gmm_traj_golden.py"))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
SETS = MG.em_window_sets()
STD = MG.WINDOWS
TOL_LL, TOL_G = 1e-11, 1e-9
MODE_TLL, MODE_TLL_GRAD = 4, 5


def _G():
    from nnmnkwii_b200 import paramgen as G
    return G


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _data(rng, n, D, D_out, dtype=np.float64, var_global=False, ratio=1.0, nw=3, sd=None):
    m = np.cumsum(rng.standard_normal((n, D)), axis=0) * 0.05 + rng.standard_normal((n, D)) * 0.3
    v = (rng.random(D) + 0.5) if var_global else (rng.random((n, D)) + 0.5)
    if ratio != 1.0 and sd:
        v[..., sd:nw * sd] /= ratio
    x = np.cumsum(rng.standard_normal((n, D_out)), axis=0) * 0.05 + rng.standard_normal((n, D_out)) * 0.2
    return x.astype(dtype), m.astype(dtype), v.astype(dtype)


def _device_grads(x, m, v, w, lens, layout=None, grad=True):
    """(ll (n_utt, D_out), g_m, g_v, g_x) as NumPy, straight from one launch."""
    G = _G()
    xt, mt, vt = _cuda(x), _cuda(m), _cuda(v)
    layout, padded, _ = G._traj_ll_check(xt, mt, vt, w, lens, None, layout)
    ll, _, grads = G._traj_ll_device(xt, mt, vt, w, lens, None, layout, padded, grad)
    out = G._traj_ll_scatter(ll, layout).cpu().numpy()
    return (out,) + (tuple(g.cpu().numpy() for g in grads) if grads else ())


def _compare(got, want, what):
    ll, gm, gv, gx = got
    rl, rgm, rgv, rgx = want
    assert np.all(np.abs(ll - rl) <= TOL_LL * np.maximum(1.0, np.abs(rl))), (what, np.abs(ll - rl).max())
    for g, r, k in ((gm, rgm, "mean"), (gv, rgv, "var"), (gx, rgx, "x")):
        g, r = np.asarray(g, np.float64), np.asarray(r, np.float64)
        scale = np.abs(r).max(axis=0) if r.ndim == 2 else np.abs(r)
        err = np.abs(g - r).max(axis=0) if r.ndim == 2 else np.abs(g - r)
        assert np.all(err <= TOL_G * np.maximum(scale, 1e-300)), (what, k, (err / np.maximum(scale, 1e-300)).max())


def _oracle_batch(x, m, v, w, lens, streams=None, banded=False):
    off = np.concatenate([[0], np.cumsum(lens)])
    lls, gms, gvs, gxs = [], [], [], []
    for a, b in zip(off[:-1], off[1:]):
        ll, gm, gv, gx = O.log_likelihood(x[a:b], m[a:b], v if v.ndim == 1 else v[a:b], w, streams,
                                          banded=banded or (b - a) > 60)
        lls.append(ll); gms.append(gm); gvs.append(gv); gxs.append(gx)
    gv = np.stack(gvs) if v.ndim == 1 else np.concatenate(gvs)
    return np.stack(lls), np.concatenate(gms), gv, np.concatenate(gxs)


def _half(w):
    return max(max(l, u) for l, u, _ in w)


# ---- agreement with the oracle -------------------------------------------------------------------------------------
@pytest.mark.parametrize("var_global", [False, True], ids=["var_frame", "var_global"])
@pytest.mark.parametrize("name", list(SETS))
def test_every_window_set_and_edge_length(name, var_global):
    w = SETS[name]
    H = _half(w)
    lens = sorted({1, 2, max(H, 1), 2 * H + 1, 31, 33, 1000})
    sd = 5
    rng = np.random.default_rng([len(name), var_global])
    x, m, v = _data(rng, sum(lens), len(w) * sd, sd, var_global=var_global)
    got = _device_grads(x, m, v, w, lens)
    want = _oracle_batch(x, m, v, w, lens)
    # (D,) variances: the device's per-utterance partials against the oracle's per-utterance sums
    _compare(got, want, (name, var_global))


def test_variance_ratio_1e4():
    w = STD
    sd, lens = 4, [300, 41]
    x, m, v = _data(np.random.default_rng(4), sum(lens), 3 * sd, sd, ratio=1e4, sd=sd)
    _compare(_device_grads(x, m, v, w, lens), _oracle_batch(x, m, v, w, lens), "ratio")
    xg, mg, vg = _data(np.random.default_rng(5), sum(lens), 3 * sd, sd, var_global=True, ratio=1e4, sd=sd)
    _compare(_device_grads(xg, mg, vg, w, lens), _oracle_batch(xg, mg, vg, w, lens), "ratio global")


def test_20000_frames():
    w = STD
    x, m, v = _data(np.random.default_rng(6), 20000, 6, 2)
    _compare(_device_grads(x, m, v, w, [20000]), _oracle_batch(x, m, v, w, [20000], banded=True), "20000")


@pytest.mark.parametrize("padded", [False, True])
def test_merlin_layout(padded):
    import torch
    G = _G()
    lens = [70, 5, 33]
    streams = [(0, 60), (180, 1), (183, 1, "copy"), (184, 1)]
    x, m, v = _data(np.random.default_rng(7), sum(lens), 187, 63)
    want = _oracle_batch(x, m, v, STD, lens, streams)
    got = _device_grads(x, m, v, STD, lens, G.merlin_layout())
    _compare(got, want, "merlin")
    assert np.all(got[0][:, 61] == 0) and not got[1][:, 183].any() and not got[3][:, 61].any()
    if padded:
        B, Tm = len(lens), max(lens)
        off = np.concatenate([[0], np.cumsum(lens)])
        px, pm, pv = (np.full((B, Tm, a.shape[1]), np.nan) for a in (x, m, v))
        for u, T in enumerate(lens):
            px[u, :T], pm[u, :T], pv[u, :T] = x[off[u]:off[u + 1]], m[off[u]:off[u + 1]], v[off[u]:off[u + 1]]
        pv[np.isnan(pv)] = -1.0
        gp = _device_grads(px, pm, pv, STD, lens, G.merlin_layout())
        assert np.array_equal(gp[0], got[0])
        for k in (1, 2, 3):
            for u, T in enumerate(lens):
                assert np.array_equal(gp[k][u, :T], got[k][off[u]:off[u + 1]])
                assert not gp[k][u, T:].any()
        llp = G.trajectory_log_likelihood_batch(_cuda(px), _cuda(pm), _cuda(pv), STD, lengths=lens,
                                                layout=G.merlin_layout())
        assert llp.is_cuda and torch.equal(llp.cpu(), torch.from_numpy(got[0]))


def test_float32_matches_the_oracle_fed_the_same_tau():
    w = SETS["nw3"]
    lens = [200, 9]
    x, m, v = _data(np.random.default_rng(8), sum(lens), 3 * 5, 5, dtype=np.float32)
    got = _device_grads(x, m, v, w, lens)
    assert got[1].dtype == np.float32 and got[3].dtype == np.float32
    want = _oracle_batch(x, m, v, w, lens)  # precisions() divides in float32 as the kernel does
    assert np.all(np.abs(got[0] - want[0]) <= TOL_LL * np.maximum(1.0, np.abs(want[0])))
    for g, r in zip(got[1:], want[1:]):
        assert np.abs(g - r).max() <= 2.0 ** -23 * np.abs(r).max()


# ---- exact equalities ----------------------------------------------------------------------------------------------
def test_batch_alone_repeat_and_ll_only_are_bit_identical():
    G = _G()
    w = SETS["hw2"]
    lens = [120, 1, 57, 4]
    x, m, v = _data(np.random.default_rng(9), sum(lens), 3 * 7, 7)
    full = _device_grads(x, m, v, w, lens)
    again = _device_grads(x, m, v, w, lens)
    for a, b in zip(full, again):
        assert np.array_equal(a, b)
    off = np.concatenate([[0], np.cumsum(lens)])
    for u, (a, b) in enumerate(zip(off[:-1], off[1:])):
        one = _device_grads(x[a:b], m[a:b], v[a:b], w, [b - a])
        assert np.array_equal(one[0][0], full[0][u])
        for k in (1, 2, 3):
            assert np.array_equal(one[k], full[k][a:b])
    ll_only = G.trajectory_log_likelihood_batch(x, m, v, w, lengths=lens)
    assert isinstance(ll_only, np.ndarray) and np.array_equal(ll_only, full[0])
    assert np.array_equal(G.trajectory_log_likelihood(x[:120], m[:120], v[:120], w), full[0][0])


def test_gradients_vanish_at_the_mlpg_trajectory():
    G = _G()
    lens = [90, 31]
    x, m, v = _data(np.random.default_rng(10), sum(lens), 9, 3)
    c = G.mlpg_batch(m, v, STD, lengths=lens)
    ll, gm, gv, gx = _device_grads(c, m, v, STD, lens)
    _, rgm, _, rgx = _device_grads(x, m, v, STD, lens)
    assert np.abs(gm).max() <= 1e-9 * np.abs(rgm).max() and np.abs(gx).max() <= 1e-9 * np.abs(rgx).max()
    assert np.all(ll >= G.trajectory_log_likelihood_batch(x, m, v, STD, lengths=lens))


def test_gradcheck():
    import torch

    from nnmnkwii_b200 import autograd as A
    rng = np.random.default_rng(11)
    lens = [6, 4]
    for var_global in (False, True):
        x, m, v = _data(rng, sum(lens), 6, 2, var_global=var_global)
        args = [_cuda(a).requires_grad_() for a in (x, m, v)]
        assert torch.autograd.gradcheck(lambda a, b, c: A.trajectory_log_likelihood(a, b, c, STD[:2] + STD[2:], lens),
                                        args, eps=1e-6, atol=1e-7, rtol=1e-5)
        pad = [torch.zeros((2, 6, a.shape[1]), dtype=torch.float64, device="cuda") for a in (x, m)]
        for p, a in zip(pad, (x, m)):
            p[0, :6], p[1, :4] = _cuda(a[:6]), _cuda(a[6:])
        pv = _cuda(v) if var_global else torch.ones((2, 6, 6), dtype=torch.float64, device="cuda")
        if not var_global:
            pv[0, :6], pv[1, :4] = _cuda(v[:6]), _cuda(v[6:])
        pargs = [t.requires_grad_() for t in (pad[0], pad[1], pv)]
        out = A.trajectory_log_likelihood(*pargs, STD, lens)
        out.sum().backward()
        assert all(not t.grad[1, 4:].any() for t in pargs[:2])


# ---- kernels, launches and errors ----------------------------------------------------------------------------------
def launch(kind, name, dt, grad):
    import torch
    w = SETS_K[name]
    x, m, v = _data(np.random.default_rng(1), 40, len(w) * 3, 3, dtype=np.float32 if dt == "f32" else np.float64)
    _device_grads(x, m, v, w, [30, 10], grad=grad)
    torch.cuda.synchronize()


# window set -> (NW, L, U, PF) of the instance that serves it; "static" is the static window alone (instance 0)
SETS_K = dict(SETS, static=[(0, 0, np.array([1.0]))])
INST = {"static": (1, 0, 0, 4), "nw3": (3, 1, 1, 4), "hw2": (3, 2, 2, 2), "hw4": (4, 4, 4, 2)}


@pytest.fixture(scope="module")
def kernels():
    cases = [(["tll", n, dt, g], r"\bmlpg_(fwd_as_)?kernel<") for n in INST for dt in ("f32", "f64") for g in (False, True)]
    res = M.profiled_in_child("test_traj_ll_gpu", "launch", cases, repeats=True)
    out = {}
    for (case, _), (names, err) in zip(cases, res):
        assert err == "None", (case, err)
        out[tuple(case[1:])] = names
    return out


@pytest.mark.parametrize("grad", [False, True])
@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("name", list(INST))
def test_every_instance_runs_by_name(name, dt, grad, kernels):
    from nnmnkwii_b200 import _lib
    NW, L, U, PF = INST[name]
    assert M.pick_instance(SETS_K[name]) == (NW, L, U)
    tin = "float" if dt == "f32" else "double"
    want = "mlpg_kernel<%s, %d, %d, %d, %d, %d>" % (tin, NW, L, U, MODE_TLL_GRAD if grad else MODE_TLL, PF)
    names = kernels[(name, dt, grad)]
    assert len(names) == 1 and want in names[0], (want, names)
    w = SETS_K[name]
    x, m, v = _data(np.random.default_rng(1), 40, len(w) * 3, 3)
    c0 = _lib.launch_count()
    _device_grads(x, m, v, w, [30, 10], grad=grad)
    assert _lib.launch_count() - c0 == 1


def test_non_positive_variance_raises():
    """Frame 20 of utterance 0, static dimension 1: precision -100 on every window makes the pivot negative; the
    error is the one mlpg_batch raises."""
    G = _G()
    x, m, v = _data(np.random.default_rng(12), 50, 9, 3)
    v[20, [1, 4, 7]] = -0.01
    with pytest.raises(np.linalg.LinAlgError) as e_fwd:
        G.mlpg_batch(m, v, STD, lengths=[30, 20])
    with pytest.raises(np.linalg.LinAlgError) as e_tll:
        G.trajectory_log_likelihood_batch(x, m, v, STD, lengths=[30, 20])
    assert str(e_tll.value) == str(e_fwd.value)
