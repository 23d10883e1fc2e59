"""paramgen.mlpg_vjp_batch and autograd.MLPGWithVariances on the GPU (mlpg_kernel in MODE_VJP, csrc/nnk_mlpg.cu)
against the float64 restatement tests/mlpg_vjp_oracle.py.

Bar: each gradient within 1e-9 of the max-abs of its oracle column (DESIGN.md 3.22)."""
import importlib.util
import os

import numpy as np
import pytest

import mlpg_vjp_oracle as O
import variant_mirror as M
from conftest import ROOT

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location("make_gmm_traj_golden",
                                               os.path.join(ROOT, "tests", "golden", "make_gmm_traj_golden.py"))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
SETS = MG.em_window_sets()
STD = MG.WINDOWS
TOL = 1e-9
MODE_VJP = 7
MERLIN = [(0, 60), (180, 1), (183, 1, "copy"), (184, 1)]


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
    go = rng.standard_normal((n, D_out))
    return m.astype(dtype), v.astype(dtype), go.astype(dtype)


def _dev(m, v, w, go, lens, layout=None):
    """(g_means, g_vars) as NumPy from mlpg_vjp_batch on CUDA tensors."""
    g_m, g_v = _G().mlpg_vjp_batch(_cuda(m), _cuda(v), w, _cuda(go), lengths=lens, layout=layout)
    return g_m.cpu().numpy(), g_v.cpu().numpy()


def _oracle_batch(m, v, w, go, lens, streams=None, banded=False):
    off = np.concatenate([[0], np.cumsum(lens)])
    gms, gvs = [], []
    for a, b in zip(off[:-1], off[1:]):
        gm, gv = O.vjp(m[a:b], v if v.ndim == 1 else v[a:b], w, go[a:b], streams, banded=banded or (b - a) > 60)
        gms.append(gm)
        gvs.append(gv)
    return np.concatenate(gms), (np.sum(gvs, axis=0) if v.ndim == 1 else np.concatenate(gvs))


def _compare(got, want, what, tol=TOL):
    """Each column within tol of its oracle max-abs.  The variance columns' scale is floored by the mean gradient's:
    where only the static window is kept (T <= 2 H, or H = 0) cbar is mu up to rounding and dL/dvar is rounding."""
    mean_scale = np.abs(np.asarray(want[0], np.float64)).max(axis=0)
    for g, r, k in zip(got, want, ("mean", "var")):
        g, r = np.asarray(g, np.float64), np.asarray(r, np.float64)
        scale = np.abs(r).max(axis=0) if r.ndim == 2 else np.abs(r)
        scale = np.maximum(scale, mean_scale if k == "var" else 1e-300)
        err = np.abs(g - r).max(axis=0) if r.ndim == 2 else np.abs(g - r)
        assert np.all(err <= tol * scale), (what, k, (err / scale).max())


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
    rng = np.random.default_rng([len(name), var_global, 7])
    m, v, go = _data(rng, sum(lens), len(w) * sd, sd, var_global=var_global)
    got = _dev(m, v, w, go, lens)
    assert got[0].shape == m.shape and got[1].shape == v.shape
    _compare(got, _oracle_batch(m, v, w, go, lens), (name, var_global))


def test_variance_ratio_1e4():
    sd, lens = 4, [300, 41]
    m, v, go = _data(np.random.default_rng(4), sum(lens), 3 * sd, sd, ratio=1e4, sd=sd)
    _compare(_dev(m, v, STD, go, lens), _oracle_batch(m, v, STD, go, lens), "ratio")
    mg, vg, gog = _data(np.random.default_rng(5), sum(lens), 3 * sd, sd, var_global=True, ratio=1e4, sd=sd)
    _compare(_dev(mg, vg, STD, gog, lens), _oracle_batch(mg, vg, STD, gog, lens), "ratio global")


def test_20000_frames():
    m, v, go = _data(np.random.default_rng(6), 20000, 6, 2)
    _compare(_dev(m, v, STD, go, [20000]), _oracle_batch(m, v, STD, go, [20000], banded=True), "20000")


@pytest.mark.parametrize("padded", [False, True])
def test_merlin_layout(padded):
    G = _G()
    lens = [70, 5, 33]
    m, v, go = _data(np.random.default_rng(7), sum(lens), 187, 63)
    want = _oracle_batch(m, v, STD, go, lens, MERLIN)
    got = _dev(m, v, STD, go, lens, G.merlin_layout())
    _compare(got, want, "merlin")
    assert np.array_equal(got[0][:, 183], go[:, 61]) and not got[1][:, 183].any()
    if padded:
        B, Tm = len(lens), max(lens)
        off = np.concatenate([[0], np.cumsum(lens)])
        pm, pv, pg = (np.full((B, Tm, a.shape[1]), np.nan) for a in (m, v, go))
        for u, T in enumerate(lens):
            pm[u, :T], pv[u, :T], pg[u, :T] = m[off[u]:off[u + 1]], v[off[u]:off[u + 1]], go[off[u]:off[u + 1]]
        pv[np.isnan(pv)] = -1.0
        gp = _dev(pm, pv, STD, pg, lens, G.merlin_layout())
        for k in (0, 1):
            assert gp[k].shape == (B, Tm, 187)
            for u, T in enumerate(lens):
                assert np.array_equal(gp[k][u, :T], got[k][off[u]:off[u + 1]])
                assert not gp[k][u, T:].any()


def test_float32_matches_the_oracle_fed_the_same_tau():
    w = SETS["nw3"]
    lens = [200, 9]
    m, v, go = _data(np.random.default_rng(8), sum(lens), 3 * 5, 5, dtype=np.float32)
    got = _dev(m, v, w, go, lens)
    assert got[0].dtype == np.float32 and got[1].dtype == np.float32
    want = _oracle_batch(m, v, w, go, lens)  # precisions() divides in float32 as the kernel does
    _compare(got, want, "float32", tol=2.0 ** -23)
    mg, vg, gog = _data(np.random.default_rng(9), sum(lens), 3 * 5, 5, dtype=np.float32, var_global=True)
    got = _dev(mg, vg, w, gog, lens)
    assert got[1].dtype == np.float32 and got[1].shape == (15,)
    # (D,): float64 partials summed in float64, then rounded once
    _compare(got, _oracle_batch(mg, vg, w, gog, lens), "float32 global", tol=2.0 ** -23)


# ---- exact equalities ----------------------------------------------------------------------------------------------
def test_repeat_and_alone_are_bit_identical():
    G = _G()
    w = SETS["hw2"]
    lens = [120, 1, 57, 4]
    m, v, go = _data(np.random.default_rng(9), sum(lens), 3 * 7, 7)
    full = _dev(m, v, w, go, lens)
    again = _dev(m, v, w, go, lens)
    for a, b in zip(full, again):
        assert np.array_equal(a, b)
    off = np.concatenate([[0], np.cumsum(lens)])
    for a, b in zip(off[:-1], off[1:]):
        one = _dev(m[a:b], v[a:b], w, go[a:b], [b - a])
        for k in (0, 1):
            assert np.array_equal(one[k], full[k][a:b])
    host = G.mlpg_vjp_batch(m, v, w, go, lengths=lens)
    assert all(isinstance(h, np.ndarray) and np.array_equal(h, f) for h, f in zip(host, full))


def test_workspace_waves_are_bit_identical(monkeypatch):
    from nnmnkwii_b200 import _device, _lib
    lens = [300, 17, 90, 1, 250]
    for var_global in (False, True):
        m, v, go = _data(np.random.default_rng(11), sum(lens), 3 * 40, 40, var_global=var_global)
        one = _dev(m, v, STD, go, lens)
        with monkeypatch.context() as mp:
            mp.setattr(_device, "WORKSPACE_CAP_BYTES", 1)
            c0 = _lib.launch_count()
            waves = _dev(m, v, STD, go, lens)
            assert _lib.launch_count() - c0 == len(lens)
        for a, b in zip(waves, one):
            assert np.array_equal(a, b)


def test_mean_gradient_is_mlpg_grad_batch():
    """mlpg_grad_batch returns float32 (from the staged kernel here); the float64 means part rounds to it."""
    G = _G()
    lens = [400, 31, 2]
    m, v, go = _data(np.random.default_rng(12), sum(lens), 187, 63)
    for var in (v, v[0]):
        gm, _ = _dev(m, var, STD, go, lens, G.merlin_layout())
        ref = G.mlpg_grad_batch(_cuda(var), STD, _cuda(go), lens, layout=G.merlin_layout()).cpu().numpy()
        err = np.abs(gm - ref).max(axis=0)
        assert np.all(err <= 2.0 ** -23 * np.abs(gm).max(axis=0)), err.max()


def test_homogeneity_on_the_device():
    """cbar is homogeneous of degree 0 in the precisions: sum_{t,w} var dL/dvar = 0 per chain."""
    w = SETS["hw2"]
    sd, lens = 6, [500, 77]
    m, v, go = _data(np.random.default_rng(13), sum(lens), 3 * sd, sd)
    _, gv = _dev(m, v, w, go, lens)
    off = np.concatenate([[0], np.cumsum(lens)])
    for a, b in zip(off[:-1], off[1:]):
        for d in range(sd):
            cols = [d, sd + d, 2 * sd + d]
            terms = v[a:b, cols] * gv[a:b, cols]
            assert abs(terms.sum()) <= 1e-12 * np.abs(terms).sum()


def test_gradcheck():
    import torch

    from nnmnkwii_b200 import autograd as A
    rng = np.random.default_rng(14)
    lens = [6, 4]
    for var_global in (False, True):
        m, v, _ = _data(rng, sum(lens), 6, 2, var_global=var_global)
        args = [_cuda(a).requires_grad_() for a in (m, v)]
        assert torch.autograd.gradcheck(lambda a, b: A.mlpg_with_variances(a, b, STD, lens), args, eps=1e-6,
                                        atol=1e-7, rtol=1e-5)
        one = [_cuda(m[:6]).requires_grad_(), _cuda(v if var_global else v[:6]).requires_grad_()]
        assert torch.autograd.gradcheck(lambda a, b: A.mlpg_with_variances(a, b, STD), one, eps=1e-6, atol=1e-7,
                                        rtol=1e-5)
        pm = torch.zeros((2, 6, 6), dtype=torch.float64, device="cuda")
        pm[0, :6], pm[1, :4] = _cuda(m[:6]), _cuda(m[6:])
        if var_global:
            pv = _cuda(v)
        else:
            pv = torch.ones((2, 6, 6), dtype=torch.float64, device="cuda")
            pv[0, :6], pv[1, :4] = _cuda(v[:6]), _cuda(v[6:])
        pargs = [pm.requires_grad_(), pv.requires_grad_()]
        assert torch.autograd.gradcheck(lambda a, b: A.mlpg_with_variances(a, b, STD, lens), pargs, eps=1e-6,
                                        atol=1e-7, rtol=1e-5)
        A.mlpg_with_variances(*pargs, STD, lens).sum().backward()
        assert not pargs[0].grad[1, 4:].any()
        if not var_global:
            assert not pargs[1].grad[1, 4:].any()


def test_autograd_forward_is_mlpg_batch_and_expand_gets_frame_gradients():
    import torch

    from nnmnkwii_b200 import autograd as A
    G = _G()
    m, v, go = _data(np.random.default_rng(15), 90, 9, 3, dtype=np.float32, var_global=True)
    vf = np.ascontiguousarray(np.broadcast_to(v, (90, 9)))
    mt, vt = _cuda(m).requires_grad_(), _cuda(v).requires_grad_()
    y = A.mlpg_with_variances(mt, vt.expand(90, 9), STD)
    assert y.dtype == torch.float32 and torch.equal(y.detach(), G.mlpg_batch(_cuda(m), _cuda(vf), STD))
    y.backward(_cuda(go))
    gm, gv = _dev(m, vf, STD, go, [90])
    assert np.array_equal(mt.grad.cpu().numpy(), gm)
    want = gv.astype(np.float64).sum(axis=0)  # autograd's expand backward sums the per-frame gradients
    assert np.all(np.abs(vt.grad.cpu().numpy() - want) <= 1e-5 * np.abs(gv).sum(axis=0))
    # a real (D,) tensor takes the per-utterance partials: the same gradient up to float32 summation
    vt2 = _cuda(v).requires_grad_()
    A.mlpg_with_variances(_cuda(m), vt2, STD).backward(_cuda(go))
    assert np.all(np.abs(vt2.grad.cpu().numpy() - want) <= 1e-5 * np.abs(gv).sum(axis=0))


# ---- kernels, launches and errors ----------------------------------------------------------------------------------
SETS_K = dict(SETS, static=[(0, 0, np.array([1.0]))])
# window set -> (NW, L, U, PF) of the instance that serves it; "static" is the static window alone (instance 0)
INST = {"static": (1, 0, 0, 4), "nw3": (3, 1, 1, 4), "hw2": (3, 2, 2, 2), "hw4": (4, 4, 4, 2)}


def launch(kind, name, dt):
    import torch
    w = SETS_K[name]
    m, v, go = _data(np.random.default_rng(1), 40, len(w) * 3, 3, dtype=np.float32 if dt == "f32" else np.float64)
    _dev(m, v, w, go, [30, 10])
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def kernels():
    cases = [(["vjp", n, dt], r"\bmlpg_(fwd_as_)?kernel<") for n in INST for dt in ("f32", "f64")]
    res = M.profiled_in_child("test_mlpg_vjp_gpu", "launch", cases, repeats=True)
    out = {}
    for (case, _), (names, err) in zip(cases, res):
        assert err == "None", (case, err)
        out[tuple(case[1:])] = names
    return out


@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("name", list(INST))
def test_every_instance_runs_by_name(name, dt, kernels):
    from nnmnkwii_b200 import _lib
    NW, L, U, PF = INST[name]
    assert M.pick_instance(SETS_K[name]) == (NW, L, U)
    tin = "float" if dt == "f32" else "double"
    want = "mlpg_kernel<%s, %d, %d, %d, %d, %d>" % (tin, NW, L, U, MODE_VJP, PF)
    names = kernels[(name, dt)]
    assert len(names) == 1 and want in names[0], (want, names)
    w = SETS_K[name]
    m, v, go = _data(np.random.default_rng(1), 40, len(w) * 3, 3)
    c0 = _lib.launch_count()
    _dev(m, v, w, go, [30, 10])
    assert _lib.launch_count() - c0 == 1


def test_non_positive_variance_raises():
    """Frame 20 of utterance 0, static dimension 1: precision -100 on every window makes the pivot negative; the
    error is the one mlpg_batch raises."""
    G = _G()
    m, v, go = _data(np.random.default_rng(16), 50, 9, 3)
    v[20, [1, 4, 7]] = -0.01
    with pytest.raises(np.linalg.LinAlgError) as e_fwd:
        G.mlpg_batch(m, v, STD, lengths=[30, 20])
    with pytest.raises(np.linalg.LinAlgError) as e_vjp:
        G.mlpg_vjp_batch(m, v, STD, go, lengths=[30, 20])
    assert str(e_vjp.value) == str(e_fwd.value)
