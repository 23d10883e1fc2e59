"""paramgen.trajectory_sample_batch on the GPU (mlpg_kernel in MODE_SAMPLE, csrc/nnk_mlpg.cu) against the float64
restatement tests/traj_sample_oracle.py fed the same seed and keys, against the model's mean and covariance, and
against itself bit for bit.

Bar: float64 samples within 1e-10 of the max-abs of their oracle column (DESIGN.md 3.21)."""
import importlib.util
import os

import numpy as np
import pytest

import traj_sample_oracle as O
import variant_mirror as M
from conftest import ROOT

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location("make_gmm_traj_golden",
                                               os.path.join(ROOT, "tests", "golden", "make_gmm_traj_golden.py"))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
SETS = MG.em_window_sets()
STD = MG.WINDOWS
MERLIN = [(0, 60), (180, 1), (183, 1, "copy"), (184, 1)]
TOL = 1e-10
MODE_SAMPLE = 6


def _G():
    from nnmnkwii_b200 import paramgen as G
    return G


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _data(rng, n, D, dtype=np.float64, var_global=False, ratio=1.0, nw=3, sd=None):
    m = np.cumsum(rng.standard_normal((n, D)), axis=0) * 0.05 + rng.standard_normal((n, D)) * 0.3
    v = (rng.random(D) + 0.5) if var_global else (rng.random((n, D)) + 0.5)
    if ratio != 1.0 and sd:
        v[..., sd:nw * sd] /= ratio
    return m.astype(dtype), v.astype(dtype)


def _dev(m, v, w, lens, **kw):
    """Samples of CUDA copies of m, v as NumPy."""
    return _G().trajectory_sample_batch(_cuda(m), _cuda(v), w, lengths=lens, **kw).cpu().numpy()


def _oracle(m, v, w, lens, n, seed, keys=None, scale=1.0, streams=None):
    off = np.concatenate([[0], np.cumsum(lens)])
    parts = [O.sample(m[a:b], v if v.ndim == 1 else v[a:b], w, n, seed, u if keys is None else keys[u], scale,
                      streams) for u, (a, b) in enumerate(zip(off[:-1], off[1:]))]
    return np.concatenate(parts, axis=1)


def _compare(got, want, what, tol=TOL):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    scale = np.abs(want).reshape(-1, want.shape[-1]).max(axis=0)
    err = np.abs(got - want).reshape(-1, want.shape[-1]).max(axis=0)
    assert np.all(err <= tol * np.maximum(scale, 1e-300)), (what, (err / np.maximum(scale, 1e-300)).max())


def _half(w):
    return max(max(l, u) for l, u, _ in w)


# ---- agreement with the oracle -------------------------------------------------------------------------------------
@pytest.mark.parametrize("var_global", [False, True], ids=["var_frame", "var_global"])
@pytest.mark.parametrize("name", list(SETS))
def test_every_window_set_and_edge_length(name, var_global):
    w = SETS[name]
    H = _half(w)
    lens = sorted({1, 2, max(H, 1), 2 * H + 1, 31, 33, 1000})
    sd = 3
    m, v = _data(np.random.default_rng([len(name), var_global]), sum(lens), len(w) * sd, var_global=var_global)
    got = _dev(m, v, w, lens, n_samples=3, seed=12345)
    _compare(got, _oracle(m, v, w, lens, 3, 12345), (name, var_global))


@pytest.mark.parametrize("n_samples", [1, 3, 16])
@pytest.mark.parametrize("scale", [0.0, 0.3, 1.0])
def test_scale_and_sample_count(scale, n_samples):
    lens = [40, 7, 64]
    m, v = _data(np.random.default_rng(3), sum(lens), 12)
    keys = [9, 2 ** 32 - 1, 0]
    got = _dev(m, v, STD, lens, n_samples=n_samples, seed=2 ** 64 - 5, keys=keys, scale=scale)
    _compare(got, _oracle(m, v, STD, lens, n_samples, 2 ** 64 - 5, keys, scale), (scale, n_samples))


def test_variance_ratio_1e4():
    sd, lens = 4, [300, 41]
    m, v = _data(np.random.default_rng(4), sum(lens), 3 * sd, ratio=1e4, sd=sd)
    _compare(_dev(m, v, STD, lens, n_samples=2, seed=4), _oracle(m, v, STD, lens, 2, 4), "ratio")
    mg, vg = _data(np.random.default_rng(5), sum(lens), 3 * sd, var_global=True, ratio=1e4, sd=sd)
    _compare(_dev(mg, vg, STD, lens, n_samples=2, seed=5), _oracle(mg, vg, STD, lens, 2, 5), "ratio global")


def test_20000_frames():
    m, v = _data(np.random.default_rng(6), 20000, 6)
    _compare(_dev(m, v, STD, [20000], n_samples=2, seed=6), _oracle(m, v, STD, [20000], 2, 6), "20000")


@pytest.mark.parametrize("padded", [False, True])
def test_merlin_layout(padded):
    import torch
    G = _G()
    lens = [70, 5, 33]
    m, v = _data(np.random.default_rng(7), sum(lens), 187)
    got = _dev(m, v, STD, lens, layout=G.merlin_layout(), n_samples=3, seed=7)
    _compare(got, _oracle(m, v, STD, lens, 3, 7, streams=MERLIN), "merlin")
    for s in range(3):
        assert np.array_equal(got[s, :, 61], m[:, 183])  # vuv copied unchanged into every sample
    if padded:
        B, Tm = len(lens), max(lens)
        off = np.concatenate([[0], np.cumsum(lens)])
        pm, pv = np.full((B, Tm, 187), np.nan), np.full((B, Tm, 187), -1.0)
        for u, T in enumerate(lens):
            pm[u, :T], pv[u, :T] = m[off[u]:off[u + 1]], v[off[u]:off[u + 1]]
        gp = G.trajectory_sample_batch(_cuda(pm), _cuda(pv), STD, n_samples=3, seed=7, lengths=lens,
                                       layout=G.merlin_layout())
        assert gp.is_cuda and gp.shape == (3, B, Tm, 63)
        gp = gp.cpu().numpy()
        for u, T in enumerate(lens):
            assert np.array_equal(gp[:, u, :T], got[:, off[u]:off[u + 1]])
            assert not gp[:, u, T:].any()
        assert torch.equal(G.trajectory_sample_batch(_cuda(pm), _cuda(pv), STD, n_samples=3, seed=7,
                                                     lengths=torch.tensor(lens), layout=G.merlin_layout()).cpu(),
                           torch.from_numpy(gp))


def test_float32_matches_the_oracle_fed_the_same_tau():
    lens = [200, 9]
    m, v = _data(np.random.default_rng(8), sum(lens), 15, dtype=np.float32)
    got = _G().trajectory_sample_batch(m, v, SETS["nw3"], n_samples=4, seed=8, lengths=lens)
    assert isinstance(got, np.ndarray) and got.dtype == np.float32
    want = _oracle(m, v, SETS["nw3"], lens, 4, 8)  # precisions() divides in float32 as the kernel does
    _compare(got, want, "float32", tol=2.0 ** -23)


# ---- against the model, independent of the oracle's formula --------------------------------------------------------
def _dense_model(mean, var, windows):
    """cbar and inv(P) of one chain from dense window matrices and the edge rule of mlpg."""
    T = mean.shape[0]
    H = _half(windows)
    P, b = np.zeros((T, T)), np.zeros(T)
    for i, (l, u, coef) in enumerate(windows):
        W = np.zeros((T, T))
        for t in range(T):
            for k in range(-l, u + 1):
                if 0 <= t + k < T:
                    W[t, t + k] = coef[l + k]
        tau = 1.0 / var[:, i]
        if i > 0:
            tau[:H] = 0.0
            tau[T - H:] = 0.0
        P += W.T @ (tau[:, None] * W)
        b += W.T @ (tau * mean[:, i])
    return np.linalg.solve(P, b), np.linalg.inv(P)


def test_samples_have_the_model_mean_and_covariance():
    T, sd, N = 48, 4, 16384
    m, v = _data(np.random.default_rng(9), T, 3 * sd)
    x = _dev(m, v, STD, [T], n_samples=N, seed=99)
    for d in range(sd):
        cols = [d, sd + d, 2 * sd + d]
        cbar, cov = _dense_model(m[:, cols], v[:, cols], STD)
        xd = x[:, :, d]
        assert np.all(np.abs(xd.mean(0) - cbar) <= 5 * np.sqrt(np.diag(cov) / N)), d
        xc = xd - cbar
        emp = xc.T @ xc / N
        for lag in range(5):
            i = np.arange(T - lag)
            j = i + lag
            se = np.sqrt((cov[i, i] * cov[j, j] + cov[i, j] ** 2) / N)
            assert np.all(np.abs(emp[i, j] - cov[i, j]) <= 5 * se), (d, lag)


# ---- exact equalities ----------------------------------------------------------------------------------------------
def test_batch_alone_shuffled_repeat_and_prefix_are_bit_identical():
    G = _G()
    w = SETS["hw2"]
    lens = [120, 1, 57, 4]
    m, v = _data(np.random.default_rng(10), sum(lens), 21)
    full = _dev(m, v, w, lens, n_samples=16, seed=3)
    assert np.array_equal(_dev(m, v, w, lens, n_samples=16, seed=3), full)
    off = np.concatenate([[0], np.cumsum(lens)])
    for u, (a, b) in enumerate(zip(off[:-1], off[1:])):
        assert np.array_equal(_dev(m[a:b], v[a:b], w, [b - a], n_samples=16, seed=3, keys=[u]), full[:, a:b])
    for k in (1, 3, 7):
        assert np.array_equal(_dev(m, v, w, lens, n_samples=k, seed=3), full[:k])
    perm = [2, 0, 3, 1]
    pm = np.concatenate([m[off[u]:off[u + 1]] for u in perm])
    pv = np.concatenate([v[off[u]:off[u + 1]] for u in perm])
    shuf = _dev(pm, pv, w, [lens[u] for u in perm], n_samples=16, seed=3, keys=perm)
    assert np.array_equal(shuf, np.concatenate([full[:, off[u]:off[u + 1]] for u in perm], axis=1))
    one = G.trajectory_sample(m[:120], v[:120], w, n_samples=2, seed=3)
    assert isinstance(one, np.ndarray) and one.shape == (2, 120, 7) and np.array_equal(one, full[:2, :120])


def test_workspace_waves_are_bit_identical(monkeypatch):
    from nnmnkwii_b200 import _device, _lib
    lens = [300, 17, 90, 1, 250]
    m, v = _data(np.random.default_rng(11), sum(lens), 3 * 40)
    one = _dev(m, v, STD, lens, n_samples=3, seed=11)
    monkeypatch.setattr(_device, "WORKSPACE_CAP_BYTES", 1)
    c0 = _lib.launch_count()
    waves = _dev(m, v, STD, lens, n_samples=3, seed=11)
    assert _lib.launch_count() - c0 == len(lens)
    assert np.array_equal(waves, one)


@pytest.mark.parametrize("name", list(SETS))
def test_scale_zero_is_mlpg_batch(name):
    """Instance 3 (half-width 3 or 4, or four windows): mlpg_batch also runs mlpg_kernel, and the samples are its
    trajectory bit for bit.  Elsewhere mlpg_batch runs the staged kernel: within 1e-12 relative."""
    G = _G()
    w = SETS[name]
    lens = [333, 20, 2]
    m, v = _data(np.random.default_rng(12), sum(lens), len(w) * 5)
    y = G.mlpg_batch(m, v, w, lengths=lens)
    s = G.trajectory_sample_batch(m, v, w, n_samples=2, seed=1, lengths=lens, scale=0.0)
    if M.pick_instance(w) == (4, 4, 4):
        assert np.array_equal(s[0], y) and np.array_equal(s[1], y)
    else:
        assert np.abs(s - y[None]).max() <= 1e-12 * np.abs(y).max()


def test_scale_is_linear():
    lens = [80, 33]
    m, v = _data(np.random.default_rng(13), sum(lens), 12)
    c = _dev(m, v, STD, lens, n_samples=4, seed=5, scale=0.0)
    one = _dev(m, v, STD, lens, n_samples=4, seed=5) - c
    for a in (0.3, 2.5):
        got = _dev(m, v, STD, lens, n_samples=4, seed=5, scale=a) - c
        assert np.abs(got - a * one).max() <= 1e-12 * max(1.0, a) * np.abs(np.concatenate([c, one])).max()


def test_different_seeds_and_keys_give_different_draws():
    lens = [50, 50]
    m, v = _data(np.random.default_rng(14), sum(lens), 9)
    base = _dev(m, v, STD, lens, n_samples=2, seed=1)
    assert not np.any(base[0] == base[1])
    for kw in (dict(seed=2), dict(seed=1 + (1 << 32)), dict(seed=1, keys=[0, 7])):
        other = _dev(m, v, STD, lens, n_samples=2, **kw)
        diff = other != base
        if "keys" in kw:
            assert not diff[:, :50].any() and diff[:, 50:].all()
        else:
            assert diff.all(), kw


# ---- kernels, launches and errors ----------------------------------------------------------------------------------
def launch(kind, name, dt):
    import torch
    w = SETS_K[name]
    m, v = _data(np.random.default_rng(1), 40, len(w) * 3, dtype=np.float32 if dt == "f32" else np.float64)
    _dev(m, v, w, [30, 10], n_samples=3)
    torch.cuda.synchronize()


# window set -> (NW, L, U, PF) of the instance that serves it; "static" is the static window alone (instance 0)
SETS_K = dict(SETS, static=[(0, 0, np.array([1.0]))])
INST = {"static": (1, 0, 0, 4), "nw3": (3, 1, 1, 4), "hw2": (3, 2, 2, 2), "hw4": (4, 4, 4, 2)}


@pytest.fixture(scope="module")
def kernels():
    cases = [(["sample", n, dt], r"\bmlpg_(fwd_as_)?kernel<") for n in INST for dt in ("f32", "f64")]
    res = M.profiled_in_child("test_traj_sample_gpu", "launch", cases, repeats=True)
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
    want = "mlpg_kernel<%s, %d, %d, %d, %d, %d>" % (tin, NW, L, U, MODE_SAMPLE, PF)
    names = kernels[(name, dt)]
    assert len(names) == 1 and want in names[0], (want, names)
    w = SETS_K[name]
    m, v = _data(np.random.default_rng(1), 40, len(w) * 3)
    c0 = _lib.launch_count()
    _dev(m, v, w, [30, 10], n_samples=3)
    assert _lib.launch_count() - c0 == 1


def test_non_positive_variance_raises():
    """Frame 20 of utterance 0, static dimension 1: precision -100 on every window makes the pivot negative; the
    error is the one mlpg_batch raises."""
    G = _G()
    m, v = _data(np.random.default_rng(15), 50, 9)
    v[20, [1, 4, 7]] = -0.01
    with pytest.raises(np.linalg.LinAlgError) as e_fwd:
        G.mlpg_batch(m, v, STD, lengths=[30, 20])
    with pytest.raises(np.linalg.LinAlgError) as e_s:
        G.trajectory_sample_batch(m, v, STD, n_samples=2, lengths=[30, 20])
    assert str(e_s.value) == str(e_fwd.value)
