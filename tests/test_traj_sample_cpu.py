"""Sampling from the trajectory model without a GPU: the float64 restatement (tests/traj_sample_oracle.py) -- its
Philox against the published known answers, its banded recurrence against the dense Cholesky form, its samples
against the model's mean and covariance, and its normals against N(0, 1); the argument errors of
paramgen.trajectory_sample_batch, raised before any launch, and those of the C entry point."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
from scipy import stats

import traj_sample_oracle as O
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
    return mean, var


# ---- the generator ---------------------------------------------------------------------------------------------
def test_philox_known_answers():
    """Random123's known-answer vectors for philox4x32-10."""
    ones = 0xFFFFFFFF
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((ones,) * 4, (ones, ones), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for c, k, want in cases:
        assert tuple(int(r) for r in O.philox(*c, *k)) == want


def test_normals_follow_the_counter_layout():
    """Frame t of sample s of column c uses counter (t >> 1, c, s, key): even frames the cosine, odd the sine."""
    seed, key = (7 << 32) | 3, 11
    z = O.normals(seed, key, 3, 9, 5)
    for s in range(3):
        for t in range(9):
            zc, zs = O.pair_normals(seed, key, s, t >> 1, 5)
            assert z[s, t] == (zs if t & 1 else zc)
    r = O.philox(4, 5, 2, key, 3, 7)
    nu = (int(r[0]) >> 6) * 2 ** 26 + (int(r[1]) >> 6)
    nv = (int(r[2]) >> 6) * 2 ** 26 + (int(r[3]) >> 6)
    R = np.sqrt(-2.0 * np.log((nu + 0.5) * 2.0 ** -52))
    assert z[2, 8] == R * np.cos(2.0 * np.pi * nv * 2.0 ** -52)


# ---- the recurrence ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SETS))
def test_banded_recurrence_equals_the_dense_form(name):
    w = SETS[name]
    rng = np.random.default_rng(17 + len(name))
    for T in (1, 2, 5, 13, 60):
        mean, var = _chain_data(rng, T, len(w))
        z = O.normals(5, 2, 3, T, 1)
        for scale in (0.0, 0.3, 1.0):
            b = O.chain(mean, var, w, z, scale)
            d = O.chain(mean, var, w, z, scale, banded=False)
            assert np.abs(b - d).max() <= 1e-12 * max(1.0, np.abs(d).max()), (T, scale)


def test_samples_have_the_model_mean_and_covariance():
    """4096 samples of one chain: the mean within 5 standard errors of cbar at every frame, and every entry of the
    covariance band within 5 standard errors of the band of inv(P)."""
    w = SETS["hw2"]
    T, N = 14, 4096
    mean, var = _chain_data(np.random.default_rng(21), T, len(w))
    z = O.normals(1234, 0, N, T, 0)
    x = O.chain(mean, var, w, z)
    cbar, cov = O.cbar_and_cov(mean, var, w)
    se = np.sqrt(np.diag(cov) / N)
    assert np.all(np.abs(x.mean(0) - cbar) <= 5 * se)
    xc = x - cbar  # the true mean: the standard error below is that of a known-mean covariance
    emp = xc.T @ xc / N
    S = 4
    for lag in range(S + 1):
        i = np.arange(T - lag)
        j = i + lag
        se = np.sqrt((cov[i, i] * cov[j, j] + cov[i, j] ** 2) / N)
        assert np.all(np.abs(emp[i, j] - cov[i, j]) <= 5 * se), lag


def test_normals_are_standard_normal():
    """2^21 normals over varying frame pairs, columns, samples, keys and seeds: mean, variance, skewness and excess
    kurtosis within 5 standard errors, a Kolmogorov-Smirnov p-value above 1e-4, and the two normals of one
    Box-Muller pair uncorrelated within 5 / sqrt(pairs)."""
    rng = np.random.default_rng(99)
    zc, zs = [], []
    for seed in (0, 1, 0xDEADBEEF, (1 << 64) - 1):
        n = 1 << 18
        pair = rng.integers(0, 1 << 20, n, dtype=np.uint64)
        col = rng.integers(0, 256, n, dtype=np.uint64)
        s = rng.integers(0, 64, n, dtype=np.uint64)
        key = rng.integers(0, 1 << 32, n, dtype=np.uint64)
        a, b = O.pair_normals(seed, key, s, pair, col)
        zc.append(a)
        zs.append(b)
    zc, zs = np.concatenate(zc), np.concatenate(zs)
    z = np.concatenate([zc, zs])
    N = z.size
    assert N == 1 << 21
    assert abs(z.mean()) <= 5 / np.sqrt(N)
    assert abs(z.var() - 1.0) <= 5 * np.sqrt(2.0 / N)
    assert abs(stats.skew(z)) <= 5 * np.sqrt(6.0 / N)
    assert abs(stats.kurtosis(z)) <= 5 * np.sqrt(24.0 / N)
    assert stats.kstest(z, "norm").pvalue > 1e-4
    assert abs(np.corrcoef(zc, zs)[0, 1]) <= 5 / np.sqrt(zc.size)


def test_layout_oracle_copies_the_copied_columns():
    w = MG.WINDOWS
    streams = [(0, 60), (180, 1), (183, 1, "copy"), (184, 1)]
    rng = np.random.default_rng(2)
    m, v = rng.standard_normal((12, 187)), rng.random((12, 187)) + 0.5
    y = O.sample(m, v, w, 3, 0, 0, 1.0, streams)
    assert y.shape == (3, 12, 63)
    assert all(np.array_equal(y[s, :, 61], m[:, 183]) for s in range(3))


# ---- argument errors -------------------------------------------------------------------------------------------
def test_argument_errors_raise_before_any_launch(monkeypatch):
    from nnmnkwii_b200 import paramgen as G

    def no_launch(*a, **k):
        raise AssertionError("launched")
    monkeypatch.setattr(G, "_traj_sample_device", no_launch)
    rng = np.random.default_rng(0)
    w = MG.WINDOWS
    m = rng.standard_normal((30, 9))
    v = rng.random((30, 9)) + 0.5
    f = G.trajectory_sample_batch
    bad = [
        lambda: f(m, v, w, n_samples=0, lengths=[30]),
        lambda: f(m, v, w, n_samples=-1, lengths=[30]),
        lambda: f(m, v, w, n_samples=2 ** 31, lengths=[30]),
        lambda: f(m, v, w, n_samples=2.0, lengths=[30]),
        lambda: f(m, v, w, n_samples=True, lengths=[30]),
        lambda: f(m, v, w, seed=-1, lengths=[30]),
        lambda: f(m, v, w, seed=2 ** 64, lengths=[30]),
        lambda: f(m, v, w, seed=1.5, lengths=[30]),
        lambda: f(m, v, w, seed=None, lengths=[30]),
        lambda: f(m, v, w, keys=[0, 1], lengths=[30]),
        lambda: f(m, v, w, keys=[-1], lengths=[30]),
        lambda: f(m, v, w, keys=[2 ** 32], lengths=[30]),
        lambda: f(m, v, w, keys=[1.0], lengths=[30]),
        lambda: f(m, v, w, keys=[[1]], lengths=[30]),
        lambda: f(m, v, w, keys=[1, 2], lengths=[10, 10, 10]),
        lambda: f(m, v, w, scale=-0.1, lengths=[30]),
        lambda: f(m, v, w, scale=float("nan"), lengths=[30]),
        lambda: f(m, v, w, scale=float("inf"), lengths=[30]),
        lambda: f(m, v, w, scale="x", lengths=[30]),
        lambda: f(m, v.astype(np.float32), w, lengths=[30]),
        lambda: f(m.astype(np.int64), v.astype(np.int64), w, lengths=[30]),
        lambda: f(m, v[:, :8], w, lengths=[30]),
        lambda: f(m, v[0, :8], w, lengths=[30]),
        lambda: f(m, v, w, lengths=[20]),
        lambda: f(m, v, w, layout=G.merlin_layout()),
        lambda: f(m, v, [], lengths=[30]),
        lambda: f(m[None], v[None], w),
        lambda: f(m[None], v[None], w, lengths=[31]),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(ValueError):
            call()
    import torch
    with pytest.raises(ValueError):  # mixed arrays and tensors
        f(torch.from_numpy(m), v, w, lengths=[30])
    with pytest.raises(ValueError):  # CPU tensors
        f(torch.from_numpy(m), torch.from_numpy(v), w, lengths=[30])


# ---- the C entry point ------------------------------------------------------------------------------------
def test_c_argument_checks():
    from nnmnkwii_b200 import _lib
    fn = _lib.lib.nnk_mlpg_traj_sample
    a, t = _lib.NnkMlpgArgs(), _lib.NnkTrajSample()
    t.n_samples, t.scale = 1, 1.0
    assert fn(None, ctypes.byref(t), None) == _lib.NNK_ERR_ARG
    assert fn(ctypes.byref(a), None, None) == _lib.NNK_ERR_ARG
    a.dtype = _lib.NNK_F64
    assert fn(ctypes.byref(a), ctypes.byref(t), None) == _lib.NNK_OK  # empty batch
    for field, value in (("n_samples", 0), ("sample_stride", -1), ("scale", -1.0), ("scale", float("nan")),
                         ("scale", float("inf"))):
        bad = _lib.NnkTrajSample()
        ctypes.memmove(ctypes.byref(bad), ctypes.byref(t), ctypes.sizeof(t))
        setattr(bad, field, value)
        assert fn(ctypes.byref(a), ctypes.byref(bad), None) == _lib.NNK_ERR_ARG, field
    a.n_utt, a.n_chain, a.max_T = 1, 1, 5
    assert fn(ctypes.byref(a), ctypes.byref(t), None) == _lib.NNK_ERR_ARG  # NULL pointers
    w = _lib.make_windows(MG.WINDOWS)
    S = 2
    assert _lib.lib.nnk_mlpg_traj_sample_workspace_bytes(3, 33, 10, ctypes.byref(w)) == 3 * 2 * 10 * (S + 2) * 32 * 8
