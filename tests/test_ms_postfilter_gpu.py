"""Modulation-spectrum post-filter on the GPU: postfilters.modspec_post_filter and modspec_statistics.

* the float64 restatement (oracle/ms_postfilter.py) at every DFT length, T = 1, odd, n - 1 and n, D = 1 and 37:
  float64 within 1e-10, float32 within 1e-4;
* the identities: k = 0 and natural == generated give the input back; with every T = n and k = 1 the output has
  the natural statistics on bins 1 .. n / 2 and the input's on bin 0; an all-zero column comes out zero, and
  every column keeps its bin 0;
* a padded batch with NaN in its padding equals per-utterance calls bit for bit (the statistics: NaN or zero
  padding gives the same bits);
* NumPy in gives NumPy out; a CUDA tensor stays on its device and dtype.

Dirty allocations, workspace reuse and a delayed side stream are checked for these entry points by the
buffers-and-streams catalogue (tests/test_buffers_and_streams_gpu.py), as for every other one."""
import numpy as np
import pytest

import oracle.ms_postfilter as O
from conftest import rel_err

pytestmark = pytest.mark.gpu

NS = (256, 512, 1024, 2048, 4096)
TOL = {np.float64: 1e-10, np.float32: 1e-4}


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _corpus(rng, B, T, D, tilt, gain=10.0):
    """(B, T, D) float64: white noise through 1 + tilt z^-1, a tilted spectrum without zeros (|tilt| < 1).

    The float32 log power of a bin is accurate to about eps * max|Y| / |Y_k|, so the float32 bar holds only where
    no bin's power sits near the float32 rounding of the largest ones; the corpus keeps the spectrum's range
    moderate for that (a random walk would put most of the power in the lowest bins)."""
    w = rng.standard_normal((B, T + 1, D))
    return gain * (w[:, 1:] + tilt * w[:, :-1])


def _check_stats(got, want, dtype, utts, n, bins=slice(None)):
    """Device ``(mean, var)`` against ``want`` on ``bins``.  The float32 variance meets the bar on the bins whose
    power is at least 1e-4 of its column's largest in every utterance of ``utts``, and 10 times the bar on all:
    a bin far below the largest carries a float32 log-power error of about eps * max|Y| / |Y_k|, and the variance
    weighs that error by the bin's distance from the mean."""
    m, v = (_np(a)[bins] for a in got)
    wm, wv = (_np(a)[bins] for a in want)
    tol = TOL[dtype]
    assert rel_err(m, wm) <= tol
    if dtype == np.float64:
        assert rel_err(v, wv) <= tol
        return
    P = np.stack([O.log_ms(_np(u), n)[2] for u in utts])[:, bins]
    ok = (P >= 1e-4 * P.max(axis=1, keepdims=True)).all(axis=0)
    assert ok.mean() > 0.9 and rel_err(v[ok], wv[ok]) <= tol and rel_err(v, wv) <= 10 * tol


def _pair(rng, B, T, D, dtype):
    """(generated, natural) corpora: the generated one is smoother and quieter."""
    return _corpus(rng, B, T, D, 0.7).astype(dtype), _corpus(rng, B, T, D, 0.2, 13.0).astype(dtype)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("n", NS)
def test_parity_with_restatement(n, dtype):
    import torch

    from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
    tol = TOL[dtype]
    rng = np.random.default_rng(n)
    for T in (1, n // 4 + 1, n - 1, n):
        for D in (1, 37):
            tag = (T, D)
            gen, nat = _pair(rng, 4, T, D, dtype)
            G, N = O.statistics(list(gen), n), O.statistics(list(nat), n)
            for corpus, want in ((gen, G), (nat, N)):
                m, v = modspec_statistics(_cuda(corpus), n=n)
                assert m.dtype == v.dtype == torch.float64 and m.shape == v.shape == (n // 2 + 1, D)
                _check_stats((m, v), want, dtype, corpus, n)
            for k in (1.0, 0.4):
                y = modspec_post_filter(_cuda(gen[0]), N, G, k=k, n=n)
                assert y.dtype == getattr(torch, np.dtype(dtype).name) and y.shape == (T, D)
                assert rel_err(_np(y), O.post_filter(gen[0], N, G, k, n)) <= tol, tag + (k,)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("n", [256, 4096])
def test_identities(n, dtype):
    from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
    tol = TOL[dtype]
    rng = np.random.default_rng(n + 1)
    gen, nat = _pair(rng, 6, n, 5, dtype)
    xt = _cuda(gen)
    G, N = modspec_statistics(xt, n=n), modspec_statistics(_cuda(nat), n=n)
    for x in (xt[0], xt[1, :n // 3 + 1]):
        assert rel_err(_np(modspec_post_filter(x, N, G, k=0.0, n=n)), _np(x)) <= tol
        assert rel_err(_np(modspec_post_filter(x, G, G, k=0.6, n=n)), _np(x)) <= tol
        assert rel_err(_np(modspec_post_filter(x, N, G, k=0.5, n=n)), _np(x)) > 1e-2
    # every T = n and k = 1, with the statistics of the input as the generated ones
    out = modspec_post_filter(xt, N, G, k=1.0, n=n)
    got = modspec_statistics(out, n=n)
    _check_stats(got, N, dtype, out, n, slice(1, None))
    _check_stats(got, G, dtype, out, n, slice(0, 1))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_zero_column_and_bin0(dtype):
    import torch

    from nnmnkwii_b200.postfilters import modspec_post_filter
    rng = np.random.default_rng(7)
    for n in NS:
        gen, nat = _pair(rng, 4, n, 4, dtype)
        G, N = O.statistics(list(gen), n), O.statistics(list(nat), n)
        x = gen[0].copy()
        x[:, 2] = 0
        y = modspec_post_filter(_cuda(x), N, G, k=1.0, n=n)
        assert not y[:, 2].any(), n
        # bin 0 of a column is the sum of its n frames
        assert rel_err(_np(y.to(torch.float64).sum(0)), x.astype(np.float64).sum(0)) <= TOL[dtype], n
        assert rel_err(_np(y), x) > 1e-2


# ---- batched == per utterance, whatever the padding ------------------------------------------------------------------
def _same(a, b):
    import torch
    return a.shape == b.shape and torch.equal(torch.view_as_real(a) if a.is_complex() else a,
                                              torch.view_as_real(b) if b.is_complex() else b)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("n", [256, 4096])
def test_batched_equals_per_utterance(n, dtype):
    import torch

    from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
    rng = np.random.default_rng(n + 2)
    T, D = min(n, 300), 7
    lens = np.array([T, 1, 0, T // 2 + 1, 17])
    tdt = getattr(torch, np.dtype(dtype).name)
    gen, nat = _pair(rng, 4, T, D, np.float64)
    G, N = O.statistics(list(gen), n), O.statistics(list(nat), n)
    utts = [_cuda((_corpus(rng, 1, T, D, 0.7)[0, :L]).astype(dtype)) for L in lens]
    want = [modspec_post_filter(u, N, G, k=0.8, n=n) for u in utts]
    padded = torch.full((len(lens), T, D), float("nan"), dtype=tdt, device="cuda")
    for b, u in enumerate(utts):
        padded[b, :len(u)] = u
    live = lens > 0  # the statistics refuse an utterance of no frames
    idx = _cuda(np.flatnonzero(live))
    stats_want = modspec_statistics(torch.nan_to_num(padded.index_select(0, idx), nan=0.0), n=n, lengths=lens[live])

    def run(x):
        return (modspec_post_filter(x, N, G, k=0.8, n=n, lengths=lens),
                modspec_statistics(x.index_select(0, idx), n=n, lengths=lens[live]))

    def check(got):
        y, stats = got
        for b, L in enumerate(lens):
            assert _same(y[b, :L], want[b]) and not y[b, L:].any(), b
        assert _same(stats[0], stats_want[0]) and _same(stats[1], stats_want[1])

    check(run(padded))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_containers(dtype):
    import torch

    from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
    n = 512
    rng = np.random.default_rng(9)
    gen, nat = _pair(rng, 3, 200, 4, dtype)
    Gn, Nn = modspec_statistics(gen, n=n), modspec_statistics(nat, n=n)
    assert all(isinstance(a, np.ndarray) and a.dtype == np.float64 and a.shape == (n // 2 + 1, 4) for a in Gn + Nn)
    Gt, Nt = modspec_statistics(_cuda(gen), n=n), modspec_statistics(_cuda(nat), n=n)
    assert all(t.is_cuda and t.dtype == torch.float64 for t in Gt + Nt)
    assert all(np.array_equal(_np(t), a) for t, a in zip(Gt + Nt, Gn + Nn))
    y = modspec_post_filter(gen[0], Nn, Gn, k=0.7, n=n)
    assert isinstance(y, np.ndarray) and y.dtype == dtype and y.shape == gen[0].shape
    yt = modspec_post_filter(_cuda(gen[0]), Nt, Gt, k=0.7, n=n)
    assert yt.is_cuda and yt.device == torch.device("cuda", torch.cuda.current_device()) and yt.dtype == _cuda(gen).dtype
    assert np.array_equal(_np(yt), y)
    yb = modspec_post_filter(gen, Nn, Gt, k=0.7, n=n, lengths=[200, 200, 200])
    assert isinstance(yb, np.ndarray) and yb.shape == gen.shape and np.array_equal(yb[0], y)
