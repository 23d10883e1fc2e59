"""Segment-level modulation-spectrum post-filter on the GPU: postfilters.modspec_post_filter / modspec_statistics
with ``segment=L`` (csrc/nnk_ms_segment.cu), against the float64 restatement oracle/ms_segment.py.

* every `ms_segment_kernel<T, LOGN, FILTER>` instance (n = 32 .. 512, float32 / float64, statistics / filter),
  checked by kernel name, at L = 4, n / 2 and n, and utterances of 1, H - 1, H and a tile edge +- 1 frames;
* utterances of 10 000 frames, past the utterance level's limit of 4096;
* padded batches of mixed lengths (0 included) with NaN padding equal their utterances run one by one, bit for bit;
* D = 1, a column group +- 1 and 60; NumPy in / NumPy out and CUDA tensors on their device;
* repeated calls give the same bits;
* the identities: k = 0 and equal statistics give the input back.
float64 within 1e-10, float32 within 1e-4 (rel_err).  The float32 statistics meet the bar plus the mean over the
segments of 64 eps max|Y| / |Y_k| (the float32 error of a bin's log power, as in test_ms_postfilter_gpu.py; the
variance weighs it by 2 |s - mean|), and 10 (mean) and 100 (variance) times the bar everywhere: a short segment's
spectrum can pass close to a zero of its z-transform."""
import re

import numpy as np
import pytest

import oracle.ms_segment as O
import variant_mirror as M
from conftest import rel_err

pytestmark = pytest.mark.gpu

NS = (32, 64, 128, 256, 512)
TOL = {np.float64: 1e-10, np.float32: 1e-4}
DT = {"f32": np.float32, "f64": np.float64}
TILE_FRAMES = 256  # SEG_TILE_FRAMES of csrc/nnk_ms_segment.cu
FAMILY = r"\bms_segment_kernel<"


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _tile(L):
    """Frames of one tile of the kernel at segment length L (an even number of hop blocks, at least 2)."""
    H = L // 2
    return max(2, (TILE_FRAMES // H) & ~1) * H


def _corpus(rng, B, T, D, tilt, gain=10.0):
    """(B, T, D) float64: white noise through 1 + tilt z^-1 (a spectrum without deep zeros)."""
    w = rng.standard_normal((B, T + 1, D))
    return gain * (w[:, 1:] + tilt * w[:, :-1])


def _check_stats(got, want, dtype, utts, n, L):
    m, v = (_np(a) for a in got)
    wm, wv = want
    assert m.shape == v.shape == wm.shape
    tol = TOL[dtype]
    if dtype == np.float64:
        assert rel_err(m, wm) <= tol and rel_err(v, wv) <= tol
        return
    # float32: the log power of a bin is good to about eps * max|Y| / |Y_k| of its segment, so each statistic is
    # held to the mean of that error over the segments (times 64) on top of the bar
    s, _, P = (np.concatenate(a) for a in zip(*[O.log_ms(_np(u), n, L) for u in utts]))
    top = P.max(axis=1, keepdims=True)
    d = 64 * np.finfo(np.float32).eps * np.sqrt(np.divide(top, P, out=np.zeros_like(P), where=P > 0))
    assert (np.abs(m - wm) <= d.mean(0) + tol * np.abs(wm).max()).all()
    assert (np.abs(v - wv) <= (2 * np.abs(s - wm) * d + d * d).mean(0) + tol * np.abs(wv).max()).all()
    assert rel_err(m, wm) <= 10 * tol and rel_err(v, wv) <= 100 * tol


def _stats_pair(rng, n, L, D):
    gen = list(_corpus(rng, 3, 120, D, 0.7))
    nat = list(_corpus(rng, 3, 120, D, 0.2, 13.0))
    return O.statistics(nat, n, L), O.statistics(gen, n, L)


# ---- 1. every instance, every segment length class and utterance edge -------------------------------------------------
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("n", NS)
def test_every_instance(n, dt):
    from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
    dtype = DT[dt]
    tol = TOL[dtype]
    rng = np.random.default_rng([n, dtype == np.float32])
    for L in sorted({4, n // 2, n}):
        H = L // 2
        N, G = _stats_pair(rng, n, L, 3)
        for T in sorted({1, max(1, H - 1), H, _tile(L) - 1, _tile(L) + 1}):
            x = _corpus(rng, 1, T, 3, 0.7)[0].astype(dtype)
            for k in (1.0, 0.4):
                y = modspec_post_filter(_cuda(x), N, G, k=k, n=n, segment=L)
                assert y.shape == x.shape and _np(y).dtype == dtype
                assert rel_err(_np(y), O.post_filter(x, N, G, k, n, L)) <= tol, (L, T, k)
        utts = [u.astype(dtype) for u in _corpus(rng, 3, 2 * _tile(L) + 3, 3, 0.5)]
        lens = np.array([len(utts[0]), 1, H + 1])
        got = modspec_statistics(_cuda(np.stack(utts)), n=n, lengths=lens, segment=L)
        want_utts = [u[:t] for u, t in zip(utts, lens)]
        _check_stats(got, O.statistics(want_utts, n, L), dtype, want_utts, n, L)


def launch(n, dt, mode):
    """One call of `mode` at (n, dt) whose kernel the profiler names (in a child process, see `kernels`)."""
    import torch

    from nnmnkwii_b200 import postfilters as PF
    K, D = n // 2 + 1, 3
    x = _cuda(_corpus(np.random.default_rng(n), 1, 40, D, 0.5)[0].astype(DT[dt]))
    if mode == "stats":
        PF.modspec_statistics(x, n=n, segment=4)
    else:
        stats = (np.zeros((K, D)), np.ones((K, D)))
        PF.modspec_post_filter(x, stats, stats, n=n, segment=4)
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def kernels():
    cases = [([n, dt, mode], FAMILY) for n in NS for dt in DT for mode in ("stats", "filter")]
    res = M.profiled_in_child("test_ms_segment_gpu", "launch", cases, repeats=True)
    out = {}
    for (case, _), (names, err) in zip(cases, res):
        assert err == "None", (case, err)
        out[tuple(case)] = names
    return out


def test_every_instance_is_launched_by_name(kernels):
    seen = set()
    for (n, dt, mode), names in kernels.items():
        assert len(names) == 1, (n, dt, mode, names)
        name = re.search(r"ms_segment_kernel<[^>]*>", names[0]).group(0)
        want = "ms_segment_kernel<%s, %d, %s>" % ("float" if dt == "f32" else "double", n.bit_length() - 1,
                                                  "true" if mode == "filter" else "false")
        assert name == want, (n, dt, mode, names)
        seen.add(name)
    assert len(seen) == 20


# ---- 2. long utterances, padded batches, column groups --------------------------------------------------------------
@pytest.mark.parametrize("dt", list(DT))
def test_ten_thousand_frames(dt):
    """One utterance of 10 000 frames (the utterance level stops at 4096) and a padded batch holding it."""
    import torch

    from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
    dtype = DT[dt]
    n, L = 64, 50
    rng = np.random.default_rng(10000)
    gen = _corpus(rng, 1, 10000, 4, 0.7)[0].astype(dtype)
    nat = _corpus(rng, 1, 10000, 4, 0.2, 13.0)[0].astype(dtype)
    Gt = modspec_statistics(_cuda(gen), n=n, segment=L)
    N = modspec_statistics(nat, n=n, segment=L)
    G = [_np(a) for a in Gt]
    _check_stats(G, O.statistics([gen], n, L), dtype, [gen], n, L)
    y = modspec_post_filter(_cuda(gen), N, Gt, k=0.8, n=n, segment=L)
    want = O.post_filter(gen, N, G, 0.8, n, L)
    assert rel_err(_np(y), want) <= TOL[dtype]
    pad = torch.full((3, 10000, 4), float("nan"), dtype=y.dtype, device="cuda")
    pad[0] = _cuda(gen)
    pad[1, :333] = _cuda(gen[:333])
    yb = modspec_post_filter(pad, N, G, k=0.8, n=n, lengths=[10000, 333, 0], segment=L)
    assert torch.equal(yb[0], y) and not yb[1, 333:].any() and not yb[2].any()
    assert rel_err(_np(yb[1, :333]), O.post_filter(gen[:333], N, G, 0.8, n, L)) <= TOL[dtype]


def _same(a, b):
    import torch
    return a.shape == b.shape and torch.equal(a, b)


@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("n,L", [(64, 50), (32, 4), (512, 512)])
def test_batched_equals_per_utterance(n, L, dt):
    import torch

    from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
    dtype = DT[dt]
    H = L // 2
    rng = np.random.default_rng([n, L])
    N, G = _stats_pair(rng, n, L, 5)
    lens = np.array([_tile(L) + 1, 0, 1, H - 1, H, _tile(L) - 1, 3 * _tile(L) + 5])
    T = int(lens.max()) + 7
    utts = [_cuda(_corpus(rng, 1, t, 5, 0.6)[0].astype(dtype)) for t in lens]
    want = [modspec_post_filter(u, N, G, k=0.8, n=n, segment=L) for u in utts]
    padded = torch.full((len(lens), T, 5), float("nan"), dtype=utts[0].dtype, device="cuda")
    for b, u in enumerate(utts):
        padded[b, :len(u)] = u
    y = modspec_post_filter(padded, N, G, k=0.8, n=n, lengths=lens, segment=L)
    for b, t in enumerate(lens):
        assert _same(y[b, :t], want[b]) and not y[b, t:].any(), b
        if 0 < t < 2000:
            assert rel_err(_np(want[b]), O.post_filter(_np(utts[b]), N, G, 0.8, n, L)) <= TOL[dtype], b
    # the statistics: NaN or zero padding give the same bits; they pool the segments of every utterance
    stats = modspec_statistics(padded, n=n, lengths=lens, segment=L)
    zero = modspec_statistics(torch.nan_to_num(padded, nan=0.0), n=n, lengths=lens, segment=L)
    assert all(_same(a, b) for a, b in zip(stats, zero))
    host = [_np(u) for u in utts]
    _check_stats(stats, O.statistics(host, n, L), dtype, host, n, L)


@pytest.mark.parametrize("dt", list(DT))
def test_column_groups(dt):
    """D of 1, one column group (16 float32 / 8 float64 columns) +- 1, and 60."""
    from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
    dtype = DT[dt]
    group = 16 if dtype == np.float32 else 8
    n, L = 64, 50
    rng = np.random.default_rng(group)
    for D in (1, group - 1, group, group + 1, 60):
        N, G = _stats_pair(rng, n, L, D)
        x = _corpus(rng, 2, 600, D, 0.7).astype(dtype)
        y = modspec_post_filter(_cuda(x), N, G, k=0.9, n=n, lengths=[600, 411], segment=L)
        assert rel_err(_np(y[0]), O.post_filter(x[0], N, G, 0.9, n, L)) <= TOL[dtype], D
        assert rel_err(_np(y[1, :411]), O.post_filter(x[1, :411], N, G, 0.9, n, L)) <= TOL[dtype], D
        got = modspec_statistics(_cuda(x), n=n, lengths=[600, 411], segment=L)
        _check_stats(got, O.statistics([x[0], x[1, :411]], n, L), dtype, [x[0], x[1, :411]], n, L)


# ---- 3. containers and determinism -----------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", list(DT))
def test_containers_and_repeats(dt):
    import torch

    from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
    dtype = DT[dt]
    n, L = 128, 80
    rng = np.random.default_rng(5)
    x = _corpus(rng, 2, 700, 6, 0.7).astype(dtype)
    Sn = modspec_statistics(x, n=n, segment=L)
    assert all(isinstance(a, np.ndarray) and a.dtype == np.float64 and a.shape == (n // 2 + 1, 6) for a in Sn)
    St = modspec_statistics(_cuda(x), n=n, segment=L)
    assert all(t.is_cuda and t.dtype == torch.float64 and t.is_contiguous() for t in St)
    assert all(np.array_equal(_np(t), a) for t, a in zip(St, Sn))
    N, _ = _stats_pair(rng, n, L, 6)
    y = modspec_post_filter(x[0], N, Sn, k=0.7, n=n, segment=L)
    assert isinstance(y, np.ndarray) and y.dtype == dtype and y.shape == x[0].shape
    yt = modspec_post_filter(_cuda(x[0]), N, St, k=0.7, n=n, segment=L)
    assert yt.is_cuda and yt.device == torch.device("cuda", torch.cuda.current_device())
    assert yt.dtype == _cuda(x).dtype and np.array_equal(_np(yt), y)
    for _ in range(3):
        assert torch.equal(modspec_post_filter(_cuda(x[0]), N, St, k=0.7, n=n, segment=L), yt)
        assert all(torch.equal(a, b) for a, b in zip(modspec_statistics(_cuda(x), n=n, segment=L), St))


# ---- 4. identities ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("n,L", [(32, 32), (64, 50), (512, 300)])
def test_identities(n, L, dt):
    from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
    dtype = DT[dt]
    tol = TOL[dtype]
    rng = np.random.default_rng([n, L, 1])
    gen = _cuda(_corpus(rng, 3, 1500, 5, 0.7).astype(dtype))
    G = modspec_statistics(gen, n=n, segment=L)
    N = modspec_statistics(_cuda(_corpus(rng, 3, 1500, 5, 0.2, 13.0).astype(dtype)), n=n, segment=L)
    for x in (gen[0], gen[1, :L // 2 + 3], gen[2, :1]):
        assert rel_err(_np(modspec_post_filter(x, N, G, k=0.0, n=n, segment=L)), _np(x)) <= tol
        assert rel_err(_np(modspec_post_filter(x, G, G, k=0.6, n=n, segment=L)), _np(x)) <= tol
    assert rel_err(_np(modspec_post_filter(gen[0], N, G, k=0.5, n=n, segment=L)), _np(gen[0])) > 1e-2
