"""GPU: postfilters.merlin_post_filter (csrc/nnk_postfilter.cu) against Merlin's SPTK output and the
restated SPTK chain (oracle/sptk_postfilter.py), over every kernel instance the launcher can select."""
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle import sptk_postfilter as P

pytestmark = pytest.mark.gpu


def _mgc(rng, T, D, zero_rows=()):
    """Cepstrum-like frames: a decaying spectrum envelope, a few all-zero (padding) rows."""
    c = rng.standard_normal((T, D)) * (0.8 / (1.0 + np.arange(D)))
    c[:, 0] += 1.5 * rng.standard_normal(T)
    c[list(zero_rows)] = 0.0
    return c


def _check64(out, ref):
    tol = 1e-10 * max(1.0, float(np.abs(ref).max()))
    assert out.dtype == np.float64 and out.shape == ref.shape
    assert np.abs(out - ref).max() <= tol, np.abs(out - ref).max()


def test_merlin_golden():
    from nnmnkwii_b200.postfilters import merlin_post_filter
    g = np.load(os.path.join(ROOT, "tests", "golden", "merlin_post_filter_golden.npz"))
    out = merlin_post_filter(g["mgc"], 0.58, weight=g["weight"])
    assert isinstance(out, np.ndarray) and out.dtype == np.float32 and out.shape == (525, 60)
    assert np.allclose(out, g["mgc_p_mgc"], atol=1e-6)
    zero = np.abs(g["mgc"]).sum(1) == 0
    assert zero.sum() == 30 and np.all(out[zero] == 0)
    # same call with the reference's explicit arguments, and float64 against the restated chain
    out2 = merlin_post_filter(g["mgc"], 0.58, minimum_phase_order=511, fftlen=1024, coef=1.4, weight=g["weight"])
    assert np.array_equal(out, out2)
    x = g["mgc"].astype(np.float64)
    _check64(merlin_post_filter(x, 0.58, weight=g["weight"]), P.merlin_post_filter(x, 0.58, weight=g["weight"]))


@pytest.mark.parametrize("alpha", [0.0, 0.31, 0.41, 0.58, 0.77, -0.3])
def test_oracle_float64_alpha(alpha):
    from nnmnkwii_b200.postfilters import merlin_post_filter
    x = _mgc(np.random.default_rng(int(abs(alpha) * 100) + 1), 97, 60, zero_rows=(5,))
    out = merlin_post_filter(x, alpha)
    _check64(out, P.merlin_post_filter(x, alpha))
    assert np.all(out[5] == 0)


@pytest.mark.parametrize("fftlen", [16, 64, 512, 1024, 2048, 4096])
def test_oracle_float64_fftlen_and_order(fftlen):
    from nnmnkwii_b200.postfilters import merlin_post_filter
    rng = np.random.default_rng(fftlen)
    D = 60
    x = _mgc(rng, 33, D)
    w = rng.uniform(0.5, 2.0, D)
    for order in sorted({0, min(D - 2, fftlen - 1), fftlen // 2 - 1, fftlen - 1}):
        _check64(merlin_post_filter(x, 0.41, order, fftlen), P.merlin_post_filter(x, 0.41, order, fftlen))
        _check64(merlin_post_filter(x, 0.41, order, fftlen, weight=w),
                 P.merlin_post_filter(x, 0.41, order, fftlen, weight=w))
    _check64(merlin_post_filter(x, 0.41, 7, fftlen, coef=1.2), P.merlin_post_filter(x, 0.41, 7, fftlen, coef=1.2))


def test_oracle_float32():
    from nnmnkwii_b200.postfilters import merlin_post_filter
    x = _mgc(np.random.default_rng(7), 200, 60).astype(np.float32)
    for alpha in (0.41, 0.58):
        out = merlin_post_filter(x, alpha)
        ref = P.merlin_post_filter(x, alpha)
        assert out.dtype == np.float32
        assert np.all(np.abs(out - ref) <= 1e-6 * np.maximum(1.0, np.abs(ref)))


# D on both sides of every 16-wide k-step (KS = 1 .. 8 instances)
_DS = [1, 7, 8, 9, 15, 16, 17, 31, 32, 33, 47, 48, 49, 59, 60, 61, 63, 64, 65, 80, 81, 96, 97, 112, 113, 127, 128]


@pytest.mark.parametrize("D", _DS)
def test_every_instance(D):
    """Each D runs `postfilter_kernel<T, ceil(D / 16)>` in both dtypes (the launcher's switch on KS is a
    function of D alone); frame counts at the 64-frame tile tails and bin counts at the tails of the 8-bin
    tiles and of the stage chunks."""
    import torch
    from nnmnkwii_b200.postfilters import merlin_post_filter
    rng = np.random.default_rng(D)
    ks = (D + 15) // 16
    x = _mgc(rng, 129, D, zero_rows=(0, 64))
    for fftlen, order in ((64, 63), (16, 5), (2, 1)):
        ref = P.merlin_post_filter(x, 0.41, order, fftlen)
        for n in (129, 65, 64, 63, 1):
            _check64(merlin_post_filter(x[:n], 0.41, order, fftlen), ref[:n])
        assert np.all(merlin_post_filter(x, 0.41, order, fftlen)[[0, 64]] == 0)
    ref = P.merlin_post_filter(x, 0.41, 31, 32)
    for dt in (torch.float32, torch.float64):
        o = merlin_post_filter(torch.from_numpy(x).to("cuda", dt), 0.41, 31, 32).double().cpu().numpy()
        tol = 1e-10 if dt == torch.float64 else 1e-6
        assert np.all(np.abs(o - ref) <= tol * np.maximum(1.0, np.abs(ref)))


def test_long_bin_streams_and_many_frames():
    """The bin streaming over many stages (fftlen 4096: 257 tiles) at D = 128 and at D = 8, and a grid of
    several thousand CTAs."""
    from nnmnkwii_b200.postfilters import merlin_post_filter
    rng = np.random.default_rng(11)
    for D in (8, 128):
        x = _mgc(rng, 45, D)
        _check64(merlin_post_filter(x, 0.55, 1000, 4096), P.merlin_post_filter(x, 0.55, 1000, 4096))
    x = _mgc(rng, 300_001, 60)
    out = merlin_post_filter(x, 0.41, 63, 128)
    idx = np.r_[0:70, 150_000:150_070, 299_930:300_001]
    _check64(out[idx], P.merlin_post_filter(x[idx], 0.41, 63, 128))


def test_empty_and_single_frame():
    import torch
    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200.postfilters import merlin_post_filter
    n0 = _lib.launch_count()
    e = merlin_post_filter(np.zeros((0, 60), np.float32), 0.41)
    assert e.shape == (0, 60) and e.dtype == np.float32
    et = merlin_post_filter(torch.zeros((0, 60), dtype=torch.float64, device="cuda"), 0.41)
    assert et.shape == (0, 60) and et.dtype == torch.float64 and et.is_cuda
    assert _lib.launch_count() == n0
    x = _mgc(np.random.default_rng(1), 1, 60)
    _check64(merlin_post_filter(x, 0.41), P.merlin_post_filter(x, 0.41))


def test_layout_and_dtype():
    import torch
    from nnmnkwii_b200.postfilters import merlin_post_filter
    rng = np.random.default_rng(5)
    x = _mgc(rng, 300, 60)
    big = torch.from_numpy(rng.standard_normal((300, 187))).cuda()
    big[:, :60] = torch.from_numpy(x).cuda()
    for dt in (torch.float32, torch.float64):
        b = big.to(dt)
        view = b[:, :60]
        assert view.stride() == (187, 1)
        a = merlin_post_filter(view, 0.41)
        c = merlin_post_filter(view.contiguous(), 0.41)
        assert a.is_cuda and a.dtype == dt and torch.equal(a, c)
        assert np.array_equal(merlin_post_filter(view.cpu().numpy(), 0.41), c.cpu().numpy())
    # a column-strided view is made contiguous first
    xs = torch.from_numpy(np.ascontiguousarray(x.T)).cuda().T
    assert torch.equal(merlin_post_filter(xs, 0.41), merlin_post_filter(xs.contiguous(), 0.41))
    # other dtypes are computed and returned as float64
    h = x.astype(np.float16)
    o16 = merlin_post_filter(h, 0.41)
    assert o16.dtype == np.float64
    _check64(o16, P.merlin_post_filter(h.astype(np.float64), 0.41))
    ot = merlin_post_filter(torch.from_numpy(h).cuda(), 0.41)
    assert ot.dtype == torch.float64 and ot.is_cuda and np.array_equal(ot.cpu().numpy(), o16)
    # explicit weight as a torch tensor, and a cached basis reused on another stream
    w = torch.linspace(0.5, 1.5, 60, dtype=torch.float64)
    _check64(merlin_post_filter(x, 0.41, weight=w), P.merlin_post_filter(x, 0.41, weight=w.numpy()))
    s = torch.cuda.Stream()
    xt = torch.from_numpy(x).cuda()
    ref = merlin_post_filter(xt, 0.41)
    with torch.cuda.stream(s):
        xs2 = xt.clone()
        o = merlin_post_filter(xs2, 0.41)
    s.synchronize()
    assert torch.equal(o, ref)
    with pytest.raises(ValueError):
        merlin_post_filter(torch.from_numpy(x), 0.41)  # a CPU tensor


def test_invalid_arguments_launch_nothing():
    import torch
    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200.postfilters import merlin_post_filter
    x = torch.zeros((10, 60), device="cuda")
    bad = [dict(fftlen=1000), dict(minimum_phase_order=-1), dict(minimum_phase_order=16, fftlen=16),
           dict(weight=np.ones(59))]
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    for kw in bad:
        with pytest.raises((ValueError, AssertionError)):
            merlin_post_filter(x, 0.41, **kw)
    with pytest.raises(ValueError):
        merlin_post_filter(x[0], 0.41)
    with pytest.raises(NotImplementedError):
        merlin_post_filter(torch.zeros((10, 129), device="cuda"), 0.41)
    with pytest.raises(NotImplementedError):
        merlin_post_filter(x, 0.41, 511, 16384)
    assert _lib.launch_count() == n0


def test_tts_chain_on_the_device():
    """mlpg_batch in the Merlin layout, then the post-filter on the mgc columns of its output in place."""
    import oracle
    import torch
    from nnmnkwii_b200 import paramgen as G
    from nnmnkwii_b200.postfilters import merlin_post_filter
    windows = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))]
    rng = np.random.default_rng(2)
    lens = np.array([40, 64, 17, 90])
    n = int(lens.sum())
    m = np.zeros((n, 187), np.float32)
    m[:, :180] = np.tile(_mgc(rng, n, 60), 3) * np.repeat([1.0, 0.1, 0.05], 60)
    m[:, 180:] = rng.random((n, 7))
    v = (rng.random((n, 187)) * 0.1 + 0.01).astype(np.float32)
    y = G.mlpg_batch(torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda(), windows, lengths=lens,
                     layout=G.merlin_layout())
    assert y.is_cuda and y.shape == (n, 63)
    out = merlin_post_filter(y[:, :60], 0.41)
    assert out.is_cuda and out.dtype == torch.float32
    out = out.cpu().numpy()
    off = np.concatenate([[0], np.cumsum(lens)])
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        # the post-filter of the device trajectories, elementwise at the float32 bar
        own = P.merlin_post_filter(y[a:b, :60].cpu().numpy(), 0.41)
        assert np.all(np.abs(out[a:b] - own) <= 1e-6 * np.maximum(1.0, np.abs(own)))
        # the whole chain against the oracle MLPG followed by the oracle post-filter, at MLPG's float32 bar
        ref = P.merlin_post_filter(oracle.mlpg(m[a:b, :180], v[a:b, :180], windows), 0.41)
        assert np.abs(out[a:b] - ref).max() <= 2e-6 * max(1.0, np.abs(ref).max()), np.abs(out[a:b] - ref).max()
