"""GPU: preprocessing.meanvar / meanstd / minmax and the scale family against the reference's outputs
(golden file) and the restatement of its loop (oracle.normalize)."""
import hashlib
import os

import numpy as np
import pytest

import oracle.normalize as R
from conftest import ROOT, rel_err

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def P():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from nnmnkwii_b200 import preprocessing
    return preprocessing


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(ROOT, "tests", "golden", "normalize_reference_golden.npz"))


def _digest(a):
    """The golden file stores the scaling outputs as 'dtype shape sha256' of their C-order bytes."""
    a = np.ascontiguousarray(a)
    return "%s %s %s" % (a.dtype.str, "x".join(map(str, a.shape)), hashlib.sha256(a.tobytes()).hexdigest())


def _ulps(a, b):
    a = np.asarray(a)
    b = np.asarray(b)
    assert a.dtype == b.dtype == np.float32
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return int(np.abs(ia - ib).max())


def _close(got, ref, tol_mean=1e-12, tol_var=1e-10, var=False, const=None, const_value=0.0):
    """float32: equal or 1 ulp apart; float64: rel_err within the mean / variance tolerance.  `const` marks
    columns that are constant in the data: there the result is exactly `const_value` (variance 0, std 1),
    while the reference's variance is the rounding residue of its mean (e.g. 7.7e-33)."""
    got = got.cpu().numpy() if torch.is_tensor(got) else got
    assert got.dtype == ref.dtype, (got.dtype, ref.dtype)
    if const is not None and const.any():
        assert (got[const] == const_value).all()
        got, ref = got[~const], ref[~const]
    if ref.dtype == np.float32:
        assert _ulps(got, ref) <= 1
    else:
        assert rel_err(got, ref) <= (tol_var if var else tol_mean)


def _pad(utts, T=None):
    T = T or max(len(u) for u in utts)
    out = np.zeros((len(utts), T, utts[0].shape[1]), dtype=utts[0].dtype)
    for i, u in enumerate(utts):
        out[i, :len(u)] = u
    return out


@pytest.mark.parametrize("name", ["X", "Y"])
@pytest.mark.parametrize("form", ["a", "b", "c"])
def test_golden_parity(P, g, name, form):
    utts = [g["%s_%d" % (name, i)] for i in range(3)]
    lens = g[name + "_lengths"]
    if form == "a":
        ds, l, key = utts, None, ""
    elif form == "b":
        ds, l, key = _pad(utts, 1000), lens, "_pad"
    else:
        ds, l, key = torch.from_numpy(_pad(utts, 1000)).cuda(), lens, "_pad"
    const = np.ptp(np.concatenate(utts), axis=0) == 0  # many linguistic columns are constant
    m, v = P.meanvar(ds, l)
    _close(m, g[name + key + "_mean"])
    _close(v, g[name + key + "_var"], var=True, const=const)
    _, s = P.meanstd(ds, l)
    _close(s, g[name + key + "_std"], var=True, const=const, const_value=1.0)
    mn, mx = P.minmax(ds, l)
    for a, k in ((mn, "_min"), (mx, "_max")):
        a = a.cpu().numpy() if torch.is_tensor(a) else a
        assert a.dtype == np.float32 and np.array_equal(a, g[name + key + k])
    if form == "c":
        assert m.is_cuda and v.dtype == torch.float32


def test_golden_scaling(P, g):
    y0, x0 = g["Y_0"], g["X_0"]
    sy = P.scale(y0, g["Y_mean"], g["Y_std"])
    assert _digest(sy) == str(g["scale_Y0"])
    assert _digest(P.inv_scale(sy, g["Y_mean"], g["Y_std"])) == str(g["inv_scale_Y0"])
    fr = (0.01, 0.99)
    sx = P.minmax_scale(x0, g["X_min"], g["X_max"], feature_range=fr)
    assert _digest(sx) == str(g["minmax_scale_X0"])
    assert _digest(P.inv_minmax_scale(sx, g["X_min"], g["X_max"], feature_range=fr)) == str(g["inv_minmax_scale_X0"])


def _random_corpus(rng, n, D, dtype, lens):
    off = rng.standard_normal(D) * 3
    return [(rng.standard_normal((int(t), D)) * (1 + np.arange(D) % 5) + off + rng.standard_normal()).astype(dtype)
            for t in lens]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("D", [1, 31, 32, 33, 187, 425])
@pytest.mark.parametrize("form", ["a", "b", "c"])
def test_random_parity(P, dtype, D, form):
    rng = np.random.default_rng(D * 7 + (dtype == np.float32))
    Tmax = 301  # not a multiple of any tile
    lens = np.array([1, Tmax, 77, 0, 129, 300, 33])
    utts = _random_corpus(rng, len(lens), D, dtype, lens)
    ref_m, ref_v = R.meanvar([u for u in utts if len(u)])
    ref_mn, ref_mx = R.minmax([u for u in utts if len(u)])
    pad = _pad(utts, Tmax)
    if form == "a":
        ds, l = utts, None
    elif form == "b":
        ds, l = pad, lens
    else:
        ds, l = torch.from_numpy(pad).cuda(), lens
    m, v, n = P.meanvar(ds, l, return_last_sample_count=True)
    assert n == int(lens.sum()) and isinstance(n, int)
    _close(m, ref_m)
    _close(v, ref_v, var=True)
    mn, mx = P.minmax(ds, l)
    mn = mn.cpu().numpy() if torch.is_tensor(mn) else mn
    mx = mx.cpu().numpy() if torch.is_tensor(mx) else mx
    assert mn.dtype == dtype and np.array_equal(mn, ref_mn) and np.array_equal(mx, ref_mx)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_chunk_tails_in_staging(P, monkeypatch, dtype):
    from nnmnkwii_b200.preprocessing import normalize
    rng = np.random.default_rng(5)
    D = 33
    lens = [50, 7, 130, 1, 64, 99]
    utts = _random_corpus(rng, len(lens), D, dtype, lens)
    monkeypatch.setattr(normalize, "STAGING_BYTES", 2 * 40 * D * np.dtype(dtype).itemsize)  # 40 rows per half
    m, v = P.meanvar(utts)
    mn, mx = P.minmax(utts)
    rm, rv = R.meanvar(utts)
    _close(m, rm)
    _close(v, rv, var=True)
    rmn, rmx = R.minmax(utts)
    assert np.array_equal(mn, rmn) and np.array_equal(mx, rmx)


def test_incremental(P, g):
    inc = np.random.RandomState(1234).randn(32, 100, 24)  # the input of the reference's test_meanvar_incremental
    m, v = P.meanvar(inc)
    ma, va, n = P.meanvar(inc[:16], return_last_sample_count=True)
    assert n == 1600
    mb, vb = P.meanvar(inc[16:], mean_=ma, var_=va, last_sample_count=n)
    for got, ref, var in ((m, g["inc_mean"], False), (v, g["inc_var"], True), (mb, g["inc_mean_b"], False),
                          (vb, g["inc_var_b"], True), (mb, m, False), (vb, v, True)):
        _close(got, ref, var=var)
    # the reference test's meanstd split, and its allclose checks against NumPy
    ma, sa, n = P.meanstd(inc[:16], return_last_sample_count=True)
    mb, sb = P.meanstd(inc[16:], mean_=ma, var_=sa ** 2, last_sample_count=n)
    assert np.allclose(mb, np.mean(inc, axis=(0, 1))) and np.allclose(sb, np.std(inc, axis=(0, 1)))
    # the same on the device, state passed as CUDA tensors
    t = torch.from_numpy(inc).cuda()
    ta, tva, n = P.meanvar(t[:16], return_last_sample_count=True)
    tb, tvb = P.meanvar(t[16:], mean_=ta, var_=tva, last_sample_count=n)
    _close(tb, g["inc_mean_b"])
    _close(tvb, g["inc_var_b"], var=True)


def test_ill_conditioned_column(P):
    rng = np.random.default_rng(11)
    utts = [1e6 + 1e-3 * rng.standard_normal((int(t), 2)) + 1e-3 * rng.standard_normal()
            for t in rng.integers(50, 400, 40)]
    ref = np.var(np.concatenate(utts), axis=0)  # two-pass float64
    for ds in (utts, torch.from_numpy(_pad(utts)).cuda()):
        l = None if isinstance(ds, list) else [len(u) for u in utts]
        _, v = P.meanvar(ds, l)
        v = v.cpu().numpy() if torch.is_tensor(v) else v
        assert np.abs(v - ref).max() / ref.max() < 1e-6


def test_defined_behaviour(P):
    rng = np.random.default_rng(3)
    utts = _random_corpus(rng, 4, 5, np.float64, [20, 30, 40, 50])
    m0, v0 = P.meanvar(utts)
    m1, v1 = P.meanvar(utts[:2] + [np.zeros((0, 5))] + utts[2:])  # an empty utterance changes nothing
    assert np.array_equal(m0, m1) and np.array_equal(v0, v1)
    bad = [u.copy() for u in utts]
    bad[2][7, 3] = np.nan
    m, v = P.meanvar(bad)
    mn, mx = P.minmax(bad)
    for a in (m, v, mn, mx):
        assert np.isnan(a[3]) and np.isfinite(np.delete(a, 3)).all()
    rm, rv = R.meanvar([np.delete(u, 3, axis=1) for u in utts])
    _close(np.delete(m, 3), rm)
    _close(np.delete(v, 3), rv, var=True)


def test_deterministic(P):
    rng = np.random.default_rng(9)
    x = torch.from_numpy(rng.standard_normal((64, 700, 187)).astype(np.float32)).cuda()
    lens = rng.integers(1, 700, 64)
    a = P.meanvar(x, lens)
    b = P.meanvar(x, lens)
    for s, t in zip(a, b):
        assert torch.equal(s, t)


@pytest.mark.parametrize("xdt,pdt", [(np.float32, np.float32), (np.float64, np.float64), (np.float32, np.float64),
                                     (np.float64, np.float32)])
def test_scaling_bit_identical(P, xdt, pdt):
    rng = np.random.default_rng(1)
    x = (rng.standard_normal((3, 57, 33)) * 7).astype(xdt)
    a = rng.standard_normal(33).astype(pdt)
    b = (rng.random(33) + 0.1).astype(pdt)
    b[4] = 0  # scale: zero std -> 1
    for got, ref in ((P.scale(x, a, b), R.scale(x, a, b)), (P.inv_scale(x, a, b), R.inv_scale(x, a, b)),
                     (P.minmax_scale(x, scale_=b, min_=a), R.minmax_scale(x, scale_=b, min_=a)),
                     (P.inv_minmax_scale(x, scale_=b + 1, min_=a), R.inv_minmax_scale(x, scale_=b + 1, min_=a))):
        assert got.dtype == ref.dtype and got.shape == ref.shape
        assert np.array_equal(got, ref)
    t = P.scale(torch.from_numpy(x).cuda(), torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda())
    assert t.is_cuda and np.array_equal(t.cpu().numpy(), R.scale(x, a, b))


def test_reference_roundtrip_and_range_checks(P, g):
    # restated from the reference's tests/test_preprocessing.py test_meanvar / test_minmax
    Y = [g["Y_%d" % i] for i in range(3)]
    lengths = [len(y) for y in Y]
    Ym, Yv = P.meanvar(Y)
    Ys = np.sqrt(Yv)
    assert np.isfinite(Ym).all() and np.isfinite(Yv).all() and Ym.shape[-1] == 187
    assert np.allclose(Ys, P.meanstd(Y)[1])
    assert np.isfinite(P.scale(Y[0], Ym, Ys)).all()
    pad = _pad(Y, 1000)
    m2, v2 = P.meanvar(pad, lengths)
    assert np.allclose(Ym, m2) and np.allclose(Yv, v2)
    assert np.allclose(pad[0], P.inv_scale(P.scale(pad[0], Ym, Ys), Ym, Ys), atol=1e-5)
    X = [g["X_%d" % i] for i in range(3)]
    Xmin, Xmax = P.minmax(X)
    xs = P.minmax_scale(X[0], Xmin, Xmax, feature_range=(0, 0.99))
    assert xs.max() <= 1 and xs.min() >= 0 and np.isfinite(xs).all()
    min_, scale_ = P.minmax_scale_params(Xmin, Xmax, feature_range=(0, 0.99))
    assert np.allclose(xs, P.minmax_scale(X[0], min_=min_, scale_=scale_))
    xp = _pad(X, 1000)
    mn2, mx2 = P.minmax(xp, [len(x) for x in X])
    assert np.allclose(Xmin, mn2) and np.allclose(Xmax, mx2)
    assert np.allclose(xp[0], P.inv_minmax_scale(P.minmax_scale(xp[0], Xmin, Xmax), Xmin, Xmax))
    assert np.allclose(xp[0], P.inv_minmax_scale(P.minmax_scale(xp[0], scale_=scale_, min_=min_),
                                                 scale_=scale_, min_=min_))


def test_device_chain_into_mlpg(P, g):
    import oracle
    from conftest import windows_set
    from nnmnkwii_b200 import paramgen as G
    windows = windows_set()[2]
    Y = [g["Y_%d" % i] for i in range(3)]
    lens = np.array([len(y) for y in Y])
    pad = torch.from_numpy(_pad(Y)).cuda()
    Ym, Yv = P.meanvar(pad, lens)
    Ys = torch.sqrt(Yv)
    assert Yv.is_cuda and tuple(Yv.shape) == (187,)
    rng = np.random.default_rng(0)
    z = torch.from_numpy(rng.standard_normal(pad.shape).astype(np.float32)).cuda()  # a model's normalised output
    out = P.inv_scale(z, Ym, Ys)
    assert out.is_cuda and out.dtype == torch.float32
    y = G.mlpg_batch(out, Yv, windows, lengths=lens, layout=G.merlin_layout())
    y = y.cpu().numpy()
    host_out = P.inv_scale(z.cpu().numpy(), Ym.cpu().numpy(), Ys.cpu().numpy())
    assert np.array_equal(host_out, out.cpu().numpy())
    var = Yv.cpu().numpy()
    for b, T in enumerate(lens):
        u = host_out[b, :T]
        for col, (start, stat) in enumerate(((0, 60), (180, 1), (184, 1))):
            cols = slice(start, start + 3 * stat)
            ref = oracle.mlpg(u[:, cols], np.tile(var[cols], (T, 1)), windows)
            ocol = {0: slice(0, 60), 1: slice(60, 61), 2: slice(62, 63)}[col]
            assert rel_err(y[b, :T, ocol], ref) < 1e-5
