"""GPU: interp1d, preemphasis / inv_preemphasis and the mu-law family against the reference's outputs
(tests/golden/wave_reference_golden.npz) and the restatement (oracle/wave.py).

interp1d and the pre-emphasis pair are bit-identical to scipy (NaN positions compared, not payloads).
The mu-law functions call libm's log1p and pow, whose last bit is implementation-defined on the host
and on the device, so they are held to ulp bars in the dtype those functions run in: 2 ulp, measured at
the magnitude of the value before the reference's exact ``- 1.0`` (otherwise a last-bit difference of
``(1 + mu) ** |y|`` near |y| = 0 counts as hundreds of ulps of the small difference).
"""
import os

import numpy as np
import pytest

import oracle.wave as R
from conftest import ROOT

pytestmark = pytest.mark.gpu

KINDS = ("linear", "slinear", "zero", "nearest", "nearest-up", "previous", "next")
IIR_L = 1024  # samples per chunk of the inverse filter (csrc/nnk_wave.cu)


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(ROOT, "tests", "golden", "wave_reference_golden.npz"))


@pytest.fixture(scope="module")
def P():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device")
    from nnmnkwii_b200 import preprocessing
    return preprocessing


def bit_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    if not np.array_equal(na, nb):
        return False
    return np.array_equal(a[~na].view(np.uint8), b[~nb].view(np.uint8)) if a.size else True


def _digest(a):
    import hashlib
    a = np.ascontiguousarray(a)
    return "%s %s %s" % (a.dtype.str, "x".join(map(str, a.shape)), hashlib.sha256(a.tobytes()).hexdigest())


# ---- interp1d ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_interp1d_golden(g, P, dt):
    import torch
    for i in range(3):
        lf0 = g["lf0_%d" % i].astype(dt)
        for kind in KINDS:
            key = "interp_%d_%s_%s" % (i, np.dtype(dt).name, kind)
            assert bit_equal(P.interp1d(lf0, kind), g[key]), key
            assert _digest(P.interp1d(lf0[:, None], kind)) == str(g[key + "_col"]), key
            t = P.interp1d(torch.from_numpy(lf0).cuda(), kind)
            assert t.is_cuda and bit_equal(t.cpu().numpy(), g[key]), key


def _f0_cases(rng, dt):
    cases = []
    for T in (1, 2, 3, 7, 255, 256, 257, 1000, 3001):
        for p_voiced in (0.0, 0.05, 0.5, 0.9, 1.0):
            f = (rng.random(T) * 4 + 3).astype(dt)
            f[rng.random(T) >= p_voiced] = 0.0
            cases.append(f)
    f = (rng.random(2000) * 4 + 3).astype(dt)
    f[100:900] = 0.0                          # a long unvoiced run
    f[:50] = -1e10                            # negative values, unvoiced start
    f[-70:] = 0.0                             # unvoiced end
    f[[300, 1200]] = np.nan                   # NaN: neither voiced nor filled
    f[[1500]] = np.inf                        # +inf is voiced
    f[1600:1700:3] = -0.0
    cases.append(f)
    one = np.zeros(500, dt)
    one[123] = 2.5                            # one voiced frame
    cases.append(one)
    g2 = np.zeros(400, dt)
    g2[[10, 11, 200]] = np.inf                # two infinite neighbours
    g2[300] = 4.0
    cases.append(g2)
    return cases


@pytest.mark.parametrize("dt", [np.float32, np.float64])
@pytest.mark.parametrize("kind", KINDS)
def test_interp1d_random_patterns(P, dt, kind):
    rng = np.random.default_rng(7)
    for f in _f0_cases(rng, dt):
        if len(f) == 1 and kind == "slinear" and f[0] > 0:
            with pytest.raises(ValueError):
                P.interp1d(f, kind)
            continue
        with np.errstate(invalid="ignore"):
            ref = R.interp1d(f.copy(), kind)
        got = P.interp1d(f, kind)
        assert bit_equal(got, ref), (kind, len(f))
        if not (f > 0).any():
            assert got is f


@pytest.mark.parametrize("dt", [np.float32, np.float64])
@pytest.mark.parametrize("kind", KINDS)
def test_interp1d_padded_batch(P, dt, kind):
    import torch
    rng = np.random.default_rng(11)
    B, Tmax = 37, 700
    lens = rng.integers(0, Tmax + 1, B)
    lens[:4] = [0, 2, Tmax, Tmax + 50]
    x = (rng.random((B, Tmax)) * 4 + 3).astype(dt)
    x[rng.random((B, Tmax)) < 0.6] = 0.0
    x[5] = 0.0                                 # a row with no voiced frame
    for tens in (False, True):
        arg = torch.from_numpy(x[:, :, None].copy()).cuda() if tens else x
        got = P.interp1d(arg, kind, lengths=lens)
        got = got.cpu().numpy().reshape(B, Tmax) if tens else got
        for b in range(B):
            n = min(int(lens[b]), Tmax)
            exp = x[b].copy()
            if n >= 2 or (n == 1 and kind != "slinear"):
                exp[:n] = R.interp1d(x[b, :n].copy(), kind) if n else exp[:n]
            assert bit_equal(got[b], exp), (b, n)


# ---- pre-emphasis --------------------------------------------------------------------------------------
def _signals(dt, rng):
    out = {}
    out["noise"] = rng.standard_normal(20000).astype(dt)
    sil = {np.float32: 5000, np.float64: 30000}[dt]
    s = np.zeros(2000 + sil, dt)
    s[:2000] = rng.standard_normal(2000).astype(dt)
    out["silence_to_denormals"] = s
    z = rng.standard_normal(5000).astype(dt)
    z[1000:1005] = [0.0, -0.0, -0.0, 0.0, -0.0]
    z[:2] = [-0.0, -0.0]
    out["signed_zeros"] = z
    n = rng.standard_normal(6000).astype(dt)
    n[2500] = np.nan
    out["nan_mid"] = n
    i = rng.standard_normal(6000).astype(dt)
    i[3100] = np.inf
    out["inf_mid"] = i
    for L in (0, 1, IIR_L - 1, IIR_L, IIR_L + 1, 3 * IIR_L + 17):
        out["len_%d" % L] = rng.standard_normal(L).astype(dt)
    return out


COEFS = (0.97, 0.86, 0.99, 0.999, 1.0, -0.97, 0.0, 1.5)


@pytest.mark.parametrize("dt", [np.float32, np.float64])
@pytest.mark.parametrize("coef", COEFS)
def test_preemphasis_pair_bit_identical(P, dt, coef):
    rng = np.random.default_rng(3)
    with np.errstate(all="ignore"):
        for name, x in _signals(dt, rng).items():
            if len(x) == 0:  # np.convolve raises on an empty signal; the device filter returns it
                assert P.preemphasis(x, coef).shape == (0,) and P.inv_preemphasis(x, coef).shape == (0,)
                continue
            assert bit_equal(P.preemphasis(x, coef), R.preemphasis(x, coef)), name
            assert bit_equal(P.inv_preemphasis(x, coef), R.inv_preemphasis(x, coef)), name


def test_denormals_reached():
    x = np.zeros(7000, np.float32)
    x[0] = 1.0
    y = R.inv_preemphasis(x, 0.97)
    assert ((y != 0) & (np.abs(y) < np.finfo(np.float32).tiny)).any()


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_preemphasis_golden(g, P, dt):
    x = (g["audio"] / 32768.0).astype(dt)
    for c in (0.97, 0.86, 0.0):
        assert _digest(P.preemphasis(x, c)) == str(g["pre_%s_%g" % (np.dtype(dt).name, c)])
        assert _digest(P.inv_preemphasis(x, c)) == str(g["inv_%s_%g" % (np.dtype(dt).name, c)])


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_preemphasis_ragged_batch(g, P, dt):
    import torch
    rng = np.random.default_rng(5)
    audio = (g["audio"] / 32768.0).astype(dt)
    B, Tmax = 9, 5 * IIR_L + 300
    x = np.stack([np.tile(audio, 1)[:Tmax] * rng.uniform(0.2, 2.0) if b % 2 else
                  rng.standard_normal(Tmax).astype(dt) for b in range(B)]).astype(dt)
    lens = np.array([0, 1, IIR_L - 1, IIR_L, IIR_L + 1, Tmax, Tmax + 9, 3 * IIR_L, 1234])
    for inverse, f, rf in ((False, P.preemphasis, R.preemphasis), (True, P.inv_preemphasis, R.inv_preemphasis)):
        for arg in (x, torch.from_numpy(x).cuda()):
            got = f(arg, 0.97, lengths=lens)
            got = got.cpu().numpy() if not isinstance(got, np.ndarray) else got
            for b in range(B):
                n = min(int(lens[b]), Tmax)
                exp = x[b].copy()
                if n:
                    exp[:n] = rf(x[b, :n], 0.97)
                assert bit_equal(got[b], exp), (inverse, b, n)
    # without lengths a padded batch means every row, full length
    assert bit_equal(P.inv_preemphasis(x, 0.97), R.inv_preemphasis(x, 0.97))
    x3 = x.reshape(3, 3, Tmax)
    assert bit_equal(P.preemphasis(x3, 0.86), R.preemphasis(x3, 0.86))


def test_inverse_long_signal_and_repair_counters(g, P):
    """One signal of 10.5 M samples (speech windows at seeded gains) in both dtypes, and a repair path
    that runs: at coef 0.999 the warm-up is capped, so some chunks start from a wrong state."""
    from nnmnkwii_b200.preprocessing import waveform
    rng = np.random.default_rng(9)
    audio = g["audio"] / 32768.0
    reps = 10_500_000 // len(audio) + 1
    x = (np.tile(audio, reps) * np.repeat(rng.uniform(0.1, 1.5, reps), len(audio)))[:10_500_000]
    for dt in (np.float32, np.float64):
        xd = x.astype(dt)
        assert bit_equal(P.inv_preemphasis(xd, 0.97), R.inv_preemphasis(xd, 0.97)), dt
        print("repair counters coef 0.97 %s: %s" % (np.dtype(dt).name, waveform._repair_counters()))
    xs = x[:400_000].astype(np.float32)
    assert bit_equal(P.inv_preemphasis(xs, 0.999), R.inv_preemphasis(xs, 0.999))
    chunks, samples = waveform._repair_counters()
    print("repair counters coef 0.999 float32: chunks %d samples %d" % (chunks, samples))
    assert chunks > 0 and samples > 0
    big = P.inv_preemphasis(xs, 1.5)  # |c| > 1: the repair walk is the whole sequential filter
    with np.errstate(all="ignore"):
        assert bit_equal(big, R.inv_preemphasis(xs, 1.5))
    assert waveform._repair_counters()[0] > 0


# ---- mu-law ----------------------------------------------------------------------------------------------
def _spacing(v, dt):
    return np.spacing(np.abs(np.asarray(v, np.float64)).astype(dt)).astype(np.float64)


def _check_mulaw(got, ref, cdt, what):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    bar = 2 * _spacing(ref, cdt)
    assert np.all(np.abs(got - ref) <= bar), (what, float(np.max(np.abs(got - ref) / np.maximum(bar, 1e-300))))


def _check_inv(got, ref, y, mu, cdt, what):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    pw = (1.0 + mu) ** np.abs(np.asarray(y, np.float64))
    bar = 2 * _spacing(ref, cdt) + 2 * _spacing(pw, cdt) / mu
    assert np.all(np.abs(got - ref) <= bar), (what, float(np.max(np.abs(got - ref) / bar)))


def _check_quant(got, x, mu, cdt, what):
    """Codes equal, except where the value before truncation lies within 4 ulp of an integer: ulp of the
    companded value sign(x) log1p(mu |x|) in the dtype log1p ran in, carried through / log1p(mu) * mu / 2."""
    ref_v = np.asarray(R.mulaw_quantize_unrounded(x, mu), np.float64)
    ref = np.trunc(ref_v).astype(np.int64)
    t = (ref_v * 2 / mu - 1) * np.log1p(mu)
    near = np.abs(ref_v - np.round(ref_v)) <= 4 * (_spacing(t, cdt) * mu / (2 * np.log1p(mu)) + _spacing(ref_v, cdt))
    diff = np.asarray(got) != ref
    print("%s: %d of %d codes near an integer, %d differ" % (what, int(near.sum()), ref.size, int(diff.sum())))
    assert not (diff & ~near).any(), what
    assert np.abs(np.asarray(got) - ref).max(initial=0) <= 1


MUS = (2, 128, 256, 512, 65536)


@pytest.mark.parametrize("mu", MUS)
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_mulaw_family(g, P, mu, dt):
    import torch
    rng = np.random.default_rng(mu)
    xs = [np.concatenate([rng.uniform(-1, 1, 50000), [-1.0, 1.0, 0.0, -0.0, 1e-30, -1e-6]]).astype(dt),
          (g["audio"] / 32768.0).astype(dt)]
    for x in xs:
        y = P.mulaw(x, mu)
        ry = R.mulaw(x, mu)
        assert y.dtype == ry.dtype
        _check_mulaw(y, ry, dt, "mulaw")
        _check_quant(P.mulaw_quantize(x, mu), x, mu, dt, "mulaw_quantize mu=%d %s" % (mu, np.dtype(dt).name))
        yy = ry.astype(dt)
        iy = P.inv_mulaw(yy, mu)
        assert iy.dtype == R.inv_mulaw(yy, mu).dtype
        _check_inv(iy, R.inv_mulaw(yy, mu), yy, mu, dt, "inv_mulaw")
        q = R.mulaw_quantize(x, mu)
        iq = P.inv_mulaw_quantize(q, mu)
        riq = R.inv_mulaw_quantize(q, mu)
        assert iq.dtype == riq.dtype == np.float32
        _check_inv(iq, riq, 2 * q.astype(np.float32) / np.float32(mu) - 1, mu, np.float32, "inv_mulaw_quantize")
        # tensors keep their dtype through the chain
        xt = torch.from_numpy(x).cuda()
        ty = P.mulaw(xt, mu)
        assert ty.is_cuda and ty.dtype == xt.dtype
        _check_mulaw(ty.cpu().numpy(), R.mulaw(xt.cpu(), mu).numpy(), dt, "mulaw tensor")
        tq = P.mulaw_quantize(xt, mu)
        assert tq.dtype == torch.int64
        _check_quant(tq.cpu().numpy(), xt.cpu(), mu, dt, "mulaw_quantize tensor mu=%d" % mu)
        tiq = P.inv_mulaw_quantize(torch.from_numpy(q).cuda(), mu)
        assert tiq.dtype == torch.float32
        _check_inv(tiq.cpu().numpy(), riq, 2 * q.astype(np.float32) / np.float32(mu) - 1, mu, np.float32, "t")


def test_mulaw_golden(g, P):
    for mu in (256, 2):
        for dt in (np.float32, np.float64):
            x = (g["audio"][:1024] / 32768.0).astype(dt)
            tag = "%d_%s" % (mu, np.dtype(dt).name)
            y = P.mulaw(x, mu)
            assert y.dtype.str == str(g["mu_mulaw_%s_dtype" % tag])
            _check_mulaw(y, g["mu_mulaw_" + tag], dt, "golden mulaw")
            q = P.mulaw_quantize(x, mu)
            assert q.dtype.str == str(g["mu_quant_%s_dtype" % tag])
            assert np.abs(q - g["mu_quant_" + tag]).max() <= 1
            iy = P.inv_mulaw(g["mu_mulaw_" + tag].astype(dt), mu)
            assert iy.dtype.str == str(g["mu_inv_%s_dtype" % tag])
            _check_inv(iy, g["mu_inv_" + tag], g["mu_mulaw_" + tag].astype(dt), mu, dt, "golden inv")
            iq = P.inv_mulaw_quantize(g["mu_quant_" + tag], mu)
            assert iq.dtype.str == str(g["mu_invq_%s_dtype" % tag])
            _check_inv(iq, g["mu_invq_" + tag], 2 * g["mu_quant_" + tag].astype(np.float32) / np.float32(mu) - 1,
                       mu, np.float32, "golden invq")


def test_mulaw_reference_corner_cases(P):
    """The reference's test_mulaw, case for case, on the device functions."""
    import torch
    assert P.mulaw_quantize(-1.0, 2) == 0
    assert P.mulaw_quantize(-0.5, 2) == 0
    assert P.mulaw_quantize(-0.001, 2) == 0
    assert P.mulaw_quantize(0.0, 2) == 1
    assert P.mulaw_quantize(0.0001, 2) == 1
    assert P.mulaw_quantize(0.5, 2) == 1
    assert P.mulaw_quantize(0.99999, 2) == 1
    assert P.mulaw_quantize(1.0, 2) == 2
    rs = np.random.RandomState(1234)
    for mu in [128, 256, 512]:
        for x in rs.rand(100):
            y = P.mulaw(x, mu)
            assert y >= 0 and y <= 1
            assert np.allclose(x, P.inv_mulaw(y, mu))
    for mu in [128, 256, 512]:
        for x, y in [(-1.0, 0), (0.0, mu // 2), (0.99999, mu - 1)]:
            y_hat = P.mulaw_quantize(x, mu)
            assert isinstance(y_hat, int) and np.allclose(y, y_hat)
            assert np.abs(x - P.inv_mulaw_quantize(y_hat, mu)) <= 0.1
    for mu in [128, 256, 512]:
        x = rs.rand(10)
        assert np.allclose(x, P.inv_mulaw(P.mulaw(x, mu), mu))
        P.inv_mulaw_quantize(P.mulaw_quantize(x))
    torch.manual_seed(1234)
    for mu in [128, 256, 512]:
        x = torch.rand(10)
        x_hat = P.inv_mulaw(P.mulaw(x, mu), mu)
        assert np.allclose(x, x_hat)
        P.inv_mulaw_quantize(P.mulaw_quantize(x))
    assert isinstance(P.mulaw(0.5), np.float64) and isinstance(P.inv_mulaw(np.float32(0.5)), np.float32)
    assert isinstance(P.inv_mulaw_quantize(3), np.float64)
    x = (np.load(os.path.join(ROOT, "tests", "golden", "wave_reference_golden.npz"))["audio"] / 32768.0).astype(np.float32)
    y = P.mulaw_quantize(x, 256)
    assert y.min() >= 0 and y.max() < 256 and y.dtype == int
    assert P.inv_mulaw_quantize(y, 256).dtype == np.float32


# ---- every kernel instance ---------------------------------------------------------------------------
def launch_group(group):
    """The calls of one group of kernel instances (run in a child process by `profiled_in_child`)."""
    import torch

    from nnmnkwii_b200 import preprocessing as Pp
    x = np.random.default_rng(0).standard_normal(3000)
    if group.startswith("f0_"):
        dt = np.float32 if group == "f0_float" else np.float64
        for kind in KINDS:
            Pp.interp1d(np.array([0.0, 2.0, 0.0, 0.0, 3.0, 0.0], dt), kind)
    elif group.startswith("filters_"):
        dt = np.float32 if group == "filters_float" else np.float64
        Pp.preemphasis(x.astype(dt))
        Pp.inv_preemphasis(x.astype(dt))
    else:
        xs = (x * 0.1).astype(np.float32)
        for dt in (np.float32, np.float64):
            Pp.inv_mulaw(xs.astype(dt))
        Pp.mulaw(xs), Pp.mulaw(torch.from_numpy(xs).cuda()), Pp.mulaw(xs.astype(np.float64))
        Pp.mulaw_quantize(xs), Pp.mulaw_quantize(torch.from_numpy(xs).cuda()), Pp.mulaw_quantize(xs.astype(np.float64))
        codes = np.arange(256)
        for c in (codes.astype(np.int64), codes.astype(np.int32), codes.astype(np.float32), codes.astype(np.float64)):
            Pp.inv_mulaw_quantize(c)
        Pp.inv_mulaw_quantize(3)
    torch.cuda.synchronize()


def test_every_kernel_instance_runs(P):
    """Each instance the launchers can select (dtype x kind x direction x mode x variant), by kernel name."""
    from variant_mirror import launched, profiled_in_child
    groups = [("f0_float", r"f0_interp_kernel"), ("f0_double", r"f0_interp_kernel"),
              ("filters_float", r"preemph_\w+_kernel"), ("filters_double", r"preemph_\w+_kernel"),
              ("mulaw", r"mulaw_kernel")]
    res = profiled_in_child("test_wave_gpu", "launch_group", [([grp], fam) for grp, fam in groups])
    names = {grp: r[0] for (grp, _), r in zip(groups, res)}
    for (grp, _), r in zip(groups, res):
        assert r[1] == "None", (grp, r[1])
    for t in ("float", "double"):
        for k in range(7):
            assert launched(names["f0_" + t], r"f0_interp_kernel<%s, %d>" % (t, k)), (t, k)
        for kern in ("fir", "est", "spec", "repair"):
            assert launched(names["filters_" + t], r"preemph_%s_kernel<%s>" % (kern, t)), (kern, t)
        assert launched(names["filters_" + t], r"preemph_carry_kernel")
    F, D, I = "float", "double", "long long"
    expect = [(0, F, F, D, D), (0, F, F, F, F), (0, D, D, D, D), (2, F, F, D, I), (2, F, F, F, I), (2, D, D, D, I),
              (1, F, F, F, F), (1, D, D, D, D), (3, F, F, F, F), (3, D, F, F, F), (3, "int", F, F, F),
              (3, I, F, F, F), (3, D, D, D, D)]
    for e in expect:
        assert launched(names["mulaw"], r"mulaw_kernel<%s>" % ", ".join(str(v) for v in e)), e
