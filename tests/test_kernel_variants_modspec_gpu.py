"""Every `modspec_kernel<T, LOGN, PF>` instance (csrc/nnk_modspec.cu) in every mode it runs, against float64 NumPy
references computed from the same float32 / float64 input, upcast.

`nnk_modspec` serves n = 256 ... 4096 with LOGN = log2 n (`dispatch_modspec`: a case per LOGN below the largest,
which is the default) and takes the PF instance exactly for the log power and the post-filter, the other one for
the power, smoothing, inverse and gradient modes: 5 lengths x 2 dtypes x 2 = 20 instances.  The references:

* power and phase: `numpy.fft.rfft` with the same norm;
* smoothing: `ms[limit:] = 0` on rfft's spectrum, in the log domain (the bin keeps its phase at unit power) or
  the power domain (the bin is 0), then `irfft`;
* inverse: `irfft(sqrt(ms) * phase)`, with random phases on every bin (irfft ignores the imaginary parts of
  bins 0 and n / 2, and so must the kernel);
* gradient: the reference's dense formula, `2 fwd^2 sum_k G_k (Re X_k cos + Im X_k sin)(-2 pi k t / n)`;
* log power and post-filter: `oracle/ms_postfilter.py`.

Groups: (1) every instance and mode at T = 1, 2, n/2 - 1, n/2, n/2 + 1, n - 1, n and D = 1, 37, with the
instance names profiled in a child process (`variant_mirror.profiled_in_child`) and compared with the mirror;
(2) smoothing with `limit_bin` at 0, 1, 2, M/2, M/2 + 1, M and K (M = n / 2, K = M + 1), directly and through
`modspec_smoothing`'s cut-off, negative cut-offs included; (3) the gradient through `autograd.ModSpec` and
`ModSpecBatch` at every n and norm; (4) 65 540 utterances, more than grid.y holds, so the kernel's utterance
loop makes a second pass; (5) the C ABI's length clip, T_in != T_out, and calls that must launch nothing.

Float32 bars (`TOL32`), measured on an H100 80GB HBM3 (700 W limit): the worst float32 error of every comparison
in the module, per mode over all five n (per-n figures in DESIGN.md section 4; `WORST` collects them in a run):

    mode        worst float32 error    bar       headroom
    power       3.50e-7                1.5e-6    4.3x    power, and the phase weighted by the amplitude
    smooth      3.50e-6                1.5e-5    4.3x    n = 4096 (the others <= 5.9e-7): unit phases of small bins
    inverse     2.16e-7                1e-6      4.6x
    grad        3.73e-7                1.5e-6    4.0x
    logpower    8.54e-8                4e-7      4.7x    amplitude-weighted (see `_logpower`; plain rel_err 2.7e-5)
    postfilter  2.02e-5                9e-5      4.5x

The post-filter and the plain log power are as far off in a float32 FFT on the host (NumPy / SciPy pocketfft,
same data: up to 2.8e-5 and 3.0e-5): a small bin's float32 power is only good to eps max |Y| / |Y_k|, and the
filter's exponent a != 1 carries that into the output.  Float64 is held to 1e-10, as in tests/test_modspec_gpu.py
(worst seen: 2.6e-13).  The module runs 105 cases in about 35 s on that GPU, 16 s of it the profiled child
process and 8 s the first case (CUDA start-up)."""
import functools
import re

import numpy as np
import pytest

import oracle.ms_postfilter as O
import variant_mirror as M
from conftest import rel_err

pytestmark = pytest.mark.gpu

NS = tuple(2 ** logn for logn in range(M.MS_LOGN_MIN, M.MS_LOGN_MAX + 1))
DT = {"f32": np.float32, "f64": np.float64}
NORMS = (None, "ortho", "forward")
MODES = {"power": 0, "smooth": 1, "inverse": 2, "grad": 3, "logpower": 4, "postfilter": 5}  # NNK_MS_*
TOL64 = 1e-10
TOL32 = {"power": 1.5e-6, "smooth": 1.5e-5, "inverse": 1e-6, "grad": 1.5e-6, "logpower": 4e-7, "postfilter": 9e-5}
WORST = {}  # (mode, n, dtype name) -> largest rel_err seen
BIG_B = 65537 + 3  # grid.y holds 65 535 utterances: five more make a second pass of the utterance loop
FAMILY = r"\bmodspec_kernel<"


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _same(a, b):
    import torch
    return a.shape == b.shape and torch.equal(torch.view_as_real(a) if a.is_complex() else a,
                                              torch.view_as_real(b) if b.is_complex() else b)


def _crel(a, b):
    """max |a - b| / max |b| of complex arrays."""
    a, b = np.asarray(a, np.complex128), np.asarray(b, np.complex128)
    return float(np.abs(a - b).max() / max(1e-300, np.abs(b).max()))


def _check(got, want, mode, n, dtype, tag, err=None, scale=None):
    """`rel_err(got, want)` (or `err`; with `scale`, max |got - want| / max |scale|) within the bar of `mode` and
    `dtype`; the worst is kept in WORST."""
    if err is not None:
        e = err
    elif scale is not None:
        e = float(np.abs(np.asarray(got, np.float64) - want).max() / max(1e-300, np.abs(scale).max()))
    else:
        e = rel_err(got, want)
    key = (mode, n, np.dtype(dtype).name)
    WORST[key] = max(WORST.get(key, 0.0), e)
    bar = TOL32[mode] if np.dtype(dtype) == np.float32 else TOL64
    assert e <= bar, (mode, n, np.dtype(dtype).name, tag, e, bar)


def _scales(norm, n):
    """(forward, inverse) scale of numpy.fft's `norm`."""
    return {None: (1.0, 1.0 / n), "ortho": (n ** -0.5, n ** -0.5), "forward": (1.0 / n, 1.0)}[norm]


def _traj(rng, T, D, tilt=0.5, gain=10.0):
    """(T, D) float64: white noise through 1 + tilt z^-1.  Its spectrum has no systematic valleys (a random walk
    would put nearly all the power in the lowest bins), but single bins still fall far below the largest, and
    the float32 error of such a bin's phase or log power grows as max |Y| / |Y_k|."""
    w = rng.standard_normal((T + 1, D))
    return gain * (w[1:] + tilt * w[:-1])


def _sizes(n):
    return (1, 2, n // 2 - 1, n // 2, n // 2 + 1, n - 1, n)


# ---- float64 references ---------------------------------------------------------------------------------------
def _smooth_ref(x, n, norm, limit, log_domain):
    """`ms[limit:] = 0` (a negative `limit` counts from the end, as the reference's slice does) in the log or the
    power domain, then irfft, cut to the frames of x."""
    X = np.fft.rfft(np.asarray(x, np.float64), n, axis=0, norm=norm)
    C = X.copy()
    C[limit:] = np.exp(1j * np.angle(X[limit:])) if log_domain else 0
    return np.fft.irfft(C, n, axis=0, norm=norm)[:len(x)]


@functools.lru_cache(maxsize=4)
def _kt_tables(n, T):
    """cos and sin of kt = -2 pi k t / n, (T, n // 2 + 1) each; k t is reduced mod n first, exactly."""
    kt = -2 * np.pi / n * ((np.arange(T)[:, None] * np.arange(n // 2 + 1)) % n)
    return np.cos(kt), np.sin(kt)


def _grad_ref(x, G, n, norm):
    """dL/dx of L = sum(G * modspec(x, n, norm)): the reference's dense formula scaled by fwd^2."""
    x, G = np.asarray(x, np.float64), np.asarray(G, np.float64)
    X = np.fft.rfft(x, n, axis=0)
    cos, sin = _kt_tables(n, len(x))
    return 2 * _scales(norm, n)[0] ** 2 * (cos @ (G * X.real) + sin @ (G * X.imag))


@functools.lru_cache(maxsize=None)
def _stats(n, D):
    """(natural, generated) float64 statistics of two corpora: the generated one smoother and quieter."""
    rng = np.random.default_rng([n, D])
    gen = [_traj(rng, n // 2, D, 0.7) for _ in range(4)]
    nat = [_traj(rng, n // 2, D, 0.2, 13.0) for _ in range(4)]
    return O.statistics(nat, n), O.statistics(gen, n)


# ---- 1. every instance, every mode ----------------------------------------------------------------------------
def _P():
    from nnmnkwii_b200 import preprocessing as P
    return P


def _power(x, n, rng, tag):
    P = _P()
    xt, dtype = _cuda(x), x.dtype
    for norm in NORMS:
        X = np.fft.rfft(x.astype(np.float64), n, axis=0, norm=norm)
        ms, ph = P.modspec(xt, n=n, norm=norm, return_phase=True)
        assert ms.shape == ph.shape == (n // 2 + 1, x.shape[1]) and ms.dtype == xt.dtype
        assert _same(P.modspec(xt, n=n, norm=norm), ms)  # the phase output changes nothing of the power
        _check(_np(ms), np.abs(X) ** 2, "power", n, dtype, tag + (norm,))
        # the phase where it matters, weighted by the amplitude; in float64 also on its own
        amp = np.sqrt(_np(ms).astype(np.float64)) * _np(ph)
        _check(None, None, "power", n, dtype, tag + (norm, "phase"), _crel(amp, X))
        if dtype == np.float64:
            _check(None, None, "power", n, dtype, tag + (norm, "unit"), _crel(_np(ph), np.exp(1j * np.angle(X))))


def _smooth(x, n, rng, tag):
    P = _P()
    xt = _cuda(x)
    for norm in NORMS:
        for log_domain in (True, False):
            y = P.modspec_smoothing(xt, 200, n=n, norm=norm, cutoff=30, log_domain=log_domain)
            assert y.shape == xt.shape and y.dtype == xt.dtype
            want = _smooth_ref(x, n, norm, int(n * 30 / 200) + 1, log_domain)
            _check(_np(y), want, "smooth", n, x.dtype, tag + (norm, log_domain))


def _inverse(x, n, rng, tag):
    """A random power and random unit phases on every bin (the frames of x only set T and D)."""
    P = _P()
    T, D = x.shape
    K = n // 2 + 1
    cdt = np.complex64 if x.dtype == np.float32 else np.complex128
    ms = (rng.exponential(size=(K, D)) * 100.0 * T).astype(x.dtype)
    ph = np.exp(2j * np.pi * rng.random((K, D))).astype(cdt)
    for norm in NORMS:
        want = np.fft.irfft(np.sqrt(ms.astype(np.float64)) * ph.astype(np.complex128), n, axis=0, norm=norm)
        y = P.inv_modspec(_cuda(ms), _cuda(ph), norm=norm)
        assert y.shape == (n, D)
        _check(_np(y), want, "inverse", n, x.dtype, tag + (norm,))
        # T_out = T frames, judged on the scale of the whole inverse (a few frames may all be small)
        yb = P.inv_modspec(_cuda(ms[None]), _cuda(ph[None]), norm=norm, lengths=[T])
        assert yb.shape == (1, T, D)
        _check(_np(yb[0]), want[:T], "inverse", n, x.dtype, tag + (norm, "lengths"), scale=want)


def _grad(x, n, rng, tag):
    from nnmnkwii_b200.preprocessing.modspec import _modspec_grad
    G = rng.standard_normal((n // 2 + 1, x.shape[1])).astype(x.dtype)
    for norm in NORMS:
        g = _modspec_grad(_cuda(x), _cuda(G), n, norm)
        assert g.shape == x.shape and g.dtype == _cuda(x).dtype
        _check(_np(g), _grad_ref(x, G, n, norm), "grad", n, x.dtype, tag + (norm,))


def _logpower(x, n, rng, tag):
    """One utterance: the mean is its log power, the variance 0.  In float32 the error of s_k is weighted by
    |Y_k| / max |Y| of its column: a float32 FFT leaves each bin an absolute error of about eps max |Y|, which
    is a large relative error of a small bin and so of its log (a float32 FFT on the host does the same)."""
    from nnmnkwii_b200.postfilters import modspec_statistics
    mean, var = modspec_statistics(_cuda(x), n=n)
    s, Y, _ = O.log_ms(x, n)
    err = None
    if x.dtype == np.float32:
        amp = np.abs(Y) / np.abs(Y).max(axis=0)
        err = float((np.abs(_np(mean) - s) * amp).max() / np.abs(s).max())
    _check(_np(mean), s, "logpower", n, x.dtype, tag, err)
    assert not _np(var).any(), tag


def _postfilter(x, n, rng, tag):
    from nnmnkwii_b200.postfilters import modspec_post_filter
    nat, gen = _stats(n, x.shape[1])
    y = modspec_post_filter(_cuda(x), nat, gen, k=0.8, n=n)
    assert y.shape == x.shape
    _check(_np(y), O.post_filter(x, nat, gen, 0.8, n), "postfilter", n, x.dtype, tag)


RUN = {"power": _power, "smooth": _smooth, "inverse": _inverse, "grad": _grad, "logpower": _logpower,
       "postfilter": _postfilter}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("n", NS)
def test_every_instance(n, dt, mode):
    rng = np.random.default_rng([n, MODES[mode], dt == "f32"])
    assert max(_sizes(n)) > M.ms_threads(n)  # the frame loops make more than one pass
    for T in _sizes(n):
        for D in (1, 37):
            RUN[mode](_traj(rng, T, D).astype(DT[dt]), n, rng, (T, D))


def launch(n, dt, mode):
    """One call of `mode` at (n, dt) whose kernel the profiler names (in a child process, see `kernels`)."""
    import torch

    from nnmnkwii_b200 import postfilters as PF
    from nnmnkwii_b200.preprocessing.modspec import _modspec_grad
    P = _P()
    dtype = DT[dt]
    K, D = n // 2 + 1, 3
    x = _cuda(_traj(np.random.default_rng(n), 9, D).astype(dtype))
    ones = torch.ones((K, D), dtype=x.dtype, device="cuda")
    if mode == "power":
        P.modspec(x, n=n, return_phase=True)
    elif mode == "smooth":
        P.modspec_smoothing(x, 200, n=n)
    elif mode == "inverse":
        P.inv_modspec(ones, ones.to(torch.complex64 if dt == "f32" else torch.complex128))
    elif mode == "grad":
        _modspec_grad(x, ones, n, None)
    elif mode == "logpower":
        PF.modspec_statistics(x, n=n)
    else:
        stats = (np.zeros((K, D)), np.ones((K, D)))
        PF.modspec_post_filter(x, stats, stats, n=n)
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def kernels():
    """(n, dt, mode) -> names of the modspec kernels its call launched, one per launch."""
    cases = [([n, dt, mode], FAMILY) for n in NS for dt in DT for mode in MODES]
    res = M.profiled_in_child("test_kernel_variants_modspec_gpu", "launch", cases, repeats=True)
    out = {}
    for (case, _), (names, err) in zip(cases, res):
        assert err == "None", (case, err)
        out[tuple(case)] = names
    return out


def test_every_instance_is_launched_by_name(kernels):
    seen = set()
    for (n, dt, mode), names in kernels.items():
        assert len(names) == 1, (n, dt, mode, names)
        name = re.search(r"modspec_kernel<[^>]*>", names[0]).group(0)
        assert name == M.modspec_kernel_for(n, DT[dt], MODES[mode]), (n, dt, mode, names)
        seen.add(name)
    assert seen == {M.modspec_kernel_for(n, dtype, mode) for n in NS for dtype in DT.values() for mode in (0, 4)}
    assert len(seen) == 20


# ---- 2. smoothing at every limit_bin edge ---------------------------------------------------------------------
def _smooth_direct(x, n, norm, limit_bin, log_domain):
    """NNK_MS_SMOOTH of one (T, D) utterance with `limit_bin` as given, into a NaN-filled output."""
    import torch

    from nnmnkwii_b200.preprocessing.modspec import _launch
    xt = _cuda(x[None])
    out = torch.full_like(xt, float("nan"))
    fwd, inv = _scales(norm, n)
    _launch(MODES["smooth"], n, xt, None, out, None, 1, x.shape[0], x.shape[0], x.shape[1], None, fwd, inv,
            limit_bin, log_domain)
    return out[0]


@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("n", [256, 4096])
def test_smoothing_at_every_limit_bin_edge(n, dt):
    rng = np.random.default_rng([n, 2, dt == "f32"])
    Mh = n // 2
    for T in (n, n // 2 + 1):
        x = _traj(rng, T, 5).astype(DT[dt])
        for limit in (0, 1, 2, Mh // 2, Mh // 2 + 1, Mh, Mh + 1):
            for log_domain in (True, False):
                y = _smooth_direct(x, n, "ortho", limit, log_domain)
                _check(_np(y), _smooth_ref(x, n, "ortho", limit, log_domain), "smooth", n, x.dtype,
                       (T, limit, log_domain))


@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("n", [256, 4096])
def test_smoothing_cutoff_edges(n, dt):
    """Cut-offs whose first removed bin `int(n cutoff / modfs) + 1` is 1, M/2 + 1 and K, none, and negative ones
    (the reference's `ms[limit:]` counts them from the end; below -K every bin goes)."""
    P = _P()
    rng = np.random.default_rng([n, 3, dt == "f32"])
    Mh, K = n // 2, n // 2 + 1
    cases = [(200, 0, 1), (200, 50, Mh // 2 + 1), (200.0, 100.0, K), (16000 / 80, None, K), (200, -50, 1 - n // 4),
             (200, -150, 1 - 3 * n // 4)]
    for T in (n, 100):
        x = _traj(rng, T, 4).astype(DT[dt])
        for modfs, cutoff, limit in cases:
            assert limit == (K if cutoff is None else int(n * cutoff / modfs) + 1)
            for log_domain in (True, False):
                y = P.modspec_smoothing(_cuda(x), modfs, n=n, cutoff=cutoff, log_domain=log_domain)
                _check(_np(y), _smooth_ref(x, n, None, limit, log_domain), "smooth", n, x.dtype,
                       (T, cutoff, log_domain))


# ---- 3. the gradient at every n and norm ------------------------------------------------------------------------
@pytest.mark.parametrize("norm", NORMS, ids=["backward", "ortho", "forward"])
@pytest.mark.parametrize("n", NS)
def test_gradient_against_the_dense_formula(n, norm):
    """autograd.ModSpec at T = 1, 200 and n, and ModSpecBatch over ragged lengths with NaN padding: each float32
    gradient against the float64 formula on its own input; frames past a length get exactly 0."""
    import torch

    from nnmnkwii_b200 import autograd as A
    rng = np.random.default_rng([n, 4, NORMS.index(norm)])
    K, D = n // 2 + 1, 5
    for dt, dtype in DT.items():
        for T in (1, 200, n):
            x = _traj(rng, T, D).astype(dtype)
            G = rng.standard_normal((K, D)).astype(dtype)
            y = _cuda(x).requires_grad_()
            (A.modspec(y, n, norm) * _cuda(G)).sum().backward()
            assert y.grad.dtype == y.dtype
            _check(_np(y.grad), _grad_ref(x, G, n, norm), "grad", n, dtype, (T,))
        lens = [n, 1, 0, min(200, n - 1), 77]
        xb = np.full((len(lens), n, D), np.nan, dtype)
        for b, L in enumerate(lens):
            xb[b, :L] = _traj(rng, L, D)
        Gb = rng.standard_normal((len(lens), K, D)).astype(dtype)
        yb = _cuda(xb).requires_grad_()
        ms = A.modspec_batch(yb, lens, n, norm)
        assert torch.isfinite(ms).all()
        (ms * _cuda(Gb)).sum().backward()
        g = _np(yb.grad)
        for b, L in enumerate(lens):
            assert np.all(g[b, L:] == 0), (dt, b)
            if L:
                _check(g[b, :L], _grad_ref(xb[b, :L], Gb[b], n, norm), "grad", n, dtype, ("batch", b, L))


# ---- 4. more utterances than grid.y holds ------------------------------------------------------------------------
def _big_run(mode, n, x, lens, G):
    """One call of `mode` over the padded batch x with `lengths`."""
    from nnmnkwii_b200.postfilters import modspec_post_filter
    from nnmnkwii_b200.preprocessing.modspec import _modspec_grad
    P = _P()
    if mode == "power":
        return P.modspec(x, n=n, lengths=lens)
    if mode == "smooth":
        return P.modspec_smoothing(x, 200, n=n, cutoff=30, lengths=lens)
    if mode == "grad":
        return _modspec_grad(x, G, n, "ortho", lens)
    nat, gen = _stats(n, x.shape[2])
    return modspec_post_filter(x, nat, gen, k=0.8, n=n, lengths=lens)


def _big_ref(mode, n, x, L, G):
    """float64 reference of one utterance of L frames, frames padded with 0 to the batch's T."""
    T, D = x.shape
    if mode == "power":
        return np.abs(np.fft.rfft(x[:L].astype(np.float64), n, axis=0)) ** 2
    out = np.zeros((T, D))
    if L:
        if mode == "smooth":
            out[:L] = _smooth_ref(x[:L], n, None, int(n * 30 / 200) + 1, True)
        elif mode == "grad":
            out[:L] = _grad_ref(x[:L], G, n, "ortho")
        else:
            nat, gen = _stats(n, D)
            out[:L] = O.post_filter(x[:L], nat, gen, 0.8, n)
    return out


@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("mode,n", [("power", 256), ("smooth", 4096), ("grad", 4096), ("postfilter", 256)])
def test_more_utterances_than_one_grid(mode, n, dt):
    """65 540 distinct utterances, lengths cycling through 0, 1, 5 and T, NaN past each length.  The batch must
    equal, bit for bit, the same utterances in two calls of fewer than 65 535 (one pass of the utterance loop
    each); every utterance from 65 535 on, which a CTA reaches on its second pass, must equal its own call and
    the reference."""
    import torch
    dtype = DT[dt]
    T, D = 8, 1 if mode == "grad" else 2
    K = n // 2 + 1
    rng = np.random.default_rng([n, 5, MODES[mode], dt == "f32"])
    lens = np.resize(np.array([0, 1, 5, T]), BIG_B)
    x = rng.standard_normal((BIG_B, T, D)).astype(dtype)
    pad = np.arange(T)[None, :] >= lens[:, None]
    x[pad] = np.nan
    xt = _cuda(x)
    G = None
    if mode == "grad":
        g = torch.Generator(device="cuda").manual_seed(n)
        G = torch.randn((BIG_B, K, D), dtype=xt.dtype, device="cuda", generator=g)
    got = _big_run(mode, n, xt, lens, G)
    assert got.shape == ((BIG_B, K, D) if mode == "power" else (BIG_B, T, D)) and torch.isfinite(got).all()
    cut = BIG_B // 2
    halves = torch.cat([_big_run(mode, n, xt[:cut], lens[:cut], None if G is None else G[:cut]),
                        _big_run(mode, n, xt[cut:], lens[cut:], None if G is None else G[cut:])])
    assert _same(got, halves)
    if mode != "power":
        assert not got[torch.from_numpy(pad).cuda()].any()
    for b in range(65535, BIG_B):
        one = _big_run(mode, n, xt[b:b + 1], lens[b:b + 1], None if G is None else G[b:b + 1])
        assert _same(got[b], one[0]), b
        want = _big_ref(mode, n, x[b], int(lens[b]), None if G is None else _np(G[b]))
        if want.any():
            _check(_np(got[b]), want, mode, n, dtype, ("utterance", b))
        else:
            assert not got[b].any(), b


# ---- 5. the C ABI: length clip, T_in != T_out, nothing to do, argument errors -------------------------------------
def _abi(mode, dtype, n, inp, in2, out, out2, B, T_in, T_out, D, lens, limit_bin=0, log_domain=0):
    import torch

    from nnmnkwii_b200 import _lib

    def ptr(t):
        return None if t is None else (torch.view_as_real(t) if t.is_complex() else t).data_ptr()
    code = _lib.NNK_F32 if np.dtype(dtype) == np.float32 else _lib.NNK_F64
    return _lib.lib.nnk_modspec(MODES[mode], code, n, ptr(inp), ptr(in2), ptr(out), ptr(out2), B, T_in, T_out, D,
                                ptr(lens), 1.0, 1.0 / n, limit_bin, log_domain,
                                torch.cuda.current_stream().cuda_stream)


def _abi_inputs(mode, dtype, n, B, T_in, D, rng):
    """(in, in2) of `mode`: frames (B, T_in, D), or for the inverse a power and unit phases (B, K, D); in2 is G for
    the gradient and the (K, D, 2) table (a, c) for the post-filter."""
    import torch
    K = n // 2 + 1
    cdt = np.complex64 if np.dtype(dtype) == np.float32 else np.complex128
    if mode == "inverse":
        return (_cuda(rng.exponential(size=(B, K, D)).astype(dtype)),
                _cuda(np.exp(2j * np.pi * rng.random((B, K, D))).astype(cdt)))
    x = _cuda(rng.standard_normal((B, T_in, D)).astype(dtype))
    if mode == "grad":
        return x, _cuda(rng.standard_normal((B, K, D)).astype(dtype))
    if mode == "postfilter":
        return x, _cuda(np.stack([rng.uniform(0.5, 1.5, (K, D)), rng.uniform(-1, 1, (K, D))], -1).astype(dtype))
    return x, torch.empty(0)


SPECTRUM = ("power", "logpower")
CLIP_SHAPES = {  # (T_in, T_out) at n = 256: frames past n, T_in < n, T_out below and above T_in
    "power": [(264, 0), (20, 0)], "logpower": [(264, 0), (20, 0)], "inverse": [(0, 264), (0, 20)],
    "smooth": [(264, 264), (40, 25), (25, 40)], "grad": [(264, 264), (40, 25), (25, 40)],
    "postfilter": [(264, 264), (40, 25), (25, 40)],
}


@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("mode", list(MODES))
def test_abi_length_clip(mode, dt):
    """Lengths -3, 0, n + 5, past T_in (or T_out) and 7 give the bits of the same call on lengths clipped to
    [0, min(n, T_in, T_out)] (T_in where the mode reads frames, T_out where it writes them); every output element
    is written (the buffers start as NaN), frames from the clipped length on as 0."""
    import torch

    from nnmnkwii_b200 import _lib
    dtype, n, B, D = DT[dt], 256, 5, 3
    K = n // 2 + 1
    rng = np.random.default_rng([MODES[mode], dt == "f32"])
    for T_in, T_out in CLIP_SHAPES[mode]:
        inp, in2 = _abi_inputs(mode, dtype, n, B, T_in, D, rng)
        in2 = in2 if in2.numel() else None
        cap = n
        if mode != "inverse":
            cap = min(cap, T_in)
        if mode not in SPECTRUM:
            cap = min(cap, T_out)
        raw = np.array([-3, 0, n + 5, max(T_in, T_out) + 2, 7], np.int32)
        clipped = np.clip(raw, 0, cap).astype(np.int32)

        def run(lens):
            shape = (B, K, D) if mode in SPECTRUM else (B, T_out, D)
            out = torch.full(shape, float("nan"), dtype=inp.dtype, device="cuda")
            cdt = torch.complex64 if dtype == np.float32 else torch.complex128
            out2 = torch.full(shape, complex("nan+nanj"), dtype=cdt, device="cuda") if mode == "power" else None
            c0 = _lib.launch_count()
            assert _abi(mode, dtype, n, inp, in2, out, out2, B, T_in, T_out, D, _cuda(lens), 20, 1) == _lib.NNK_OK
            assert _lib.launch_count() - c0 == 1
            return out, out2

        tag = (T_in, T_out)
        out, out2 = run(raw)
        want, want2 = run(clipped)
        assert not torch.isnan(out).any(), tag
        assert _same(out, want), tag
        if out2 is not None:
            assert not torch.isnan(torch.view_as_real(out2)).any() and _same(out2, want2), tag
        if mode not in SPECTRUM:
            for b, L in enumerate(clipped):
                assert not out[b, L:].any(), (tag, b)
        if mode == "smooth" and dtype == np.float64:  # the frames a call reads are the clipped ones
            x = _np(inp)
            for b, L in enumerate(clipped):
                if L:
                    _check(_np(out[b, :L]), _smooth_ref(x[b, :L], n, None, 20, True), "smooth", n, dtype, tag + (b,))


def test_abi_calls_that_launch_nothing():
    """B = 0, D = 0 and T_out = 0 in a frame mode return NNK_OK without a launch; every argument error returns
    NNK_ERR_ARG without one.  No output element is touched."""
    import torch

    from nnmnkwii_b200 import _lib
    n, B, T, D, K = 256, 2, 30, 3, 129
    rng = np.random.default_rng(6)
    x, G = _abi_inputs("grad", np.float64, n, B, T, D, rng)
    ms, ph = _abi_inputs("inverse", np.float64, n, B, T, D, rng)
    table = _abi_inputs("postfilter", np.float64, n, B, T, D, rng)[1]
    spec = torch.full((B, K, D), float("nan"), dtype=torch.float64, device="cuda")
    spec2 = torch.full((B, K, D), complex("nan+nanj"), dtype=torch.complex128, device="cuda")
    frames = torch.full((B, T, D), float("nan"), dtype=torch.float64, device="cuda")
    lens = _cuda(np.array([T, 5], np.int32))
    in2 = {"power": None, "logpower": None, "smooth": None, "inverse": ph, "grad": G, "postfilter": table}

    def call(mode, rc, n=n, B=B, T_out=T, D=D, in2_=None, out2=None, **kw):
        c0 = _lib.launch_count()
        inp = ms if mode == "inverse" else x
        out = spec if mode in SPECTRUM else frames
        assert _abi(mode, np.float64, n, inp, in2[mode] if in2_ is None else in2_, out, out2, B,
                    T, 0 if mode in SPECTRUM else T_out, D, lens, **kw) == rc, (mode, n, B, T_out, D)
        torch.cuda.synchronize()
        assert _lib.launch_count() == c0, (mode, n, B, T_out, D)

    for mode in MODES:
        call(mode, _lib.NNK_OK, B=0)
        call(mode, _lib.NNK_OK, D=0)
        if mode not in SPECTRUM:
            call(mode, _lib.NNK_OK, T_out=0)
        for bad_n in (128, 8192, 768):
            call(mode, _lib.NNK_ERR_ARG, n=bad_n)
    call("logpower", _lib.NNK_ERR_ARG, out2=spec2)
    call("postfilter", _lib.NNK_ERR_ARG, out2=spec2)
    for mode in ("inverse", "grad", "postfilter"):
        null = torch.empty(0)  # data_ptr() of an empty tensor is NULL
        assert null.data_ptr() == 0
        call(mode, _lib.NNK_ERR_ARG, in2_=null)
    assert torch.isnan(spec).all() and torch.isnan(frames).all() and torch.isnan(torch.view_as_real(spec2)).all()
