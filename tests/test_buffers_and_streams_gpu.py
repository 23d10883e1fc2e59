"""Results that do not depend on what is already in a buffer, work that runs on the caller's stream only, and
cached device tables that outlive the kernels reading them.

Every public entry point that launches a kernel has a case in ``CATALOGUE``: seeded inputs, the call, the
family's own reference at its usual bar, and the outputs to compare.  Each case runs four ways, and every way
must give outputs bit-identical (NaN positions included) to the plain run:

1. plain, as users call it (and checked against the reference);
2. with every floating-point (real or complex) CUDA tensor from ``torch.empty`` / ``empty_like`` /
   ``Tensor.new_empty`` filled with 0xFF bytes (NaN), then with 0x7F bytes (a huge finite value).  Integer and
   uint8 allocations carry indices and workspace tables: they are zero-filled in all three runs, never filled with
   arbitrary bytes;
3. with every workspace request served by the block a larger valid call of the same entry point (other data,
   other lengths) just used, as that call left it (a spy on ``_device.workspace`` hands the blocks over and
   asserts that every request was served), compared with the case run straight after
   ``torch.cuda.empty_cache()``;
4. on a fresh side stream S behind a ~20 ms ``torch.cuda._sleep``: CUDA inputs are NaN on the default stream
   and only get their real values on S, outputs are copied on S and only S is synchronised.  Every launching C
   call must name S as its stream, and the legacy default stream is held by a longer sleep for the whole
   call, so that stray work on it cannot finish before S copies the outputs.

Every run starts with the cached device tables dropped, so that they are built under that run's poison.

The eviction tests hold a kernel back on a sleeping S while the default stream evicts the cache entry it
reads and refills the entry's block with valid other content."""
import contextlib
import math

import numpy as np
import pytest

import oracle
import stream_catalogue as SC
from conftest import rel_err, windows_set

pytestmark = pytest.mark.gpu

W2 = windows_set()[1]
W3 = windows_set()[2]
SLEEP_CYCLES = 40_000_000  # about 20 ms on an H100
LEGACY_HOLD_CYCLES = 600_000_000  # about 300 ms: longer than any case's call on the side stream
EVICT_SLEEP_CYCLES = 400_000_000  # about 200 ms: longer than evicting a cache from the default stream
REACHED = set()
RUN_CASES = set()


# ---- the recording proxy over the C ABI ---------------------------------------------------------------------------
# while STREAM_CHECK["on"], every launching call must pass the current stream as its last argument
STREAM_CHECK = {"on": False, "bad": []}


def _stream_value(arg):
    return int(getattr(arg, "value", arg) or 0)


@pytest.fixture(scope="module", autouse=True)
def _record_exports():
    import torch

    from nnmnkwii_b200 import _lib
    lib = _lib.lib
    saved = {}
    for name in SC.launching_exports(_lib.EXPORTS):
        fn = getattr(lib, name)
        saved[name] = fn

        def proxy(*a, _fn=fn, _name=name):
            REACHED.add(_name)
            if STREAM_CHECK["on"] and _name not in SC.EXPORTS_OWN_STREAMS:
                want = torch.cuda.current_stream().cuda_stream
                if _stream_value(a[-1]) != want:
                    STREAM_CHECK["bad"].append((_name, _stream_value(a[-1]), want))
            return _fn(*a)
        setattr(lib, name, proxy)
    yield
    for name, fn in saved.items():
        setattr(lib, name, fn)


# ---- allocation poison and the workspace spy ------------------------------------------------------------------------
@contextlib.contextmanager
def allocations(fill=None):
    """Patch torch.empty / empty_like / Tensor.new_empty (and _device.workspace): floating-point (real or complex)
    CUDA results get every byte set to ``fill`` (None: left as they are); integer, bool and uint8 results are
    zeroed."""
    import torch

    from nnmnkwii_b200 import _device as dev
    orig = (torch.empty, torch.empty_like, torch.Tensor.new_empty, dev.workspace)

    def treat(t):
        if isinstance(t, torch.Tensor) and t.is_cuda and t.numel():
            if t.is_floating_point() or t.is_complex():
                if fill is not None:
                    t.reshape(-1).view(torch.uint8).fill_(fill)
            else:
                t.zero_()
        return t

    def empty(*a, **k):
        return treat(orig[0](*a, **k))

    def empty_like(*a, **k):
        return treat(orig[1](*a, **k))

    def new_empty(self, *a, **k):
        return treat(orig[2](self, *a, **k))

    def workspace(device, nbytes):
        return treat(orig[3](device, nbytes))

    torch.empty, torch.empty_like, torch.Tensor.new_empty, dev.workspace = empty, empty_like, new_empty, workspace
    try:
        yield
    finally:
        torch.empty, torch.empty_like, torch.Tensor.new_empty, dev.workspace = orig


@contextlib.contextmanager
def recycled_workspace(kept, served):
    """Spy on _device.workspace.  With ``served`` None, every block is appended to ``kept`` (and so stays
    allocated).  Otherwise the i-th request gets the first bytes of ``kept[i]``, exactly as that earlier call
    left them, and appends True to ``served``; a request larger than that block appends False and gets a
    fresh allocation."""
    from nnmnkwii_b200 import _device as dev
    orig = dev.workspace

    def spy(device, nbytes):
        if served is None:
            ws = orig(device, nbytes)
            kept.append(ws)
            return ws
        n = int(max(nbytes, 256))
        i = len(served)
        ok = i < len(kept) and kept[i].numel() >= n
        served.append(ok)
        return kept[i][:n] if ok else orig(device, nbytes)
    dev.workspace = spy
    try:
        yield
    finally:
        dev.workspace = orig


# ---- comparing outputs ----------------------------------------------------------------------------------------------
def _as_tensor(o):
    import torch
    if isinstance(o, torch.Tensor):
        return o.detach().cpu()
    if isinstance(o, np.ndarray) or isinstance(o, np.generic):
        return torch.from_numpy(np.array(o, copy=True))
    return torch.tensor(o)


def same(a, b):
    """Bit-identical outputs: equal shapes, dtypes, NaN positions and every other value."""
    import torch
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        x, y = _as_tensor(x), _as_tensor(y)
        assert x.dtype == y.dtype and x.shape == y.shape, (k, x.dtype, y.dtype, x.shape, y.shape)
        if x.is_complex():
            x, y = torch.view_as_real(x), torch.view_as_real(y)
        if x.is_floating_point():
            nx, ny = torch.isnan(x), torch.isnan(y)
            assert torch.equal(nx, ny), "output %d: NaN positions differ (%d vs %d NaN)" % (k, int(nx.sum()), int(ny.sum()))
            x, y = torch.where(nx, 0, x), torch.where(ny, 0, y)
        assert torch.equal(x, y), "output %d differs (max |diff| %s)" % (
            k, (x.double() - y.double()).abs().max().item() if x.numel() else None)


def _h(o):
    """A NumPy copy of a tensor / array output."""
    import torch
    return o.detach().cpu().numpy() if isinstance(o, torch.Tensor) else np.asarray(o)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ---- the catalogue ----------------------------------------------------------------------------------------------------
class Case(object):
    """``make(rng, big)`` -> dict of inputs (NumPy arrays, CUDA tensors, anything else); ``big`` asks for another
    valid call with larger shapes.  ``call(inp)`` -> list of outputs.  ``check(inp, out)`` asserts the family's
    reference bar.  ``ws``: the call takes scratch from _device.workspace.  ``prepare(inp)`` runs before the
    call, on the default stream in the side-stream way (objects constructed once, stepped later)."""

    def __init__(self, name, covers, make, call, check, ws=False, prepare=None):
        self.name, self.covers, self.make, self.call, self.check, self.ws = name, covers, make, call, check, ws
        self.prepare = prepare or (lambda inp: inp)


CATALOGUE = []


def case(name, covers, ws=False, prepare=None):
    def deco(fn):
        make, call, check = fn()
        CATALOGUE.append(Case(name, covers, make, call, check, ws, prepare))
        return fn
    return deco


def _G():
    from nnmnkwii_b200 import paramgen
    return paramgen


def _mv(rng, T, D, dt, var_global=False):
    m = rng.standard_normal((T, D)).astype(dt)
    v = ((rng.random(D) if var_global else rng.random((T, D))) + 0.1).astype(dt)
    return m, v


def _lens(rng, n, lo, hi):
    return rng.integers(lo, hi, n).astype(np.int64)


MS_N = 512  # DFT length of the modulation-spectrum cases


def _nan_padded(rng, lens, T, D, dt):
    """(B, T, D): utterance b is lens[b] frames of noise through 1 + 0.7 z^-1, then NaN padding."""
    x = np.full((len(lens), T, D), np.nan, dt)
    for b, L in enumerate(lens):
        w = rng.standard_normal((L + 1, D))
        x[b, :L] = w[1:] + 0.7 * w[:-1]
    return x


def _crel(a, b):
    """max |a - b| / max |b| of complex arrays."""
    a, b = np.asarray(a, np.complex128), np.asarray(b, np.complex128)
    return float(np.abs(a - b).max() / max(1e-300, np.abs(b).max()))


# ---- paramgen ----
@case("mlpg_numpy_f64_per_frame", [("paramgen", "mlpg")])
def _c():
    def make(rng, big):
        m, v = _mv(rng, 60 if big else 33, 3 * (7 if big else 5), np.float64)
        return {"m": m, "v": v}
    return (make, lambda i: [_G().mlpg(i["m"], i["v"], W3)],
            lambda i, o: _bar(rel_err(o[0], oracle.mlpg(i["m"], i["v"], W3)) < 1e-10))


@case("mlpg_cuda_f32_global_var", [("paramgen", "mlpg")], ws=True)
def _c():
    def make(rng, big):
        m, v = _mv(rng, 70 if big else 41, 3 * (9 if big else 6), np.float32, var_global=True)
        return {"m": _cuda(m), "v": _cuda(v)}
    return (make, lambda i: [_G().mlpg(i["m"], i["v"], W3)],
            lambda i, o: _bar(rel_err(_h(o[0]), oracle.mlpg(_h(i["m"]), np.tile(_h(i["v"]), (i["m"].shape[0], 1)),
                                                            W3)) < 1e-6))


def _merlin_ref(m, v, lens, y):
    off = np.concatenate([[0], np.cumsum(lens)])
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        if b > a:
            ref = oracle.mlpg(m[a:b, :180].astype(np.float64), v[a:b, :180].astype(np.float64), W3)
            _bar(rel_err(y[a:b, :60], ref) < 1e-6)
            _bar(np.array_equal(y[a:b, 61], m[a:b, 183]))  # vuv is copied


@case("mlpg_batch_cuda_flat_merlin_f32", [("paramgen", "mlpg_batch")], ws=True)
def _c():
    def make(rng, big):
        lens = _lens(rng, 5 if big else 3, 2, 90 if big else 50)
        m, v = _mv(rng, int(lens.sum()), 187, np.float32)
        return {"m": _cuda(m), "v": _cuda(v), "lens": lens}
    return (make, lambda i: [_G().mlpg_batch(i["m"], i["v"], W3, lengths=i["lens"], layout=_G().merlin_layout())],
            lambda i, o: _merlin_ref(_h(i["m"]), _h(i["v"]), i["lens"], _h(o[0])))


@case("mlpg_batch_numpy_flat_merlin_f64", [("paramgen", "mlpg_batch")])
def _c():
    def make(rng, big):
        lens = _lens(rng, 4 if big else 3, 3, 80 if big else 40)
        m, v = _mv(rng, int(lens.sum()), 187, np.float64)
        return {"m": m, "v": v, "lens": lens}
    return (make, lambda i: [_G().mlpg_batch(i["m"], i["v"], W3, lengths=i["lens"], layout=_G().merlin_layout())],
            lambda i, o: _merlin_ref(i["m"], i["v"], i["lens"], o[0]))


def _padded(rng, lens, D, dt, pad_value=0.0):
    B, Tmax = len(lens), int(max(lens))
    m = np.full((B, Tmax, D), pad_value, dtype=dt)
    v = np.ones((B, Tmax, D), dtype=dt)
    for b, n in enumerate(lens):
        m[b, :n], v[b, :n] = _mv(rng, int(n), D, dt)
    return m, v


@case("mlpg_batch_cuda_padded_f64", [("paramgen", "mlpg_batch")], ws=True)
def _c():
    def make(rng, big):
        lens = np.array([30, 1, 17, 0, 44])[: 5 if big else 4] + (9 if big else 0)
        m, v = _padded(rng, lens, 3 * 4, np.float64)
        return {"m": _cuda(m), "v": _cuda(v), "lens": lens}

    def check(i, o):
        m, v, y = _h(i["m"]), _h(i["v"]), _h(o[0])
        for b, n in enumerate(i["lens"]):
            if n:
                _bar(rel_err(y[b, :n], oracle.mlpg(m[b, :n], v[b, :n], W3)) < 1e-10)
            _bar(not y[b, n:].any())
    return make, lambda i: [_G().mlpg_batch(i["m"], i["v"], W3, lengths=i["lens"])], check


@case("mlpg_grad_cuda_f32_go", [("paramgen", "mlpg_grad")], ws=True)
def _c():
    def make(rng, big):
        T, sd = (64, 7) if big else (37, 5)
        m, v = _mv(rng, T, 3 * sd, np.float32)
        return {"m": _cuda(m), "v": _cuda(v), "go": _cuda(rng.standard_normal((T, sd)).astype(np.float32))}
    return (make, lambda i: [_G().mlpg_grad(i["m"], i["v"], W3, i["go"])],
            lambda i, o: _bar(rel_err(_h(o[0]), oracle.mlpg_grad(_h(i["m"]), _h(i["v"]), W3, _h(i["go"]))) < 2e-6))


@case("mlpg_grad_numpy_f64_go", [("paramgen", "mlpg_grad")], ws=True)
def _c():
    def make(rng, big):
        T, sd = (50, 6) if big else (29, 4)
        m, v = _mv(rng, T, 2 * sd, np.float64)
        return {"m": m, "v": v, "go": rng.standard_normal((T, sd))}
    return (make, lambda i: [_G().mlpg_grad(i["m"], i["v"], W2, i["go"])],
            lambda i, o: _bar(rel_err(o[0], oracle.mlpg_grad(i["m"], i["v"], W2, i["go"])) < 2e-6))


def _grad_batch_check(i, o):
    v, go, g = _h(i["v"]), _h(i["go"]), _h(o[0])
    for b, n in enumerate(i["lens"]):
        if n:
            ref = oracle.mlpg_grad(np.zeros_like(v[b, :n]), v[b, :n], W3, go[b, :n].astype(np.float64))
            _bar(rel_err(g[b, :n], ref) < 2e-6)
        _bar(not g[b, n:].any())


@case("mlpg_grad_batch_cuda_padded_f32_go", [("paramgen", "mlpg_grad_batch")], ws=True)
def _c():
    def make(rng, big):
        lens = np.array([25, 3, 0, 40])[: 4 if big else 3] + (8 if big else 0)
        _, v = _padded(rng, lens, 3 * 5, np.float32)
        go = rng.standard_normal((len(lens), int(lens.max()), 5)).astype(np.float32)
        return {"v": _cuda(v), "go": _cuda(go), "lens": lens}
    return make, lambda i: [_G().mlpg_grad_batch(i["v"], W3, i["go"], i["lens"])], _grad_batch_check


@case("mlpg_grad_batch_cuda_padded_f64_go", [("paramgen", "mlpg_grad_batch")], ws=True)
def _c():
    def make(rng, big):
        lens = np.array([19, 1, 33])[: 3] + (11 if big else 0)
        _, v = _padded(rng, lens, 3 * 3, np.float64)
        go = rng.standard_normal((len(lens), int(lens.max()), 3))
        return {"v": _cuda(v), "go": _cuda(go), "lens": lens}
    return make, lambda i: [_G().mlpg_grad_batch(i["v"], W3, i["go"], i["lens"])], _grad_batch_check


@case("unit_variance_mlpg_matrix_solve", [("paramgen", "unit_variance_mlpg_matrix")], ws=True)
def _c():
    def make(rng, big):
        return {"T": 61 if big else 26}
    return (make, lambda i: [_G().unit_variance_mlpg_matrix(W3, i["T"])],
            lambda i, o: _bar(np.abs(o[0] - oracle.unit_variance_mlpg_matrix(W3, i["T"])).max() < 2e-7))


def _gv_model(rng, sd):
    return np.full(sd, 0.05) + 0.01 * rng.random(sd), np.full(sd, 1e-4)


@case("mlpg_gv_numpy_f64", [("paramgen", "mlpg_gv")], ws=True)
def _c():
    import oracle.gv as ogv

    def make(rng, big):
        T, sd = (60, 6) if big else (40, 4)
        m, v = _mv(rng, T, 3 * sd, np.float64)
        gm, gvv = _gv_model(rng, sd)
        return {"m": m * 0.3, "v": v, "gm": gm, "gv": gvv}
    return (make, lambda i: [_G().mlpg_gv(i["m"], i["v"], W3, i["gm"], i["gv"], n_iter=5)],
            lambda i, o: _bar(np.abs(o[0] - ogv.mlpg_gv(i["m"], i["v"], W3, i["gm"], i["gv"], n_iter=5)).max()
                              <= 1e-8 * np.abs(o[0]).max()))


@case("mlpg_gv_batch_cuda_padded_f64", [("paramgen", "mlpg_gv_batch")], ws=True)
def _c():
    import oracle.gv as ogv

    def make(rng, big):
        lens = np.array([35, 2, 20])[: 3] + (15 if big else 0)
        m, v = _padded(rng, lens, 3 * 3, np.float64)
        gm, gvv = _gv_model(rng, 3)
        return {"m": _cuda(m * 0.3), "v": _cuda(v), "lens": lens, "gm": gm, "gv": gvv}

    def check(i, o):
        m, v, y = _h(i["m"]), _h(i["v"]), _h(o[0])
        for b, n in enumerate(i["lens"]):
            ref = ogv.mlpg_gv(m[b, :n], v[b, :n], W3, i["gm"], i["gv"], n_iter=5)
            _bar(np.abs(y[b, :n] - ref).max() <= 1e-8 * max(1e-300, np.abs(ref).max()))
            _bar(not y[b, n:].any())
    return make, lambda i: [_G().mlpg_gv_batch(i["m"], i["v"], W3, i["gm"], i["gv"], lengths=i["lens"], n_iter=5)], check


@case("global_variance_and_gv_statistics", [("paramgen", "global_variance"), ("paramgen", "gv_statistics")])
def _c():
    def make(rng, big):
        lens = _lens(rng, 6 if big else 4, 1, 40)
        return {"x": _cuda((rng.standard_normal((int(lens.sum()), 33)) + 1e3).astype(np.float32)), "lens": lens}

    def call(i):
        G = _G()
        return [G.global_variance(i["x"], lengths=i["lens"])] + list(G.gv_statistics(i["x"], lengths=i["lens"]))

    def check(i, o):
        x = _h(i["x"]).astype(np.float64)
        off = np.concatenate([[0], np.cumsum(i["lens"])])
        gv = np.stack([x[off[u]:off[u + 1]].var(axis=0) for u in range(len(i["lens"]))])
        _bar(rel_err(_h(o[0]), gv) < 1e-12)
        _bar(rel_err(_h(o[1]), gv.mean(axis=0)) < 1e-12 and rel_err(_h(o[2]), gv.var(axis=0)) < 1e-10)
    return make, call, check


MS_MARGIN = 1e-9  # an accept decision whose relative margin is below this could flip under rounding


def _ms_walk(rng, T, sd):
    """Means (T, 3 sd) whose static part is a smooth walk, per-frame variances (tests/test_ms_gen_gpu.py)."""
    m = np.concatenate([np.cumsum(rng.standard_normal((T, sd)), 0) * 0.1, 0.05 * rng.standard_normal((T, 2 * sd))], 1)
    return m, rng.random((T, 3 * sd)) + 0.5


def _ms_clear(ref_fn):
    """The restatement's result, asserting that every accept decision on its path is clear of rounding (margin
    inf: the trial moves c by at most 1e-11 of its size, so either decision gives the same result)."""
    traces = []
    ref = ref_fn(traces)
    worst = min(t[2] for tr in traces for t in tr)
    _bar(worst > MS_MARGIN)
    return ref


def _ms_check(i, o, ref_fn):
    """Every utterance of the batch (o[0]) and the single-utterance call (o[1], utterance i["one"]) within 1e-9
    of the restatement ``ref_fn(m, v, traces)``."""
    m, v, y = _h(i["m"]), _h(i["v"]), _h(o[0])
    off = np.concatenate([[0], np.cumsum(i["lens"])])
    for u in range(len(i["lens"])):
        a, b = off[u], off[u + 1]
        if b > a:
            ref = _ms_clear(lambda tr: ref_fn(m[a:b], v[a:b], tr))
            _bar(np.abs(y[a:b] - ref).max() <= 1e-9 * np.abs(ref).max())
            if u == i["one"]:
                _bar(np.abs(_h(o[1]) - ref).max() <= 1e-9 * np.abs(ref).max())


MS_ARGS = dict(n_iter=4, step=0.1, weight=1.0)  # on these inputs some trials are accepted and some rejected


def _ms_call(i, **kw):
    G = _G()
    a, b = (int(x) for x in np.cumsum(i["lens"])[i["one"] - 1:i["one"] + 1])
    return [G.mlpg_ms_batch(i["m"], i["v"], W3, i["mm"], i["mv"], lengths=i["lens"], **MS_ARGS, **kw),
            G.mlpg_ms(i["m"][a:b], i["v"][a:b], W3, i["mm"], i["mv"], **MS_ARGS, **kw)]


@case("mlpg_ms_batch_and_mlpg_ms_f64", [("paramgen", "mlpg_ms_batch"), ("paramgen", "mlpg_ms")], ws=True)
def _c():
    import oracle.ms_gen as OMS

    def make(rng, big):
        n, sd = (2048, 8) if big else (1024, 6)
        lens = [1500, 30, 0, 2000, 40] if big else [900, 17, 0, 1024]
        m, v = _ms_walk(rng, sum(lens), sd)
        nat = rng.standard_normal((8, n, sd)) * 0.3 + np.cumsum(rng.standard_normal((8, n, sd)), 1) * 0.05
        s = np.log(np.maximum(np.abs(np.fft.rfft(nat, n, axis=1)) ** 2, OMS.TINY))
        return {"m": _cuda(m), "v": _cuda(v), "lens": lens, "one": 3, "mm": s.mean(0), "mv": s.var(0) + 0.5}

    return make, _ms_call, lambda i, o: _ms_check(
        i, o, lambda m, v, tr: OMS.mlpg_ms(m, v, W3, i["mm"], i["mv"], traces=tr, **MS_ARGS))


@case("mlpg_ms_batch_and_mlpg_ms_segment_f64", [("paramgen", "mlpg_ms_batch"), ("paramgen", "mlpg_ms")], ws=True)
def _c():
    import ms_gen_segment_oracle as OMSS
    import oracle.ms_segment as oseg
    n = L = 128

    def make(rng, big):
        sd = 8 if big else 6
        lens = [9500, 30, 0, 1100, 40] if big else [9000, 17, 0, 1024]
        m, v = _ms_walk(rng, sum(lens), sd)
        nat = rng.standard_normal((4, 4 * n, sd)) * 0.3 + np.cumsum(rng.standard_normal((4, 4 * n, sd)), 1) * 0.05
        mean, var = oseg.statistics(list(nat), n, L)
        return {"m": _cuda(m), "v": _cuda(v), "lens": lens, "one": 3, "mm": mean, "mv": var + 0.5}

    return make, lambda i: _ms_call(i, segment=L), lambda i, o: _ms_check(
        i, o, lambda m, v, tr: OMSS.mlpg_ms(m, v, W3, i["mm"], i["mv"], L, traces=tr, **MS_ARGS))


def _merlin_like(D):
    """The Merlin layout with D - 7 mgc columns (D = 187: merlin_layout()); the larger calls use D = 211."""
    mgc = D - 7
    return _G().StreamLayout(D, [(0, mgc // 3), (mgc, 1), (mgc + 3, 1, "copy"), (mgc + 4, 1)])


MERLIN_STREAMS = [(0, 60), (180, 1), (183, 1, "copy"), (184, 1)]


@case("mlpg_mixture_batch_and_mlpg_mixture_merlin_f64", [("paramgen", "mlpg_mixture_batch"),
                                                          ("paramgen", "mlpg_mixture")], ws=True)
def _c():
    def make(rng, big):
        lens, M, D = ([1000, 30, 0, 400, 20], 8, 211) if big else ([900, 17, 0, 300], 8, 187)
        T = sum(lens)
        lw = rng.standard_normal((T, M)) * 0.5
        mu = np.cumsum(rng.standard_normal((T, M, D)), axis=0) * 0.1 + rng.standard_normal((1, M, D))
        s2 = rng.random((T, M, D)) * 0.5 + 0.1
        return {"lw": _cuda(lw), "mu": _cuda(mu), "s2": _cuda(s2), "lens": lens, "D": D}

    def call(i):
        G = _G()
        y, L = G.mlpg_mixture_batch(i["lw"], i["mu"], i["s2"], W3, lengths=i["lens"],
                                    layout=_merlin_like(i["D"]), n_iter=4, return_log_likelihood=True)
        T, mgc = i["lens"][0], i["D"] - 7
        y1, L1 = G.mlpg_mixture(i["lw"][:T], i["mu"][:T, :, :mgc].contiguous(), i["s2"][:T, :, :mgc].contiguous(),
                                W3, n_iter=4, return_log_likelihood=True)
        return [y, L, y1, L1]

    def check(i, o):
        import mix_gen_oracle as OMG
        lw, mu, s2, y, L = _h(i["lw"]), _h(i["mu"]), _h(i["s2"]), _h(o[0]), _h(o[1])
        off = np.concatenate([[0], np.cumsum(i["lens"])])
        for u in range(len(i["lens"])):
            a, b = off[u], off[u + 1]
            if a == b:
                _bar(np.all(L[u] == 0.0))
                continue
            want, Lw = OMG.mlpg_mixture(lw[a:b], mu[a:b], s2[a:b], W3, 4, streams=MERLIN_STREAMS)
            _bar(rel_err(y[a:b], want) <= 1e-9 and np.all(np.abs(L[u] - Lw) <= 1e-10 * np.abs(Lw)))
        T = i["lens"][0]
        want, Lw = OMG.mlpg_mixture(lw[:T], mu[:T, :, :180], s2[:T, :, :180], W3, 4)
        _bar(rel_err(_h(o[2]), want) <= 1e-9 and np.all(np.abs(_h(o[3]) - Lw) <= 1e-10 * np.abs(Lw)))
    return make, call, check


def _traj_data(rng, lens, D, D_out):
    """Targets, means and per-frame variances of the trajectory-model tests, float64."""
    n = sum(lens)
    m = np.cumsum(rng.standard_normal((n, D)), axis=0) * 0.05 + rng.standard_normal((n, D)) * 0.3
    v = rng.random((n, D)) + 0.5
    x = np.cumsum(rng.standard_normal((n, D_out)), axis=0) * 0.05 + rng.standard_normal((n, D_out)) * 0.2
    return x, m, v


def _traj_make(rng, big):
    lens, D = ([1000, 30, 400, 20], 211) if big else ([900, 17, 300], 187)
    x, m, v = _traj_data(rng, lens, D, (D - 7) // 3 + 3)
    go = rng.standard_normal((sum(lens), (D - 7) // 3 + 3))
    return {"x": _cuda(x), "m": _cuda(m), "v": _cuda(v), "vg": _cuda(rng.random(D) + 0.5), "go": _cuda(go),
            "lens": lens, "D": D}


def _one(i, k):
    """Utterance 0 of input ``k`` in the single-stream layout: the mgc columns (the static ones of targets)."""
    T, mgc = i["lens"][0], i["D"] - 7
    return i[k][:T, :mgc // 3 if k == "x" else mgc].contiguous()


@case("trajectory_log_likelihood_batch_single_and_autograd_merlin_f64",
      [("paramgen", "trajectory_log_likelihood_batch"), ("paramgen", "trajectory_log_likelihood"),
       ("autograd", "TrajectoryLogLikelihood")], ws=True)
def _c():
    def call(i):
        import torch
        G, lay = _G(), _merlin_like(i["D"])
        ll = G.trajectory_log_likelihood_batch(i["x"], i["m"], i["v"], W3, lengths=i["lens"], layout=lay)
        ll1 = G.trajectory_log_likelihood(_one(i, "x"), _one(i, "m"), _one(i, "v"), W3)
        x, m, v = (i[k].clone().requires_grad_(True) for k in ("x", "m", "v"))
        la = _AF().TrajectoryLogLikelihood.apply(x, m, v, W3, i["lens"], lay)
        la.backward(torch.ones_like(la))
        return [ll, ll1, la.detach(), x.grad, m.grad, v.grad]

    def check(i, o):
        from test_traj_ll_gpu import _compare, _oracle_batch
        x, m, v = (_h(i[k]) for k in ("x", "m", "v"))
        ll, gm, gv, gx = _oracle_batch(x, m, v, W3, i["lens"], MERLIN_STREAMS)
        _compare([_h(o[2]), _h(o[4]), _h(o[5]), _h(o[3])], (ll, gm, gv, gx), "autograd")
        _bar(np.all(np.abs(_h(o[0]) - ll) <= 1e-11 * np.maximum(1.0, np.abs(ll))))
        T = i["lens"][0]
        ll1 = _oracle_batch(x[:T, :60], m[:T, :180], v[:T, :180], W3, [T])[0][0]
        _bar(np.all(np.abs(_h(o[1]) - ll1) <= 1e-11 * np.maximum(1.0, np.abs(ll1))))
    return _traj_make, call, check


@case("trajectory_sample_batch_and_single_merlin_f64", [("paramgen", "trajectory_sample_batch"),
                                                         ("paramgen", "trajectory_sample")], ws=True)
def _c():
    def call(i):
        G = _G()
        return [G.trajectory_sample_batch(i["m"], i["v"], W3, n_samples=3, seed=16, lengths=i["lens"],
                                          layout=_merlin_like(i["D"])),
                G.trajectory_sample(_one(i, "m"), _one(i, "v"), W3, n_samples=3, seed=16)]

    def check(i, o):
        from test_traj_sample_gpu import _compare, _oracle
        m, v = _h(i["m"]), _h(i["v"])
        _compare(_h(o[0]), _oracle(m, v, W3, i["lens"], 3, 16, streams=MERLIN_STREAMS), "batch")
        T = i["lens"][0]
        _compare(_h(o[1]), _oracle(m[:T, :180], v[:T, :180], W3, [T], 3, 16), "single")
    return _traj_make, call, check


@case("mlpg_vjp_batch_and_MLPGWithVariances_merlin_f64", [("paramgen", "mlpg_vjp_batch"),
                                                           ("autograd", "MLPGWithVariances")], ws=True)
def _c():
    def call(i):
        G, lay = _G(), _merlin_like(i["D"])
        out = list(G.mlpg_vjp_batch(i["m"], i["v"], W3, i["go"], lengths=i["lens"], layout=lay))
        out += list(G.mlpg_vjp_batch(i["m"], i["vg"], W3, i["go"], lengths=i["lens"], layout=lay))
        m, v = i["m"].clone().requires_grad_(True), i["v"].clone().requires_grad_(True)
        y = _AF().MLPGWithVariances.apply(m, v, W3, i["lens"], lay)
        y.backward(i["go"])
        return out + [y.detach(), m.grad, v.grad]

    def check(i, o):
        from test_mlpg_vjp_gpu import _compare, _oracle_batch
        m, v, vg, go = (_h(i[k]) for k in ("m", "v", "vg", "go"))
        want = _oracle_batch(m, v, W3, go, i["lens"], MERLIN_STREAMS)
        _compare([_h(o[0]), _h(o[1])], want, "per-frame")
        _compare([_h(o[2]), _h(o[3])], _oracle_batch(m, vg, W3, go, i["lens"], MERLIN_STREAMS), "(D,)")
        _merlin_ref(m, v, i["lens"], _h(o[4]))
        _compare([_h(o[5]), _h(o[6])], want, "autograd")
    return _traj_make, call, check


# ---- autograd ----
def _AF():
    from nnmnkwii_b200 import autograd
    return autograd


@case("autograd_MLPG_forward_backward", [("autograd", "MLPG")], ws=True)
def _c():
    def make(rng, big):
        T, sd = (55, 6) if big else (40, 5)
        m, v = _mv(rng, T, 3 * sd, np.float32)
        return {"m": _cuda(m), "v": _cuda(v), "go": _cuda(rng.standard_normal((T, sd)).astype(np.float32))}

    def call(i):
        mu = i["m"].clone().requires_grad_(True)
        y = _AF().MLPG.apply(mu, i["v"], W3)
        y.backward(i["go"])
        return [y.detach(), mu.grad]

    def check(i, o):
        m, v, go = _h(i["m"]), _h(i["v"]), _h(i["go"])
        _bar(rel_err(_h(o[0]), oracle.mlpg(m, v, W3)) < 1e-6)
        _bar(rel_err(_h(o[1]), oracle.mlpg_grad(m, v, W3, go)) < 2e-6)
    return make, call, check


@case("autograd_MLPGBatch_forward_backward", [("autograd", "MLPGBatch")], ws=True)
def _c():
    def make(rng, big):
        lens = np.array([30, 12, 1])[: 3] + (10 if big else 0)
        m, v = _padded(rng, lens, 3 * 4, np.float32)
        go = rng.standard_normal((3, int(lens.max()), 4)).astype(np.float32)
        return {"m": _cuda(m), "v": _cuda(v), "go": _cuda(go), "lens": lens}

    def call(i):
        mu = i["m"].clone().requires_grad_(True)
        y = _AF().MLPGBatch.apply(mu, i["v"], W3, i["lens"])
        y.backward(i["go"])
        return [y.detach(), mu.grad]

    def check(i, o):
        m, v, go, y, g = _h(i["m"]), _h(i["v"]), _h(i["go"]), _h(o[0]), _h(o[1])
        for b, n in enumerate(i["lens"]):
            _bar(rel_err(y[b, :n], oracle.mlpg(m[b, :n], v[b, :n], W3)) < 1e-6)
            _bar(rel_err(g[b, :n], oracle.mlpg_grad(m[b, :n], v[b, :n], W3, go[b, :n])) < 2e-6)
            _bar(not y[b, n:].any() and not g[b, n:].any())
    return make, call, check


def _toeplitz_R(rng, T, nw, K):
    """A dense R whose rows are all one random filter per window: the Toeplitz path (the taps do not factor)."""
    taps = rng.standard_normal((nw, 2 * K + 1)).astype(np.float32)
    R = np.zeros((T, nw * T), dtype=np.float32)
    for t in range(T):
        for w in range(nw):
            for k in range(-K, K + 1):
                if 0 <= t + k < T:
                    R[t, w * T + t + k] = taps[w, k + K]
    return R


def _uv_case(kind):
    def make(rng, big):
        if kind == "table":
            T = 40 if big else 32
            R = oracle.unit_variance_mlpg_matrix(W3, T).astype(np.float64)
        elif kind == "factored":
            T = 160 if big else 128
            R = oracle.unit_variance_mlpg_matrix(W3, T).astype(np.float32)
        else:
            T = 150 if big else 120
            R = _toeplitz_R(np.random.default_rng(5), T, 2, 3)
        nw = R.shape[1] // T
        x = rng.standard_normal((2, T, nw * 4)).astype(R.dtype)
        go = rng.standard_normal((2, T, 4)).astype(R.dtype)
        return {"R": _cuda(R), "x": _cuda(x), "go": _cuda(go)}

    def call(i):
        from nnmnkwii_b200 import _uvmlpg as uv
        mu = i["x"].clone().requires_grad_(True)
        y = _AF().UnitVarianceMLPG.apply(mu, i["R"])
        y.backward(i["go"])
        b = uv.band_of(i["R"], i["R"].device)
        path = "factored" if b.fact is not None else "toeplitz" if b.toep is not None else "table"
        assert path == kind, (path, kind)
        return [y.detach(), mu.grad]

    def check(i, o):
        R, x, go = _h(i["R"]).astype(np.float64), _h(i["x"]).astype(np.float64), _h(i["go"]).astype(np.float64)
        T = R.shape[0]
        nw = R.shape[1] // T
        Rm = R.reshape(T, nw, T)
        xs = x.reshape(2, T, nw, -1)
        y = np.einsum("tws,bswd->btd", Rm, xs)
        g = np.einsum("tws,btd->bswd", Rm, go).reshape(x.shape)
        tol = 1e-12 if kind == "table" else 1e-4
        _bar(rel_err(_h(o[0]), y) < tol and rel_err(_h(o[1]), g) < tol)
    return make, call, check


for _kind in ("table", "toeplitz", "factored"):
    CATALOGUE.append(Case("autograd_UnitVarianceMLPG_" + _kind, [("autograd", "UnitVarianceMLPG")],
                          *_uv_case(_kind)))


@case("autograd_ModSpec_and_ModSpecBatch_f64", [("autograd", "ModSpec"), ("autograd", "ModSpecBatch")])
def _c():
    K = MS_N // 2 + 1

    def make(rng, big):
        T, D = (200, 5) if big else (150, 4)
        lens = np.array([T, 1, 0, T // 3])
        return {"x": _cuda(_nan_padded(rng, [T], T, D, np.float64)[0]), "go": _cuda(rng.standard_normal((K, D))),
                "xb": _cuda(_nan_padded(rng, lens, T, D, np.float64)), "lens": lens,
                "gob": _cuda(rng.standard_normal((len(lens), K, D)))}

    def call(i):
        y = i["x"].clone().requires_grad_(True)
        ms = _AF().ModSpec.apply(y, MS_N, None)
        ms.backward(i["go"])
        yb = i["xb"].clone().requires_grad_(True)
        msb = _AF().ModSpecBatch.apply(yb, MS_N, "ortho", i["lens"])
        msb.backward(i["gob"])
        return [ms.detach(), y.grad, msb.detach(), yb.grad]

    def reference(x, G, scale):
        """scale |X|^2 and the reference's dense gradient scale * 2 G (R cos + I sin), kt = -2 pi k t / n."""
        X = np.fft.rfft(x, MS_N, axis=0)
        kt = -2 * np.pi / MS_N * np.arange(K)[:, None] * np.arange(len(x))
        grad = np.stack([G[:, d] @ (2 * (X.real[:, d, None] * np.cos(kt) + X.imag[:, d, None] * np.sin(kt)))
                         for d in range(x.shape[1])], axis=1)
        return scale * (X.real ** 2 + X.imag ** 2), scale * grad

    def check(i, o):
        o = [_h(t) for t in o]
        pw, g = reference(_h(i["x"]), _h(i["go"]), 1.0)
        _bar(rel_err(o[0], pw) < 1e-10 and rel_err(o[1], g) < 1e-10)
        xb, gob = _h(i["xb"]), _h(i["gob"])
        for b, L in enumerate(i["lens"]):
            pw, g = reference(xb[b, :L], gob[b], 1.0 / MS_N)  # norm "ortho": |X|^2 / n
            _bar(rel_err(o[2][b], pw) < 1e-10 and not o[3][b, L:].any())
            _bar(L == 0 or rel_err(o[3][b, :L], g) < 1e-10)
    return make, call, check


# ---- metrics ----
def _metric_inputs(rng, big):
    B, T = (4, 50) if big else (3, 30)
    lens = rng.integers(1, T + 1, B)
    X = rng.standard_normal((B, T, 24)).astype(np.float32)
    Y = X + 0.1 * rng.standard_normal(X.shape).astype(np.float32)
    f0 = rng.random((B, T)) + 4.0
    g0 = f0 + 0.01 * rng.standard_normal((B, T))
    vx, vy = (rng.random((B, T)) > 0.3).astype(np.float64), (rng.random((B, T)) > 0.3).astype(np.float64)
    return {"X": _cuda(X), "Y": _cuda(Y), "lens": lens, "f0": f0, "g0": g0, "vx": vx, "vy": vy}


@case("metrics_all_four", [("metrics", "melcd"), ("metrics", "mean_squared_error"),
                           ("metrics", "lf0_mean_squared_error"), ("metrics", "vuv_error")])
def _c():
    def call(i):
        from nnmnkwii_b200 import metrics as Mt
        return [Mt.melcd(i["X"], i["Y"], lengths=i["lens"]), Mt.melcd(i["X"][0], i["Y"][0]),
                Mt.mean_squared_error(i["X"], i["Y"], lengths=i["lens"]),
                Mt.lf0_mean_squared_error(i["f0"], i["vx"], i["g0"], i["vy"], lengths=i["lens"]),
                Mt.vuv_error(i["vx"], i["vy"], lengths=i["lens"])]

    def check(i, o):
        X, Y, lens = _h(i["X"]).astype(np.float64), _h(i["Y"]).astype(np.float64), i["lens"]
        mask = np.arange(X.shape[1])[None, :] < lens[:, None]
        _bar(abs(o[0] - oracle.melcd(X, Y, lens)) < 1e-5 * o[0])
        _bar(abs(o[1] - oracle.melcd(X[0], Y[0])) < 1e-5 * o[1])
        mse = math.sqrt(((X - Y) ** 2).sum(-1)[mask].sum() / (lens.sum() * X.shape[-1]))
        _bar(abs(o[2] - mse) < 1e-6 * mse)
        both = mask & (i["vx"] > 0) & (i["vy"] > 0)
        lf0 = math.sqrt(((i["f0"] - i["g0"]) ** 2)[both].mean())
        _bar(abs(o[3] - lf0) < 1e-10 * lf0)
        _bar(abs(o[4] - float((i["vx"] != i["vy"])[mask].sum()) / lens.sum()) < 1e-12)
    return _metric_inputs, call, check


# ---- preprocessing ----
def _P():
    from nnmnkwii_b200 import preprocessing
    return preprocessing


@case("delta_features_lengths", [("preprocessing", "delta_features")])
def _c():
    def make(rng, big):
        lens = _lens(rng, 4 if big else 3, 5, 40)
        return {"x": rng.standard_normal((int(lens.sum()), 9 if big else 7)).astype(np.float32), "lens": lens}

    def check(i, o):
        off = np.concatenate([[0], np.cumsum(i["lens"])])
        for u in range(len(i["lens"])):
            ref = oracle.delta_features(i["x"][off[u]:off[u + 1]].astype(np.float64), W3)
            _bar(rel_err(o[0][off[u]:off[u + 1]], ref) < 1e-6)
    return make, lambda i: [_P().delta_features(i["x"], W3, lengths=i["lens"])], check


def _stats_inputs(form):
    def make(rng, big):
        B, T, D = (5, 60, 11) if big else (4, 40, 9)
        x = (rng.standard_normal((B, T, D)) * 3 + 10).astype(np.float32)
        lens = rng.integers(1, T + 1, B)
        if form == "a":
            return {"data": [x[b] for b in range(B)], "lens": lens, "x": x}
        return {"data": x if form == "b" else _cuda(x), "lens": lens, "x": x}
    return make


for _form in ("a", "b", "c"):
    def _stats_case(form=_form):
        from oracle import normalize as ON

        def call(i):
            P = _P()
            return (list(P.meanvar(i["data"], i["lens"])) + list(P.meanstd(i["data"], i["lens"]))
                    + list(P.minmax(i["data"], i["lens"])))

        def check(i, o):
            x = i["x"]
            refs = list(ON.meanvar(x, i["lens"])) + list(ON.meanstd(x, i["lens"])) + list(ON.minmax(x, i["lens"]))
            for got, ref in zip(o, refs):
                _bar(rel_err(_h(got), ref) < 1e-5)
        return _stats_inputs(form), call, check
    CATALOGUE.append(Case("meanvar_meanstd_minmax_form_" + _form,
                          [("preprocessing", "meanvar"), ("preprocessing", "meanstd"), ("preprocessing", "minmax")],
                          *_stats_case(), ws=True))


@case("scaling_family_cuda", [("preprocessing", n) for n in ("scale", "inv_scale", "minmax_scale", "inv_minmax_scale")])
def _c():
    from oracle import normalize as ON

    def make(rng, big):
        x = rng.standard_normal((60 if big else 37, 13)).astype(np.float32)
        mean, std = rng.standard_normal(13).astype(np.float32), (rng.random(13) + 0.5).astype(np.float32)
        std[3] = 0
        lo, hi = x.min(0), x.max(0)
        return {"x": _cuda(x), "mean": mean, "std": std, "lo": lo, "hi": hi}

    def call(i):
        P = _P()
        return [P.scale(i["x"], i["mean"], i["std"]), P.inv_scale(i["x"], i["mean"], i["std"]),
                P.minmax_scale(i["x"], i["lo"], i["hi"], feature_range=(0.01, 0.99)),
                P.inv_minmax_scale(i["x"], i["lo"], i["hi"], feature_range=(0.01, 0.99))]

    def check(i, o):
        x = _h(i["x"])
        refs = [ON.scale(x, i["mean"], i["std"]), ON.inv_scale(x, i["mean"], i["std"]),
                ON.minmax_scale(x, i["lo"], i["hi"], feature_range=(0.01, 0.99)),
                ON.inv_minmax_scale(x, i["lo"], i["hi"], feature_range=(0.01, 0.99))]
        for got, ref in zip(o, refs):
            _bar(np.array_equal(_h(got), ref))
    return make, call, check


@case("interp1d_padded_cuda", [("preprocessing", "interp1d")], ws=True)
def _c():
    from oracle import wave as OW

    def make(rng, big):
        B, T = (5, 90) if big else (3, 60)
        f0 = np.where(rng.random((B, T)) > 0.4, rng.random((B, T)) * 100 + 100, 0.0)
        lens = rng.integers(T // 2, T + 1, B)
        return {"f0": _cuda(f0), "lens": lens}

    def check(i, o):
        f0, y = _h(i["f0"]), _h(o[0])
        for b, n in enumerate(i["lens"]):
            _bar(np.allclose(y[b, :n], OW.interp1d(f0[b, :n].copy()), rtol=1e-12, atol=0))
            _bar(np.array_equal(y[b, n:], f0[b, n:]))
    return make, lambda i: [_P().interp1d(i["f0"], lengths=i["lens"])], check


@case("preemphasis_and_inverse_with_repair", [("preprocessing", "preemphasis"), ("preprocessing", "inv_preemphasis")],
      ws=True)
def _c():
    from oracle import wave as OW

    def make(rng, big):
        x = rng.standard_normal((3, 9000 if big else 6000)).astype(np.float32)
        return {"x": _cuda(x), "lens": np.array([x.shape[1], 4000, 1])}

    def call(i):
        from nnmnkwii_b200.preprocessing import waveform
        P = _P()
        out = [P.preemphasis(i["x"], 0.97, lengths=i["lens"]), P.inv_preemphasis(i["x"], 0.97, lengths=i["lens"]),
               P.inv_preemphasis(i["x"][0], 1.5)]
        assert waveform._repair_counters()[0] > 0  # |coef| > 1: the repair walk runs
        return out

    def check(i, o):
        x = _h(i["x"])
        for b, n in enumerate(i["lens"]):
            _bar(np.array_equal(_h(o[0])[b, :n], OW.preemphasis(x[b, :n], 0.97)))
            _bar(np.array_equal(_h(o[1])[b, :n], OW.inv_preemphasis(x[b, :n], 0.97)))
        ref = OW.inv_preemphasis(x[0], 1.5)
        got = _h(o[2])
        fin = np.isfinite(ref)
        _bar(np.array_equal(np.isfinite(got), fin) and np.array_equal(got[fin], ref[fin]))
    return make, call, check


@case("mulaw_family_cuda", [("preprocessing", n) for n in ("mulaw", "inv_mulaw", "mulaw_quantize", "inv_mulaw_quantize")])
def _c():
    from oracle import wave as OW

    def make(rng, big):
        return {"x": _cuda(rng.uniform(-1, 1, 5000 if big else 3000).astype(np.float32))}

    def call(i):
        P = _P()
        q = P.mulaw_quantize(i["x"], 256)
        return [P.mulaw(i["x"], 256), P.inv_mulaw(i["x"], 256), q, P.inv_mulaw_quantize(q, 256)]

    def check(i, o):
        x = _h(i["x"])
        _bar(np.allclose(_h(o[0]), OW.mulaw(x, 256), rtol=1e-6, atol=1e-7))
        _bar(np.allclose(_h(o[1]), OW.inv_mulaw(x, 256), rtol=1e-6, atol=1e-7))
        _bar(np.abs(_h(o[2]).astype(np.int64) - OW.mulaw_quantize(x, 256)).max() <= 1)
        _bar(np.allclose(_h(o[3]), OW.inv_mulaw_quantize(_h(o[2]), 256), rtol=1e-6, atol=1e-7))
    return make, call, check


def _modspec_case(dt, n):
    K, tol = n // 2 + 1, 1e-4 if dt == np.float32 else 1e-10

    def make(rng, big):
        T, D = (min(n, 300), 6) if big else (240, 5)
        lens = np.array([T, 1, 0, T // 2 + 1])
        ph = np.exp(1j * rng.uniform(-np.pi, np.pi, (len(lens), K, D)))
        return {"x": _cuda(_nan_padded(rng, lens, T, D, dt)), "lens": lens,
                "ms": _cuda((rng.random((len(lens), K, D)) ** 2).astype(dt)),
                "ph": _cuda(ph.astype(np.complex64 if dt == np.float32 else np.complex128))}

    def call(i):
        P = _P()
        x, lens = i["x"], i["lens"]
        ms, ph = P.modspec(x, n=n, return_phase=True, lengths=lens)
        return [ms, ph, P.modphase(x, n=n, norm="ortho", lengths=lens),
                P.inv_modspec(i["ms"], i["ph"], lengths=lens), P.inv_modspec(i["ms"], i["ph"]),
                P.modspec_smoothing(x, 200, n=n, cutoff=40, lengths=lens),
                P.modspec_smoothing(x, 200, n=n, cutoff=40, log_domain=False, lengths=lens)]

    def check(i, o):
        x, o = _h(i["x"]).astype(np.float64), [_h(t) for t in o]
        Y = np.sqrt(_h(i["ms"]).astype(np.float64)) * _h(i["ph"])
        cut = np.arange(K)[:, None] >= int(n * 40 / 200) + 1
        for b, L in enumerate(i["lens"]):
            X = np.fft.rfft(x[b, :L], n, axis=0)
            pw = X.real ** 2 + X.imag ** 2
            _bar(rel_err(o[0][b], pw) <= tol)
            for ph in (o[1], o[2]):  # the phase is judged where it matters, weighted by the amplitude
                _bar(_crel(np.sqrt(pw) * ph[b], X) <= tol)
            _bar(rel_err(o[4][b], np.fft.irfft(Y[b], n, axis=0)) <= tol)
            refs = (np.fft.irfft(Y[b], n, axis=0), np.fft.irfft(np.where(cut, np.exp(1j * np.angle(X)), X), n, axis=0),
                    np.fft.irfft(np.where(cut, 0, X), n, axis=0))
            for got, ref in zip((o[3], o[5], o[6]), refs):  # inv_modspec with lengths, smoothing log / linear
                _bar(not got[b, L:].any() and (L == 0 or rel_err(got[b, :L], ref[:L]) <= tol))
    return make, call, check


for _dt, _n in ((np.float32, 512), (np.float64, 256)):
    CATALOGUE.append(Case("modspec_family_padded_%s_n%d" % (np.dtype(_dt).name, _n),
                          [("preprocessing", f) for f in ("modspec", "modphase", "inv_modspec", "modspec_smoothing")],
                          *_modspec_case(_dt, _n)))


def _dtw_case(radius):
    def make(rng, big):
        N, Tx, Ty, D = (3, 60, 70, 5) if big else (2, 40, 48, 5)
        X = np.zeros((N, Ty, D), np.float32)
        Y = (np.cumsum(rng.standard_normal((N, Ty, D)), 1) * 0.3).astype(np.float32)
        lx = []
        for n in range(N):
            t = Tx - 3 * n
            X[n, :t] = (np.cumsum(rng.standard_normal((t, D)), 0) * 0.3).astype(np.float32)
            lx.append(t)
        return {"X": X, "Y": Y, "lx": lx}

    def call(i):
        from nnmnkwii_b200.metrics import melcd
        from nnmnkwii_b200.preprocessing.alignment import DTWAligner
        al = DTWAligner(dist=melcd, radius=radius) if radius is not None else DTWAligner(radius=None)
        return list(al.transform((i["X"], i["Y"])))

    def check(i, o):
        for n, t in enumerate(i["lx"]):
            kind = "melcd" if radius is not None else "euclid"
            _, pi, pj, _ = oracle.fastdtw(i["X"][n, :t], i["Y"][n], -1 if radius is None else radius, kind)
            _bar(np.array_equal(o[0][n, :len(pi)], i["X"][n][pi]) and np.array_equal(o[1][n, :len(pj)], i["Y"][n][pj]))
            _bar(not o[0][n, len(pi):].any())
    return make, call, check


CATALOGUE.append(Case("DTWAligner_fastdtw_melcd", [("preprocessing.alignment", "DTWAligner")], *_dtw_case(1), ws=True))
CATALOGUE.append(Case("DTWAligner_exact", [("preprocessing.alignment", "DTWAligner")], *_dtw_case(None), ws=True))


# ---- postfilters ----
PF = dict(alpha=0.41, minimum_phase_order=127, fftlen=256)


@case("merlin_post_filter_cuda", [("postfilters", "merlin_post_filter")])
def _c():
    from oracle import sptk_postfilter as OP

    def make(rng, big):
        mgc = rng.standard_normal((33 if big else 21, 25)) * 0.2
        mgc[4] = 0.0  # an all-zero frame comes out exactly zero
        return {"mgc": _cuda(mgc)}

    def check(i, o):
        mgc, out = _h(i["mgc"]), _h(o[0])
        ref = OP.merlin_post_filter(mgc, PF["alpha"], PF["minimum_phase_order"], PF["fftlen"])
        _bar(np.all(np.abs(out - ref) <= 1e-6 * np.maximum(1.0, np.abs(ref))))
        _bar(not out[4].any())
    return make, lambda i: [__import__("nnmnkwii_b200.postfilters", fromlist=["x"]).merlin_post_filter(i["mgc"], **PF)], check


@case("modspec_statistics_and_post_filter_f64", [("postfilters", "modspec_statistics"),
                                                 ("postfilters", "modspec_post_filter")])
def _c():
    import oracle.ms_postfilter as OM

    def make(rng, big):
        T, D = (260, 5) if big else (200, 4)
        glens, lens = np.array([T, T // 2, 1, 37]), np.array([T, 1, 0, T // 4 + 1])
        return {"gen": _cuda(_nan_padded(rng, glens, T, D, np.float64)), "glens": glens,
                "nat": _cuda(rng.standard_normal((5, T, D))), "x": _cuda(_nan_padded(rng, lens, T, D, np.float64)),
                "lens": lens}

    def call(i):
        from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
        G = modspec_statistics(i["gen"], n=MS_N, lengths=i["glens"])
        N = modspec_statistics(i["nat"], n=MS_N)
        return list(G) + list(N) + [modspec_post_filter(i["x"], N, G, k=0.8, n=MS_N, lengths=i["lens"])]

    def check(i, o):
        gen, x, o = _h(i["gen"]), _h(i["x"]), [_h(t) for t in o]
        want = (OM.statistics([gen[b, :L] for b, L in enumerate(i["glens"])], MS_N)
                + OM.statistics(list(_h(i["nat"])), MS_N))
        for got, w in zip(o[:4], want):
            _bar(rel_err(got, w) < 1e-10)
        for b, L in enumerate(i["lens"]):  # the filter against the restatement given the device's statistics
            y = o[4][b]
            _bar(not y[L:].any() and (L == 0 or rel_err(y[:L], OM.post_filter(x[b, :L], o[2:4], o[0:2], 0.8, MS_N))
                                      < 1e-10))
    return make, call, check


def _ms_segment_case(dt):
    n, L, tol = 64, 50, 1e-4 if dt == np.float32 else 1e-10

    def make(rng, big):
        T, D = (1000, 10) if big else (900, 9)
        lens = np.array([1000, 30, 0, 600, 5] if big else [900, 17, 0, 512])
        w = rng.standard_normal((3, 401, D))
        return {"x": _cuda(_nan_padded(rng, lens, T, D, dt)), "lens": lens,
                "nat": _cuda((13.0 * (w[:, 1:] + 0.2 * w[:, :-1])).astype(dt))}

    def call(i):
        from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
        G = modspec_statistics(i["x"], n=n, lengths=i["lens"], segment=L)
        N = modspec_statistics(i["nat"], n=n, segment=L)
        return list(G) + list(N) + [modspec_post_filter(i["x"], N, G, k=0.8, n=n, lengths=i["lens"], segment=L)]

    def check(i, o):
        import oracle.ms_segment as OS
        from test_ms_segment_gpu import _check_stats
        x = _h(i["x"])
        for got, utts in ((o[0:2], [x[b, :Lb] for b, Lb in enumerate(i["lens"]) if Lb]), (o[2:4], list(_h(i["nat"])))):
            _check_stats(got, OS.statistics(utts, n, L), dt, utts, n, L)
        G, N = [_h(t).astype(np.float64) for t in o[0:2]], [_h(t).astype(np.float64) for t in o[2:4]]
        for b, Lb in enumerate(i["lens"]):  # the filter against the restatement given the device's statistics
            y = _h(o[4])[b]
            _bar(not y[Lb:].any() and (Lb == 0 or rel_err(y[:Lb], OS.post_filter(x[b, :Lb], N, G, 0.8, n, L)) <= tol))
    return make, call, check


for _dt in (np.float32, np.float64):
    CATALOGUE.append(Case("modspec_statistics_and_post_filter_segment_%s" % np.dtype(_dt).name,
                          [("postfilters", "modspec_statistics"), ("postfilters", "modspec_post_filter")],
                          *_ms_segment_case(_dt)))


# ---- baseline.gmm ----
def _joint_gmm(rng, Mx, dim):
    import types
    A = rng.standard_normal((Mx, 2 * dim, 2 * dim)) / np.sqrt(2 * dim)
    cov = A @ A.transpose(0, 2, 1) + 0.5 * np.eye(2 * dim)
    w = rng.random(Mx) + 0.1
    return types.SimpleNamespace(means_=rng.standard_normal((Mx, 2 * dim)), covariances_=cov, weights_=w / w.sum(),
                                 covariance_type="full")


@case("gmm_MLPG_transform_and_posterior_mean", [("baseline.gmm", "MLPG"), ("baseline.gmm", "MLPGBase")], ws=True)
def _c():
    def make(rng, big):
        return {"gmm": _joint_gmm(np.random.default_rng(3), 4, 8), "src": rng.standard_normal((50 if big else 30, 8))}

    def call(i):
        from nnmnkwii_b200.baseline.gmm import MLPG, MLPGBase
        return [MLPG(i["gmm"], windows=W2).transform(i["src"]), MLPGBase(i["gmm"]).transform(i["src"])]

    def check(i, o):
        from nnmnkwii_b200.baseline.gmm import MLPGBase
        from test_kernel_variants_gmm_gpu import gmm_map_reference
        lp, Em, post, Dm = gmm_map_reference(MLPGBase(i["gmm"]), i["src"])
        mix = lp.argmax(1)
        _bar(rel_err(o[0], oracle.mlpg(Em[np.arange(len(mix)), mix], Dm[mix], W2)) < 1e-9)
        _bar(rel_err(o[1], post) < 1e-9)
    return make, call, check


@case("gmm_MLPG_transform_em", [("baseline.gmm", "MLPG")], ws=True)
def _c():
    import oracle.gmm_traj_em as OT

    # one workspace request per MLPG solve: ``big`` keeps n_iter and the number of utterances, only the lengths grow
    def make(rng, big):
        return {"gmm": _joint_gmm(np.random.default_rng(11), 6, 24),
                "srcs": [rng.standard_normal((T, 24)) for T in ((150, 20, 90) if big else (120, 7, 65))]}

    def call(i):
        from nnmnkwii_b200.baseline.gmm import MLPG
        m = MLPG(i["gmm"], windows=W3, diff=True)
        ys, L = m.transform_em_batch(i["srcs"], n_iter=3, return_log_likelihood=True)
        return [np.concatenate(ys), L, m.transform_em(i["srcs"][0], n_iter=2)]

    def check(i, o):
        off = np.concatenate([[0], np.cumsum([len(s) for s in i["srcs"]])])
        for u, src in enumerate(i["srcs"]):
            want, Lw = OT.transform_em(i["gmm"], W3, src, 3, diff=True)
            _bar(rel_err(o[0][off[u]:off[u + 1]], want) <= 1e-9 and np.all(np.abs(o[1][u] - Lw) <= 1e-10 * np.abs(Lw)))
        _bar(rel_err(o[2], OT.transform_em(i["gmm"], W3, i["srcs"][0], 2, diff=True)[0]) <= 1e-9)
    return make, call, check


REG = 1e-6


def _em_prepare(i):
    from nnmnkwii_b200.baseline.gmm import _EmState
    i = dict(i)
    i["st"] = _EmState(i["X"], i["K"], REG)
    return i


@case("gmm_EmState_one_step", [("baseline.gmm", "GaussianMixture")], ws=True, prepare=_em_prepare)
def _c():
    def make(rng, big):
        N, D, K = (900, 7, 5) if big else (600, 6, 4)
        X = rng.standard_normal((N, D)) * rng.uniform(0.5, 2.0, D) + rng.standard_normal(D)
        return {"X": _cuda(X), "K": K, "resp": rng.dirichlet(np.ones(K), size=N)}

    def call(i):
        st = i["st"]
        st.put("resp", i["resp"])
        st.mstep(1)
        st.factor(True)
        st.check_status()
        st.estep()
        return [st.weights.clone(), st.means.clone(), st.covariances.clone(), st.prec_chol.clone(), st.resp.clone(),
                st.lower_bound.clone()]

    def check(i, o):
        from test_kernel_variants_gmm_gpu import em_estep_reference, em_mstep_reference
        X = _h(i["X"])
        _, _, w1, means, cov, pc = em_mstep_reference(X, i["resp"], REG)
        for got, want in zip(o[:4], (w1, means, cov, pc)):
            _bar(rel_err(_h(got), want) < 1e-10)
        resp, lb = em_estep_reference(X, w1, means, pc)
        _bar(np.abs(_h(o[4]) - resp).max() < 1e-10 and abs(float(_h(o[5])[0]) - lb) <= 1e-12 * abs(lb))
    return make, call, check


@case("gmm_GaussianMixture_init_device_kmeans", [("baseline.gmm", "GaussianMixture")], ws=True)
def _c():
    def make(rng, big):
        K, D = 4, 5
        centres = rng.standard_normal((K, D)) * 4
        X = centres[rng.integers(0, K, 1200 if big else 800)] + rng.standard_normal((1200 if big else 800, D))
        return {"X": X, "K": K}

    def call(i):
        import warnings

        from nnmnkwii_b200.baseline.gmm import GaussianMixture
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            g = GaussianMixture(n_components=i["K"], init_params="kmeans", init_device=True, random_state=0, max_iter=5)
            labels = g.fit_predict(i["X"])
        return [labels, g.weights_, g.means_, g.covariances_]

    def check(i, o):
        import warnings

        from sklearn.mixture import GaussianMixture as Sk
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            s = Sk(n_components=i["K"], init_params="kmeans", random_state=0, max_iter=5).fit(i["X"])
        _bar(np.array_equal(o[0], s.predict(i["X"])))
        for got, want in zip(o[1:], (s.weights_, s.means_, s.covariances_)):
            _bar(rel_err(got, want) < 1e-8)
    return make, call, check


@case("gmm_kmeans_with_empty_clusters_and_plusplus", [("baseline.gmm", "GaussianMixture")], ws=True)
def _c():
    def make(rng, big):
        N, D = (1500, 5) if big else (1000, 4)
        X = rng.standard_normal((6, D))[rng.integers(0, 6, N)] * 3 + rng.standard_normal((N, D))
        init = X[np.random.default_rng(1).choice(N, 8, replace=False)].copy()
        init[:2] = 1e4 + np.arange(2)[:, None]  # far from every frame: empty after the first assignment
        return {"X": _cuda(X), "init": init}

    def call(i):
        import warnings

        from nnmnkwii_b200.baseline.gmm import _device_kmeans, _device_kmeans_plusplus
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            labels, centres, inertia, n_iter = _device_kmeans(i["X"], 8, init=i["init"], max_iter=20)
        seeds, idx = _device_kmeans_plusplus(i["X"], 5, 0)
        return [labels, centres, inertia, n_iter, seeds, idx]

    def check(i, o):
        import warnings

        from sklearn.cluster import KMeans, kmeans_plusplus
        X = _h(i["X"])
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = KMeans(n_clusters=8, n_init=1, init=i["init"], max_iter=20).fit(X)
        _bar(np.array_equal(_h(o[0]), ref.labels_) and o[3] == ref.n_iter_)
        _bar(rel_err(_h(o[1]), ref.cluster_centers_) < 1e-10 and abs(o[2] - ref.inertia_) <= 1e-10 * ref.inertia_)
        c, idx = kmeans_plusplus(X, 5, random_state=0)
        _bar(np.array_equal(_h(o[5]), idx) and rel_err(_h(o[4]), c) < 1e-12)
    return make, call, check


# ---- util ----
@case("util_cholesky_inv_dense_and_banded", [("util.linalg", "cholesky_inv"), ("util.linalg", "cholesky_inv_banded")])
def _c():
    def make(rng, big):
        B, N = (3, 40) if big else (2, 24)
        A = rng.standard_normal((B, N, N))
        L = np.linalg.cholesky(A @ A.transpose(0, 2, 1) + N * np.eye(N))
        Lb = np.tril(L) * (np.subtract.outer(np.arange(N), np.arange(N)) < 3)
        Lb[:, np.arange(N), np.arange(N)] = np.abs(Lb[:, np.arange(N), np.arange(N)]) + 1
        return {"L": _cuda(L), "Lb": _cuda(Lb)}

    def call(i):
        from nnmnkwii_b200.util import linalg
        return [linalg.cholesky_inv(i["L"], lower=True), linalg.cholesky_inv_banded(i["Lb"], width=3)]

    def check(i, o):
        L, Lb = _h(i["L"]), _h(i["Lb"])
        for b in range(L.shape[0]):
            _bar(rel_err(_h(o[0])[b], np.linalg.inv(L[b] @ L[b].T)) < 1e-10)
            _bar(rel_err(_h(o[1])[b], np.linalg.inv(Lb[b] @ Lb[b].T)) < 1e-10)
    return make, call, check


@case("util_apply_each2d_trim_and_padded", [("util", "apply_each2d_trim"), ("util", "apply_each2d_padded")])
def _c():
    def make(rng, big):
        N, T, D = (4, 50, 6) if big else (3, 30, 5)
        X = np.zeros((N, T, D), np.float32)
        lens = rng.integers(2, T, N)
        for n in range(N):
            X[n, :lens[n]] = rng.standard_normal((lens[n], D)) + 2
        return {"X": _cuda(X), "lens": lens}

    def call(i):
        from nnmnkwii_b200 import util
        P = _P()
        return [util.apply_each2d_trim(P.delta_features, i["X"], W2),
                util.apply_each2d_padded(P.delta_features, i["X"], i["lens"], W2)]

    def check(i, o):
        X = _h(i["X"])
        for got in o:
            g = _h(got)
            for n, t in enumerate(i["lens"]):
                _bar(rel_err(g[n, :t], oracle.delta_features(X[n, :t].astype(np.float64), W2)) < 1e-6)
                _bar(not g[n, t:].any())
    return make, call, check


def _bar(ok):
    assert ok


# ---- the four ways ----------------------------------------------------------------------------------------------------
def _inputs(c, seed, big=False):
    return c.make(np.random.default_rng(seed), big)


def _cold_caches():
    """Drop the cached device tables (chain tables and weights, UV bands, post-filter bases), so that the next
    call builds them under the allocation poison of its run.  Every run ends synchronised, so nothing reads
    them any more."""
    from nnmnkwii_b200 import _device as dev
    from nnmnkwii_b200 import _uvmlpg, postfilters
    dev._const_cache.clear()
    _uvmlpg._band_cache.clear()
    postfilters._basis_cache.clear()


def _plain(c, inp, fill=None):
    import torch
    _cold_caches()
    with allocations(fill=fill):
        out = c.call(c.prepare(inp))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("c", CATALOGUE, ids=lambda c: c.name)
def test_case_four_ways(c):
    import torch
    RUN_CASES.add(c.name)
    seed = sum(map(ord, c.name))
    inp = _inputs(c, seed)

    # 1. plain, against the reference
    plain = _plain(c, inp)
    c.check(inp, plain)

    # 3. (first, so that no poison from 2. is left in the pool) recycled scratch: the case's workspace
    # requests get the blocks a larger valid call just used, as that call left them; compared with the case
    # run straight after torch.cuda.empty_cache()
    torch.cuda.empty_cache()
    fresh = _plain(c, inp)
    same(fresh, plain)
    kept, served = [], []
    _cold_caches()
    with recycled_workspace(kept, None):
        c.call(c.prepare(_inputs(c, seed + 1, big=True)))
    torch.cuda.synchronize()
    with recycled_workspace(kept, served):
        recycled = c.call(c.prepare(inp))
    torch.cuda.synchronize()
    assert bool(served) == c.ws, ("workspace requests", len(served), "case marked ws", c.ws)
    assert all(served), "a workspace request of the case was larger than the larger call's: %s" % served
    same(recycled, fresh)
    del kept

    # 2. poisoned floating-point allocations
    for fill in (0xFF, 0x7F):
        same(_plain(c, inp, fill), plain)

    # 4. a delayed side stream, the legacy default stream held back, every launch checked for its stream
    same(_side_stream(c, inp), plain)


def _map_tensors(inp, fn):
    import torch
    out = {}
    for k, v in inp.items():
        if isinstance(v, torch.Tensor) and v.is_cuda:
            out[k] = fn(v)
        elif isinstance(v, list) and v and all(isinstance(t, torch.Tensor) and t.is_cuda for t in v):
            out[k] = [fn(t) for t in v]
        else:
            out[k] = v
    return out


def _side_stream(c, inp):
    """The case on a fresh stream S behind a sleep; inputs NaN (complex: NaN in both parts; integers 0) until S
    copies them in.

    Most calls synchronise S on a host-to-device upload before their launch, so by then S's sleep is over.
    Two things make the arm independent of that timing.  Every launching C call must pass S as its stream
    (the recording proxy checks the argument).  And the legacy default stream, which a kernel or copy given
    stream 0 inside the library would use, is held by a longer sleep for the whole call: such work could not
    finish before S copies the outputs (S does not wait for it), and the test asserts the hold outlasted
    the call."""
    import torch
    holders = _map_tensors(inp, lambda t: torch.full_like(t, float("nan")) if t.is_floating_point()
                           else torch.full_like(t, complex(math.nan, math.nan)) if t.is_complex()
                           else torch.zeros_like(t))
    _cold_caches()
    with allocations(fill=0xFF):
        prepared = c.prepare(holders)  # constructed on the default stream
    torch.cuda.synchronize()
    S = torch.cuda.Stream()
    legacy = torch.cuda.default_stream()
    torch.cuda._sleep(LEGACY_HOLD_CYCLES)  # on the default stream, the current one here
    held = torch.cuda.Event()
    held.record(legacy)
    STREAM_CHECK["on"], STREAM_CHECK["bad"] = True, []
    try:
        with torch.cuda.stream(S):
            torch.cuda._sleep(SLEEP_CYCLES)
            for k, v in inp.items():
                if isinstance(holders[k], torch.Tensor) and holders[k] is not v:
                    holders[k].copy_(v)
                elif isinstance(v, list) and holders[k] is not v:
                    for h, t in zip(holders[k], v):
                        h.copy_(t)
            with allocations(fill=0xFF):
                out = c.call(prepared)
            copies = [torch.full_like(o, float("nan")).copy_(o) if isinstance(o, torch.Tensor) and o.is_cuda
                      and o.is_floating_point() else o.clone() if isinstance(o, torch.Tensor) and o.is_cuda else o
                      for o in out]
        S.synchronize()
        still_held = not held.query()
    finally:
        STREAM_CHECK["on"] = False
    assert not STREAM_CHECK["bad"], "launches not on the caller's stream (name, got, want): %s" % STREAM_CHECK["bad"]
    assert still_held, "the legacy default stream's hold ended during the call: the arm proved nothing"
    torch.cuda.synchronize()
    return copies


def test_every_catalogue_entry_point_and_launching_export_is_reached():
    """Run last: each public entry point named by the catalogue has a case, and every launching C symbol
    was reached by some case of this module."""
    from nnmnkwii_b200 import _lib
    covered = set()
    for c in CATALOGUE:
        covered |= set(c.covers)
    assert covered == SC.COVERED, (sorted(SC.COVERED - covered), sorted(covered - SC.COVERED))
    if RUN_CASES != {c.name for c in CATALOGUE}:
        pytest.skip("needs every case of the catalogue in the same run")
    missing = sorted(set(SC.launching_exports(_lib.EXPORTS)) - REACHED)
    assert not missing, "launching C symbols no case reached: %s" % missing


# ---- cache eviction while a kernel is pending on another stream --------------------------------------------------------
def _refill(ptr, nbytes, content, limit):
    """Allocate blocks on the current stream (at most ``limit``) until they cover the byte range
    [ptr, ptr + nbytes) of a freed block, and copy ``content`` (a CUDA tensor of nbytes bytes) into that range.
    The freed block may have merged with free neighbours, so several allocations may share the range; once
    part of it is covered, each request asks for the shortest uncovered piece.  Returns the allocations (to
    keep them alive) if the range was covered, else None."""
    import torch
    src = content.reshape(-1).view(torch.uint8)
    held, gaps = [], [(ptr, ptr + nbytes)]
    size = nbytes
    for _ in range(limit):
        t = torch.empty(size, dtype=torch.uint8, device="cuda")
        held.append(t)
        a, e = t.data_ptr(), t.data_ptr() + size
        left = []
        for lo, hi in gaps:
            clo, chi = max(lo, a), min(hi, e)
            if clo < chi:
                t[clo - a:chi - a].copy_(src[clo - ptr:chi - ptr])
                left += [g for g in ((lo, clo), (chi, hi)) if g[0] < g[1]]
            else:
                left.append((lo, hi))
        gaps = left
        if not gaps:
            return held
        size = -(-min(hi - lo for lo, hi in gaps) // 512) * 512
    return None


def _block(t):
    return t.data_ptr(), t.numel() * t.element_size()


def _refill_bound(nbytes):
    """Allocations of at least 512 bytes that reach every free block of the pool the evicted block of
    ``nbytes`` belongs to: each one takes at least 512 of the pool's free bytes."""
    import torch
    torch.empty(1, device="cuda")  # an allocation makes the allocator release blocks whose streams finished
    pool = "small" if nbytes <= 1 << 20 else "large"
    st = torch.cuda.memory_stats()
    return int(st["inactive_split_bytes.%s_pool.current" % pool]) // 512 + int(st["inactive_split.%s_pool.current" % pool]) + 16


def _evict_and_refill(S, block, alt, evict):
    """``block``: (data_ptr, nbytes) of the cached tensor a kernel pending on S reads, no longer referenced
    outside the cache; ``alt``: valid other content of its shape.  Evicts from the default stream while S is
    still busy, then refills the block with ``alt`` as soon as the allocator hands it out.  Returns whether
    that happened while S was still busy.  Once S has finished the block must come back."""
    import torch
    ptr, nbytes = block
    evict()
    assert not S.query(), "S finished before the eviction: the test proves nothing"
    kept = _refill(ptr, nbytes, alt, 512)
    early = kept is not None and not S.query()
    S.synchronize()
    if kept is None:
        kept = _refill(ptr, nbytes, alt, _refill_bound(nbytes))
    assert kept is not None, "the evicted block never came back: %s" % (_block_state(ptr),)
    torch.cuda.synchronize()
    return early


def _block_state(ptr):
    """(segment stream, block state, block size) of the allocator block holding ``ptr``."""
    import torch
    for seg in torch.cuda.memory_snapshot():
        addr = seg["address"]
        for blk in seg["blocks"]:
            if addr <= ptr < addr + blk["size"]:
                return seg.get("stream"), blk["state"], blk["size"], seg["segment_type"]
            addr += blk["size"]
    return None


def _until_cleared(cache, add):
    """Call ``add(k)`` for k = 0, 1, ... until the bounded ``cache`` has just been cleared (it then holds only
    the entry of the last call, made before the clear), so nothing is allocated after the eviction."""
    for k in range(1000):
        add(k)
        if len(cache) == 1:
            return
    raise AssertionError("the cache was never cleared")


def _sleeping_stream():
    import torch
    torch.cuda.synchronize()
    S = torch.cuda.Stream()
    with torch.cuda.stream(S):
        torch.cuda._sleep(EVICT_SLEEP_CYCLES)
    return S


def test_const_cache_eviction_behind_a_pending_postfilter():
    """_device._const_cache (the post-filter weights) evicted and refilled with other weights while the
    filter is still queued on S."""
    import torch

    from nnmnkwii_b200 import _device as dev
    from nnmnkwii_b200 import postfilters
    _cold_caches()  # the entry is built below, on the default stream
    rng = np.random.default_rng(1)
    mgc = _cuda(rng.standard_normal((40, 25)) * 0.2)
    weight = np.linspace(0.5, 1.5, 25)
    plain = postfilters.merlin_post_filter(mgc, weight=weight, **PF).clone()
    S = _sleeping_stream()
    with torch.cuda.stream(S):
        out = postfilters.merlin_post_filter(mgc, weight=weight, **PF)
    block = _block(dev.constant_on_device(weight, mgc.device))
    alt = _cuda(weight[::-1].copy())
    early = _evict_and_refill(S, block, alt, lambda: _until_cleared(
        dev._const_cache, lambda k: dev.constant_on_device(np.array([k], np.float64), mgc.device)))
    assert not early, "the weights' block was handed out while the filter on S had yet to read it"
    same([out], [plain])


def test_const_cache_eviction_behind_a_pending_mlpg_chain_table():
    """_device._const_cache (an MLPG chain table) evicted and refilled with the same table, out_col permuted,
    while the solve is still queued on S.  mlpg_batch synchronises S on its host-to-device copies, so the
    sleep is enqueued from the workspace request, right before the launch."""
    import torch

    from nnmnkwii_b200 import _device as dev
    G = _G()
    _cold_caches()  # the entry is built below, on the default stream
    rng = np.random.default_rng(2)
    lens = np.array([40, 17, 64])
    m, v = _mv(rng, int(lens.sum()), 187, np.float32)
    m, v = _cuda(m), _cuda(v)
    layout = G.merlin_layout()
    plain = G.mlpg_batch(m, v, W3, lengths=lens, layout=layout).clone()
    torch.cuda.synchronize()
    S = torch.cuda.Stream()
    orig = dev.workspace

    def sleepy_workspace(device, nbytes):
        torch.cuda._sleep(EVICT_SLEEP_CYCLES)
        return orig(device, nbytes)
    dev.workspace = sleepy_workspace
    try:
        with torch.cuda.stream(S):
            out = G.mlpg_batch(m, v, W3, lengths=lens, layout=layout, check=False)
    finally:
        dev.workspace = orig
    block = _block(dev.chains_on_device(layout.chains, m.device))
    perm = layout.chains.copy()
    perm["out_col"] = np.roll(perm["out_col"], 1)
    alt = _cuda(perm.view(np.int32).reshape(-1, 4))
    early = _evict_and_refill(S, block, alt, lambda: _until_cleared(
        dev._const_cache, lambda k: dev.constant_on_device(np.array([k], np.int32), m.device)))
    assert not early, "the chain table's block was handed out while the solve on S had yet to read it"
    same([out], [plain])


def test_band_cache_eviction_behind_a_pending_unit_variance_mlpg():
    """_uvmlpg._band_cache evicted and the band table's block refilled with the transposed table while the
    stencil is still queued on S."""
    import torch

    from nnmnkwii_b200 import _uvmlpg as uv
    AF = _AF()
    _cold_caches()  # the entry is built below, on the default stream
    rng = np.random.default_rng(3)
    R = _cuda(oracle.unit_variance_mlpg_matrix(W3, 32).astype(np.float64))
    x = _cuda(rng.standard_normal((2, 32, 12)))
    plain = AF.UnitVarianceMLPG.apply(x, R).clone()
    band = uv.band_of(R, R.device)
    assert band.toep is None  # the per-row table path reads Rb for every row
    alt = band.RbT.clone()
    Rs = [_cuda(oracle.unit_variance_mlpg_matrix(W3, 8 + k).astype(np.float64)) for k in range(17)]
    S = _sleeping_stream()
    with torch.cuda.stream(S):
        out = AF.UnitVarianceMLPG.apply(x, R)
    block = _block(band.Rb)
    del band
    early = _evict_and_refill(S, block, alt, lambda: _until_cleared(
        uv._band_cache, lambda k: uv.band_of(Rs[k], R.device)))
    assert not early, "the band table's block was handed out while the stencil on S had yet to read it"
    same([out], [plain])


def test_basis_cache_eviction_behind_a_pending_postfilter():
    """postfilters._basis_cache evicted and the basis block refilled with another alpha's basis while the
    filter is still queued on S.  Each basis build synchronises only the default stream, not S."""
    import torch

    from nnmnkwii_b200 import postfilters
    _cold_caches()  # the entry is built below, on the default stream
    rng = np.random.default_rng(4)
    mgc = _cuda(rng.standard_normal((40, 25)) * 0.2)
    plain = postfilters.merlin_post_filter(mgc, **PF).clone()
    args = (mgc.device, PF["alpha"], 25, PF["minimum_phase_order"], PF["fftlen"])
    alt = postfilters._basis(mgc.device, 0.55, *args[2:]).clone()
    S = _sleeping_stream()
    with torch.cuda.stream(S):
        out = postfilters.merlin_post_filter(mgc, **PF)
    block = _block(postfilters._basis(*args))
    early = _evict_and_refill(S, block, alt, lambda: _until_cleared(
        postfilters._basis_cache, lambda k: postfilters._basis(mgc.device, 0.3 + 0.001 * k, *args[2:])))
    assert not early, "the basis block was handed out while the filter on S had yet to read it"
    same([out], [plain])


def test_metric_workspace_cache_is_per_stream():
    """metrics._ws_cache: each entry is allocated and used on one stream, and the reduction reads its result
    back before returning, so no kernel is pending when an entry is dropped.  An entry made on S and evicted
    from the default stream is never handed to an allocation on the default stream."""
    import torch

    from nnmnkwii_b200 import metrics
    rng = np.random.default_rng(5)
    X, Y = _cuda(rng.standard_normal((3, 50, 24))), _cuda(rng.standard_normal((3, 50, 24)))
    plain = metrics.melcd(X, Y, lengths=[50, 20, 7])
    S = torch.cuda.Stream()
    with torch.cuda.stream(S):
        on_s = metrics.melcd(X, Y, lengths=[50, 20, 7])
    key = (str(X.device), S.cuda_stream)
    target = metrics._ws_cache[key]
    ptr, nbytes = target.data_ptr(), target.numel()
    del target
    # 31 more pool streams of S's priority and 8 of high priority: 39 keys other than S's (the pool has 32
    # streams per priority, so a 32nd normal one would be S again)
    streams = [torch.cuda.Stream() for _ in range(31)] + [torch.cuda.Stream(priority=-1) for _ in range(8)]
    for st in streams:
        with torch.cuda.stream(st):
            metrics.melcd(X, Y, lengths=[50, 20, 7])
    assert key not in metrics._ws_cache
    assert _refill(ptr, nbytes, torch.zeros(nbytes, dtype=torch.uint8, device="cuda"), 256) is None
    with torch.cuda.stream(S):
        again = metrics.melcd(X, Y, lengths=[50, 20, 7])
    assert on_s == plain and again == plain
