"""Every kernel instance the metric launchers (csrc/nnk_metrics.cu) can select, against float64 references.

`dispatch_frame` runs `frame_metric_tile_kernel<T>` for contiguous frames narrower than 128 and
`frame_metric_kernel<T, G>`, G = min(32, pow2 >= D) lanes per frame, otherwise; `metrics.py` always passes
contiguous frames, so the G < 32 instances run only for strided frames (the mgc columns of a wider
acoustic row read in place).  These cases call the C ABI `nnk_frame_metric` / `nnk_f0_metric` on D
columns at an offset inside a wider (B, T, W) buffer, with lengths 0, 1, T, above T and negative, and
compare the returned sum and count with a reference that takes the difference (and, for the tile kernel,
the square) in the input dtype as the kernels do.  Integer-valued inputs make every sum of squares exact
in float64, so there the sum must match bit for bit.  The kernel names are checked against
`variant_mirror.metric_kernel_for` in a child process (`variant_mirror.profiled_in_child`).

The module is named to sort after every module that asserts kernel names from the pytest process: with these
cases run before them, torch.profiler came back empty for the UnitVarianceMLPG variant cases in a full GPU run on
an H100 (they pass alone and after these modules alone), so their names are collected in child processes and
their numbers come last."""
import ctypes

import numpy as np
import pytest

import oracle
import variant_mirror as M

pytestmark = pytest.mark.gpu

FRAME_D = [1, 2, 3, 4, 5, 8, 9, 16, 17, 33, 128, 129, 513]
TILE_D = [1, 3, 25, 60, 127]
COL0, PAD = 1, 3  # the metric columns start at column 1 of a D + 3 wide row



def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _code(dt):
    from nnmnkwii_b200 import _lib
    return _lib.NNK_F32 if np.dtype(dt) == np.float32 else _lib.NNK_F64


def _reduce(call, B, T):
    """(sum, count) of one C-ABI reduction into a fresh zeroed workspace."""
    import torch

    from nnmnkwii_b200 import _lib
    ws = torch.zeros(int(_lib.lib.nnk_metric_workspace_bytes(max(1, B), max(1, T))), dtype=torch.uint8, device="cuda")
    res = torch.full((2,), -1.0, dtype=torch.float64, device="cuda")
    _lib.check(call(ctypes.c_void_p(res.data_ptr()), ctypes.c_void_p(res.data_ptr() + 8), ctypes.c_void_p(ws.data_ptr()),
                    ctypes.c_int64(ws.numel()), _stream()), "nnk metric")
    return float(res[0].item()), int(res[1:2].view(torch.int64).item())


def _lengths(T, B, rng):
    fixed = [0, 1, T, T + 9, -4]
    return np.array(fixed + list(rng.integers(0, T + 1, B - len(fixed))), np.int32)[:B]


def _data(shape, dt, rng, integer):
    if integer:
        return rng.integers(-8, 9, shape).astype(dt)
    return (rng.standard_normal(shape) * 2).astype(dt)


def frame_reference(x, y, lens, kind, square_in_dtype):
    """(sum, count): per item the first clip(len, 0, T) frames; z = x - y in the input dtype, squared in the input
    dtype too when `square_in_dtype` (the tile kernel), summed per frame in float64; kind 0 adds the frames'
    square roots, kind 1 the sums themselves."""
    s, n = 0.0, 0
    for b in range(x.shape[0]):
        L = min(max(int(lens[b]), 0), x.shape[1])
        z = x[b, :L] - y[b, :L]
        per = (z * z).astype(np.float64).sum(-1) if square_in_dtype else np.square(z.astype(np.float64)).sum(-1)
        s += float((np.sqrt(per) if kind == 0 else per).sum())
        n += L
    return s, n


def _frame_case(D, dt, T, B, strided, integer, seed):
    rng = np.random.default_rng(seed)
    W = D + PAD if strided else D
    return _data((B, T, W), dt, rng, integer), _data((B, T, W), dt, rng, integer), _lengths(T, B, rng), W


def _frame_run(xb, yb, lens, D, kind, strided):
    import torch

    from nnmnkwii_b200 import _lib
    B, T, W = xb.shape
    x, y = torch.from_numpy(xb).cuda(), torch.from_numpy(yb).cuda()
    ln = torch.from_numpy(lens).cuda()
    off = (COL0 if strided else 0) * xb.itemsize

    def call(sp, cp, wp, wn, st):
        return _lib.lib.nnk_frame_metric(x.data_ptr() + off, y.data_ptr() + off, _code(xb.dtype), B, T, D, T * W, W,
                                         ln.data_ptr(), kind, sp, cp, wp, wn, st)
    return _reduce(call, B, T)


def _check_frames(D, dt, T, strided):
    for integer in (False, True):
        xb, yb, lens, W = _frame_case(D, dt, T, 8, strided, integer, seed=D + T + integer)
        cols = slice(COL0, COL0 + D) if strided else slice(0, D)
        tile = M.metric_kernel_for(D, W, dt)[0] == "tile"
        for kind in (0, 1):
            s, n = _frame_run(xb, yb, lens, D, kind, strided)
            rs, rn = frame_reference(xb[:, :, cols], yb[:, :, cols], lens, kind, square_in_dtype=tile)
            assert n == rn, (D, dt, kind, n, rn)
            assert abs(s - rs) <= 1e-12 * abs(rs), (D, dt, kind, integer, s, rs)
            if integer and kind == 1:
                assert s == rs, (D, dt, s, rs)  # every partial sum is an exact integer


@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("D", FRAME_D)
def test_frame_kernel_every_group_width(D, dt):
    assert M.metric_kernel_for(D, D + PAD, dt)[0] == "frame"
    _check_frames(D, dt, 37, strided=True)
    if D >= 128:  # contiguous wide frames run the same kernel
        _check_frames(D, dt, 37, strided=False)


@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("D", TILE_D)
def test_tile_kernel(D, dt):
    kind, F = M.metric_kernel_for(D, D, dt)
    assert kind == "tile"
    if dt == "float64" and D == 127:
        assert F == M.MT_MIN_TILE_FRAMES
    _check_frames(D, dt, 5 * F + 7, strided=False)  # partial last tile; T + 9 and F-multiples via the lengths


# ---- F0 metrics -----------------------------------------------------------------------------------------------------
F0_W, F0_COL, VUV_COL = 5, 1, 3  # lf0 and vuv columns of a 5-wide acoustic row


def _f0_case(dt, T, B, seed):
    rng = np.random.default_rng(seed)
    src = rng.uniform(4.0, 6.0, (B, T, F0_W)).astype(dt)
    tgt = rng.uniform(4.0, 6.0, (B, T, F0_W)).astype(dt)
    src[:, :, VUV_COL] = rng.integers(0, 2, (B, T))
    tgt[:, :, VUV_COL] = rng.integers(0, 2, (B, T))
    return src, tgt, _lengths(T, B, rng)


def f0_reference(src, tgt, lens, kind):
    """(sum, count) of lf0 MSE (kind 0), linear-domain MSE (1) or vuv error (2), masked like metrics/__init__.py."""
    s, n = 0.0, 0
    for b in range(src.shape[0]):
        L = min(max(int(lens[b]), 0), src.shape[1])
        xv, yv = src[b, :L, VUV_COL], tgt[b, :L, VUV_COL]
        if kind == 2:
            s += float((xv != yv).sum())
            n += L
            continue
        m = (xv + yv) >= 2
        a, c = src[b, :L, F0_COL][m], tgt[b, :L, F0_COL][m]
        if kind == 1:
            a, c = np.exp(a), np.exp(c)
        s += float(np.square((a - c).astype(np.float64)).sum())
        n += int(m.sum())
    return s, n


def _f0_run(src, tgt, lens, kind):
    import torch

    from nnmnkwii_b200 import _lib
    B, T, W = src.shape
    xs, ys = torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda()
    ln = torch.from_numpy(lens).cuda()
    es = src.itemsize

    def call(sp, cp, wp, wn, st):
        return _lib.lib.nnk_f0_metric(xs.data_ptr() + F0_COL * es, xs.data_ptr() + VUV_COL * es,
                                      ys.data_ptr() + F0_COL * es, ys.data_ptr() + VUV_COL * es, _code(src.dtype), B, T,
                                      T * W, W, ln.data_ptr(), kind, sp, cp, wp, wn, st)
    return _reduce(call, B, T)


@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_f0_kernel_strided_columns(kind, dt):
    for T in (1, 300, 2500):
        src, tgt, lens = _f0_case(dt, T, 9, seed=T + kind)
        s, n = _f0_run(src, tgt, lens, kind)
        rs, rn = f0_reference(src, tgt, lens, kind)
        assert n == rn, (kind, dt, T, n, rn)
        if kind == 2:
            assert s == rs, (dt, T, s, rs)
        else:  # float32 exp: CUDA's expf and NumPy's may differ by an ulp or two
            tol = 1e-5 if (kind == 1 and dt == "float32") else 1e-12
            assert abs(s - rs) <= tol * abs(rs), (kind, dt, T, s, rs)


def test_public_api_zips_short_lengths():
    """`lengths` with fewer entries than B: the reference's zip(X, Y, lengths) stops at the shorter one."""
    from nnmnkwii_b200 import metrics
    rng = np.random.default_rng(21)
    B, T, D = 6, 50, 9
    X, Y = rng.standard_normal((B, T, D)), rng.standard_normal((B, T, D))
    lens = [50, 3, 0, 41]
    assert abs(metrics.melcd(X, Y, lens) - oracle.melcd(X, Y, lens)) <= 1e-12 * oracle.melcd(X, Y, lens)
    mse = sum(float(np.square(X[b, :n] - Y[b, :n]).sum()) for b, n in enumerate(lens)) / (sum(lens) * D)
    assert abs(metrics.mean_squared_error(X, Y, lens) - mse ** 0.5) <= 1e-12 * mse ** 0.5
    va, vb = rng.integers(0, 2, (B, T)).astype(np.float64), rng.integers(0, 2, (B, T)).astype(np.float64)
    vuv = sum(float((va[b, :n] != vb[b, :n]).sum()) for b, n in enumerate(lens)) / sum(lens)
    assert metrics.vuv_error(va, vb, lens) == vuv


# ---- kernel names ---------------------------------------------------------------------------------------------------
def launch(kind, D, dt, strided):
    if kind == "f0":
        src, tgt, lens = _f0_case(dt, 300, 9, seed=1)
        _f0_run(src, tgt, lens, 0)
        return
    xb, yb, lens, _ = _frame_case(D, dt, 37 if strided else 300, 8, strided, False, seed=1)
    _frame_run(xb, yb, lens, D, 1, strided)


def test_kernel_names_follow_the_mirror():
    family = r"\b(frame_metric_\w*|f0_metric_)kernel<"
    cases, want = [], []
    for dt in ("float32", "float64"):
        T = "float" if dt == "float32" else "double"
        for D, strided in [(D, True) for D in FRAME_D] + [(D, False) for D in TILE_D + [128, 513]]:
            cases.append([["frame", D, dt, strided], family])
            kind, arg = M.metric_kernel_for(D, D + PAD if strided else D, dt)
            want.append("frame_metric_tile_kernel<%s>" % T if kind == "tile" else "frame_metric_kernel<%s, %d>" % (T, arg))
        cases.append([["f0", 1, dt, True], family])
        want.append("f0_metric_kernel<%s>" % T)
    got = M.profiled_in_child("test_variants_metrics_gpu", "launch", cases)
    for (case, _), w, (names, err) in zip(cases, want, got):
        assert err == "None", (case, err)
        assert names and all(w in n for n in names), (case, w, names)
    seen = {w for w in want}
    assert {"frame_metric_kernel<%s, %d>" % (T, G) for T in ("float", "double") for G in (1, 2, 4, 8, 16, 32)} <= seen
