"""Every instance of the data-movement launchers, through their C ABI, against exact NumPy references:
`delta_kernel<T>` (`nnk_delta_features`, csrc/nnk_delta.cu), `segment_copy_kernel<uint4 / uint32_t>`
(`nnk_segment_copy`, csrc/nnk_shard.cu), and `trim_len_kernel<T>` / `gather_rows_kernel<T>`
(`nnk_trim_lengths` / `nnk_gather_rows`, csrc/nnk_dtw.cu).

The Python wrappers send one shape of argument each (`x_ld = D`, no `utt_len`, zero padding only, a second
GPU for the segment copy), so these cases call the C ABI with strided rows, guard rows and columns, explicit
lengths and pointer offsets.  Every result is compared bit for bit: the delta reference adds the taps in
the kernel's order in float64 (`acc + c * x`, no FMA), the others move or count values.  The kernel names
are checked against `variant_mirror` in a child process (`variant_mirror.profiled_in_child`).

The module is named to sort after every module that asserts kernel names from the pytest process: with these
cases run before them, torch.profiler came back empty for the UnitVarianceMLPG variant cases in a full GPU run on
an H100 (they pass alone and after these modules alone), so their names are collected in child processes and
their numbers come last.  The `delta_features` CPU-tensor case is here for the same reason."""
import ctypes

import numpy as np
import pytest

import oracle
import variant_mirror as M
from conftest import rel_err

pytestmark = pytest.mark.gpu

SENTINEL = -7777.0



def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _tdt(name):
    import torch
    return getattr(torch, name)


def _code(name):
    from nnmnkwii_b200 import _lib
    return _lib.NNK_F32 if name == "float32" else _lib.NNK_F64


def _tname(name):
    return "float" if name == "float32" else "double"


# ---- delta_kernel --------------------------------------------------------------------------------------------------
def _delta_windows(taps, seed):
    """One window of M taps per entry: (l, u) = ((M - 1) // 2, M - 1 - l), random float64 coefficients."""
    rng = np.random.default_rng(seed)
    return [((m - 1) // 2, m - 1 - (m - 1) // 2, rng.standard_normal(m) / 3) for m in taps]


def _delta_case(taps, D, dt, seed, n_utt=37, max_T=45):
    """Host data of one call: utterances with lengths at every tap count, 1, 8, 16, 17 and max_T (% 8 != 0),
    `utt_len` up to 2 rows shorter than the offset gap, x_ld = D + 3 and out_ld = nw * D + 5."""
    rng = np.random.default_rng(seed)
    fixed = list(taps) + [max(taps), 1, 8, 16, 17, max_T]
    lens = np.array(fixed + list(rng.integers(1, max_T + 1, n_utt - len(fixed))), np.int64)[:n_utt]
    gaps = lens + rng.integers(0, 3, n_utt)
    off = np.concatenate([[0], np.cumsum(gaps)]).astype(np.int64)
    x_ld, out_ld = D + 3, len(taps) * D + 5
    x = (rng.standard_normal((int(off[-1]), x_ld)) * 4).astype(dt)
    return dict(taps=taps, D=D, dt=dt, lens=lens, off=off, x=x, x_ld=x_ld, out_ld=out_ld, max_T=int(lens.max()),
                windows=_delta_windows(taps, seed + 1))


def delta_reference(c):
    """The kernel's arithmetic in NumPy: per window, taps m = 0 .. M-1 centred at M // 2, `acc + coef * x` in
    float64 (two roundings per tap), frames outside [0, len) skipped, rounded to x's dtype; every other element
    of the output buffer keeps SENTINEL."""
    D, x, lens, off = c["D"], c["x"], c["lens"], c["off"]
    x64 = x[:, :D].astype(np.float64)
    out = np.full((x.shape[0], c["out_ld"]), SENTINEL, x.dtype)
    row = np.concatenate([off[u] + np.arange(n) for u, n in enumerate(lens)])
    t = np.concatenate([np.arange(n) for n in lens])
    tn = np.repeat(lens, lens)
    base = np.repeat(off[:-1], lens)
    for w, (l, u, coef) in enumerate(c["windows"]):
        taps = l + u + 1
        acc = np.zeros((len(row), D))
        for m in range(taps):
            s = t + m - taps // 2
            ok = (s >= 0) & (s < tn)
            val = x64[base + np.where(ok, s, 0)]
            acc = np.where(ok[:, None], acc + float(coef[m]) * val, acc)
        out[row, w * D:(w + 1) * D] = acc.astype(x.dtype)
    return out


def _delta_run(c):
    """Launch `nnk_delta_features` on case c; returns (return code, output buffer on the device)."""
    import torch

    from nnmnkwii_b200 import _lib
    dt = np.dtype(c["dt"]).name
    x = torch.from_numpy(c["x"]).cuda()
    out = torch.full((c["x"].shape[0], c["out_ld"]), SENTINEL, dtype=_tdt(dt), device="cuda")
    off = torch.from_numpy(c["off"]).cuda()
    lens = torch.from_numpy(c["lens"].astype(np.int32)).cuda()
    win = _lib.make_windows(c["windows"])
    rc = _lib.lib.nnk_delta_features(x.data_ptr(), _code(dt), c["D"], c["x_ld"], off.data_ptr(), lens.data_ptr(),
                                     len(c["lens"]), c["max_T"], ctypes.byref(win), out.data_ptr(), c["out_ld"],
                                     _stream())
    return rc, out


DELTA_TAPS = [(1,), (2,), (3,), (4,), (5,), (6,), (7,), (8,), (9,), (6, 1), (3, 4, 7), (9, 2, 5, 8)]
DELTA_D = [1, 31, 32, 33, 65, 200]


@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("taps", DELTA_TAPS, ids=lambda t: "taps" + "_".join(map(str, t)))
def test_delta_every_tap_count(taps, dt):
    from nnmnkwii_b200 import _lib
    for D in DELTA_D:
        c = _delta_case(taps, D, dt, seed=D + 10 * len(taps) + sum(taps))
        rc, out = _delta_run(c)
        _lib.check(rc, "nnk_delta_features")
        got = out.cpu().numpy()
        assert np.array_equal(got, delta_reference(c)), (taps, D, dt)
        # np.correlate(..., "same") of the reference, per utterance long enough for "same" to keep its length
        ws = [w[2] for w in c["windows"]]
        for u, n in enumerate(c["lens"]):
            if n < max(taps):
                continue
            a = int(c["off"][u])
            xs = c["x"][a:a + n, :D]
            ref = oracle.delta_features(xs if dt == "float64" else xs.astype(np.float64), ws)
            part = got[a:a + n, :len(taps) * D]
            assert rel_err(part, ref) <= (1e-15 if dt == "float64" else 2 ** -24), (taps, D, dt, u)


def test_delta_grid_limit_in_utterances():
    """65 535 utterances fill grid.z; 65 536 raise a clean error and launch nothing."""
    from nnmnkwii_b200 import _lib
    rng = np.random.default_rng(4)
    lens = (np.arange(65535) % 3 + 1).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    c = dict(taps=(3,), D=1, dt="float64", lens=lens, off=off, x=rng.standard_normal((int(off[-1]), 1)), x_ld=1,
             out_ld=1, max_T=3, windows=_delta_windows((3,), 5))
    rc, out = _delta_run(c)
    _lib.check(rc, "nnk_delta_features")
    assert np.array_equal(out.cpu().numpy(), delta_reference(c))
    lens2 = np.ones(65536, np.int64)
    c2 = dict(c, lens=lens2, off=np.arange(65537, dtype=np.int64), x=rng.standard_normal((65536, 1)))
    n0 = _lib.launch_count()
    rc, out = _delta_run(c2)
    assert rc == _lib.NNK_ERR_ARG and "too many utterances" in _lib.last_error()
    assert _lib.launch_count() == n0
    assert bool((out == SENTINEL).all())


# ---- segment_copy_kernel --------------------------------------------------------------------------------------------
SEG_LENS = [200, 0, 64, 65, 1, 129, 63, 128, 17]
# (name, element bytes, cols, src_ld, dst_ld, src byte offset, dst byte offset)
SEG_CASES = [("vector_f32", 4, 8, 12, 16, 0, 0), ("vector_f64", 8, 6, 10, 8, 0, 0), ("odd_cols", 4, 7, 8, 8, 0, 0),
             ("odd_pitch", 4, 8, 9, 12, 0, 0), ("src_offset_4_bytes", 4, 8, 12, 16, 4, 0),
             ("dst_offset_4_bytes", 8, 6, 10, 8, 0, 4)]


def _seg_case(es, cols, src_ld, dst_ld, src_off, dst_off, seed=0):
    """Segments placed in scrambled order, with gaps, in both matrices; buffers filled with random words."""
    rng = np.random.default_rng(seed)
    lens = np.array(SEG_LENS, np.int64)

    def place(order):
        rows = np.zeros(len(lens), np.int64)
        r = 0
        for s in order:
            r += int(rng.integers(0, 3))
            rows[s] = r
            r += int(lens[s])
        return rows, r + 2
    src_row, src_rows = place(rng.permutation(len(lens)))
    dst_row, dst_rows = place(rng.permutation(len(lens)))
    src = rng.integers(-2 ** 31, 2 ** 31, (src_rows * src_ld * es + 16) // 4, dtype=np.int64).astype(np.int32)
    dst = rng.integers(-2 ** 31, 2 ** 31, (dst_rows * dst_ld * es + 16) // 4, dtype=np.int64).astype(np.int32)
    return dict(es=es, cols=cols, src_ld=src_ld, dst_ld=dst_ld, src_off=src_off, dst_off=dst_off, lens=lens,
                src_row=src_row, dst_row=dst_row, src=src, dst=dst)


def segment_reference(c):
    src, dst = c["src"].view(np.uint8), c["dst"].copy().view(np.uint8)
    rb, sp, dp = c["cols"] * c["es"], c["src_ld"] * c["es"], c["dst_ld"] * c["es"]
    for s, n in enumerate(c["lens"]):
        for r in range(int(n)):
            a = c["src_off"] + (int(c["src_row"][s]) + r) * sp
            b = c["dst_off"] + (int(c["dst_row"][s]) + r) * dp
            dst[b:b + rb] = src[a:a + rb]
    return dst.view(np.int32)


def _seg_run(c):
    import torch

    from nnmnkwii_b200 import _lib
    src, dst = torch.from_numpy(c["src"]).cuda(), torch.from_numpy(c["dst"]).cuda()
    sr, dr = torch.from_numpy(c["src_row"]).cuda(), torch.from_numpy(c["dst_row"]).cuda()
    ln = torch.from_numpy(c["lens"].astype(np.int32)).cuda()
    sp, dp = src.data_ptr() + c["src_off"], dst.data_ptr() + c["dst_off"]
    rc = _lib.lib.nnk_segment_copy(sp, dp, c["es"], c["cols"], c["src_ld"], c["dst_ld"], sr.data_ptr(), dr.data_ptr(),
                                   ln.data_ptr(), len(c["lens"]), int(c["lens"].max()), _stream())
    _lib.check(rc, "nnk_segment_copy")
    return dst, sp, dp


@pytest.mark.parametrize("case", SEG_CASES, ids=lambda c: c[0])
def test_segment_copy(case):
    _, es, cols, src_ld, dst_ld, so, do = case
    c = _seg_case(es, cols, src_ld, dst_ld, so, do, seed=cols + src_ld)
    dst, sp, dp = _seg_run(c)
    vec = M.segment_copy_vec(cols, es, src_ld, dst_ld, sp, dp)
    assert vec == case[0].startswith("vector")
    assert np.array_equal(dst.cpu().numpy(), segment_reference(c))


# ---- trim_len_kernel ------------------------------------------------------------------------------------------------
TRIM_EPS = 1e-7
TRIM_D = [1, 5, 7, 8, 9, 16, 127, 128, 129, 300, 1000]


def _straddling_rows(D, dt, rng, pairwise_keeps):
    """Rows whose |x| sums, in NumPy's pairwise order and in plain sequential order, fall on opposite sides of
    eps (in dtype): `pairwise_keeps` picks the row that the pairwise sum keeps and the sequential sum drops.
    None for D < 8, where the two orders are the same."""
    if D < 8:
        return None
    eps = dt(TRIM_EPS)
    ulp = float(np.finfo(dt).eps)
    for _ in range(50):
        base = rng.uniform(0.5, 1.5, (2048, D)) * rng.choice([-1.0, 1.0], (2048, D))
        target = float(eps) * (1.0 + rng.uniform(-6.0, 6.0, 2048) * ulp)
        rows = (base / np.abs(base).sum(1, keepdims=True) * target[:, None]).astype(dt)
        pw = np.sum(np.abs(rows), axis=1)
        seq = np.cumsum(np.abs(rows), axis=1)[:, -1]
        hit = (pw >= eps) & (seq < eps) if pairwise_keeps else (seq >= eps) & (pw < eps)
        if hit.any():
            return rows[np.argmax(hit)]
    raise AssertionError("no straddling row found for D=%d %s" % (D, dt))


def _trim_case(D, dt, ld, seed):
    """(n_pairs, T, ld) frames: full, empty, zero tails, rows below eps, NaN, and rows on both sides of eps."""
    rng = np.random.default_rng(seed)
    dt = np.dtype(dt).type
    T = 40
    pairs = []

    def frames(last):
        x = np.zeros((T, D), dt)
        x[:last] = rng.standard_normal((last, D))
        return x
    pairs.append(frames(T))
    pairs.append(np.zeros((T, D), dt))
    x = frames(17)
    x[17:30] = (TRIM_EPS / (4 * D))  # below eps after the sum: trimmed with the zeros
    pairs.append(x)
    x = frames(3)
    x[22, D // 2] = np.nan  # NaN is not < eps: kept
    pairs.append(x)
    x = frames(0)
    x[T - 1, 0] = dt(TRIM_EPS)  # exactly eps: kept
    pairs.append(x)
    for keep in (True, False):
        row = _straddling_rows(D, dt, rng, keep)
        if row is None:
            continue
        for last in (5, T - 1):
            x = frames(2)
            x[last] = row
            pairs.append(x)
    X = np.full((len(pairs), T, ld), 1e3, dt)  # columns past D must be ignored
    for p, x in enumerate(pairs):
        X[p, :, :D] = x
    return X


def _trim_run(X, D):
    import torch

    from nnmnkwii_b200 import _lib
    P, T, ld = X.shape
    dt = np.dtype(X.dtype).name
    xd = torch.from_numpy(X).cuda()
    out = torch.full((P,), -1, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib.nnk_trim_lengths(xd.data_ptr(), _code(dt), T * ld, ld, T, D, TRIM_EPS, P, out.data_ptr(),
                                         _stream()), "nnk_trim_lengths")
    return out


@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("D", TRIM_D)
def test_trim_lengths(D, dt):
    for ld in (D, D + 3):
        X = _trim_case(D, dt, ld, seed=D)
        got = _trim_run(X, D).cpu().numpy()
        want = [oracle.trim_zeros_frames_len(np.ascontiguousarray(x[:, :D]), eps=TRIM_EPS) for x in X]
        assert want[:5] == [40, 0, 17, 23, 40]
        # rows the pairwise order keeps (last row 5, then 39) and rows only the sequential order would keep
        assert want[5:] == ([6, 40, 2, 2] if D >= 8 else [])
        assert got.tolist() == want, (D, dt, ld)


# ---- gather_rows_kernel ---------------------------------------------------------------------------------------------
def _gather_case(D, dt, out_rows, seed):
    """Paths with repeated indices (monotone, like a DTW path) and in random order; lengths 0, 1, < and = out_rows."""
    rng = np.random.default_rng(seed)
    T, x_ld, path_ld = 50, D + 2, out_rows + 7
    lens = np.array([out_rows, 0, 1, out_rows // 3, T], np.int32)
    path = np.full((len(lens), path_ld), 10 ** 6, np.int32)  # entries past a length must not be read
    for p, n in enumerate(lens):
        path[p, :n] = np.sort(rng.integers(0, T, n)) if p % 2 == 0 else rng.integers(0, T, n)
    X = (rng.standard_normal((len(lens), T, x_ld)) * 3).astype(dt)
    return X, path, lens


def _gather_run(X, path, lens, out_rows, D):
    import torch

    from nnmnkwii_b200 import _lib
    P, T, x_ld = X.shape
    dt = np.dtype(X.dtype).name
    xd, pd, ld = (torch.from_numpy(a).cuda() for a in (X, path, lens))
    out = torch.full((P, out_rows, D), float("nan"), dtype=_tdt(dt), device="cuda")
    _lib.check(_lib.lib.nnk_gather_rows(xd.data_ptr(), _code(dt), T * x_ld, x_ld, pd.data_ptr(), path.shape[1],
                                        ld.data_ptr(), out.data_ptr(), out_rows * D, out_rows, D, P, _stream()),
               "nnk_gather_rows")
    return out


@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("D,out_rows", [(1, 120), (7, 120), (64, 333), (300, 1000)])
def test_gather_rows(D, out_rows, dt):
    X, path, lens = _gather_case(D, dt, out_rows, seed=D)
    got = _gather_run(X, path, lens, out_rows, D).cpu().numpy()
    want = np.zeros((len(lens), out_rows, D), X.dtype)
    for p, n in enumerate(lens):
        want[p, :n] = X[p, path[p, :n], :D]
    assert np.array_equal(got, want)


# ---- kernel names ---------------------------------------------------------------------------------------------------
def launch(kind, *args):
    """One call of each launcher, repeatable, for `variant_mirror.profiled_in_child`."""
    if kind == "delta":
        taps, D, dt = args
        rc, _ = _delta_run(_delta_case(tuple(taps), D, dt, seed=1))
        assert rc == 0
    elif kind == "segment":
        _seg_run(_seg_case(*args))
    elif kind == "trim":
        D, dt = args
        _trim_run(_trim_case(D, dt, D, seed=D), D)
    else:
        D, dt, out_rows = args
        X, path, lens = _gather_case(D, dt, out_rows, seed=D)
        _gather_run(X, path, lens, out_rows, D)


def test_kernel_names_follow_the_mirror():
    cases, want = [], []
    for dt in ("float32", "float64"):
        T = _tname(dt)
        cases.append([["delta", [9, 2, 5, 8], 33, dt], r"\bdelta_kernel<"])
        want.append("delta_kernel<%s>" % T)
        cases.append([["trim", 129, dt], r"\btrim_len_kernel<"])
        want.append("trim_len_kernel<%s>" % T)
        cases.append([["gather", 300, dt, 1000], r"\bgather_rows_kernel<"])
        want.append("gather_rows_kernel<%s>" % T)
    for name, es, cols, src_ld, dst_ld, so, do in SEG_CASES:
        cases.append([["segment", es, cols, src_ld, dst_ld, so, do], r"\bsegment_copy_kernel<"])
        want.append("segment_copy_kernel<uint4>" if name.startswith("vector") else "segment_copy_kernel<unsigned int>")
    for (case, _), w, (names, err) in zip(cases, want, M.profiled_in_child("test_variants_data_gpu", "launch",
                                                                            cases)):
        assert err == "None", (case, err)
        assert names and all(w in n for n in names), (case, w, names)


def test_delta_features_cpu_tensor_is_computed_on_the_gpu():
    """A CPU tensor goes to the GPU and comes back as a CPU tensor of its dtype, equal to the NumPy result."""
    import torch

    from nnmnkwii_b200.preprocessing import delta_features
    rng = np.random.default_rng(5)
    ws = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))]
    for dt in (np.float32, np.float64):
        x = rng.standard_normal((120, 7)).astype(dt)
        ref = delta_features(x, ws, lengths=[50, 70])
        y = delta_features(torch.from_numpy(x), ws, lengths=[50, 70])
        assert y.device.type == "cpu" and y.dtype == torch.from_numpy(x).dtype
        assert np.array_equal(y.numpy(), ref)
