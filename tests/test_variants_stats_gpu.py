"""Every kernel instance of the corpus-statistics and per-column affine launchers (csrc/nnk_stats.cu), against
float64 and NumPy references.

`frame_stats_kernel<T>`: `stats_shape` picks the column strips, the strip width CW (32 ... 256), the row slices
RS (1 ... 8), tile_rows = 64 RS and a grid that may be far smaller than the tile count.  These cases call
`nnk_frame_stats` directly at widths on both sides of every strip and slice change, with lengths around
tile_rows, `ld > D`, padded and packed batches and an incoming state, and compare the float64 state vector
with a two-pass float64 mean / m2 over the concatenated valid rows (count, min and max exactly).

`column_affine_kernel<Tin, T, FORM>`: the grid is capped at kNumSMs * 16 blocks, so a thread makes a second
grid-stride pass, which advances its column by `stride % D`, only above 2 162 688 elements.  Each of the six
instances runs at one, two and three passes and must equal the NumPy expression bit for bit.  The kernel
names are checked against `variant_mirror` in a child process (`variant_mirror.profiled_in_child`).

The module is named to sort after every module that asserts kernel names from the pytest process: with these
cases run before them, torch.profiler came back empty for the UnitVarianceMLPG variant cases in a full GPU run on
an H100 (they pass alone and after these modules alone), so their names are collected in child processes and
their numbers come last."""
import ctypes

import numpy as np
import pytest

import variant_mirror as M
from conftest import rel_err

pytestmark = pytest.mark.gpu

STATS_D = [1, 32, 33, 100, 129, 256, 257, 513, 769]



def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _code(dt):
    from nnmnkwii_b200 import _lib
    return _lib.NNK_F32 if np.dtype(dt) == np.float32 else _lib.NNK_F64


# ---- frame_stats_kernel ---------------------------------------------------------------------------------------------
def _columns(rng, n, D, dt):
    """Rows with per-column offsets and scales (well-conditioned, not centred)."""
    mu, sd = rng.uniform(-3.0, 3.0, D), rng.uniform(0.5, 2.0, D)
    return (rng.standard_normal((n, D)) * sd + mu).astype(dt)


def _incoming(rng, D, n0):
    """[count, mean, m2, min, max] of n0 earlier float64 rows (n0 = 0: the empty state) and the rows."""
    rows = _columns(rng, n0, D, np.float64) if n0 else np.zeros((0, D))
    st = np.empty(1 + 4 * D)
    st[0] = n0
    if n0:
        mean = rows.mean(0)
        st[1:1 + D], st[1 + D:1 + 2 * D] = mean, np.square(rows - mean).sum(0)
        st[1 + 2 * D:1 + 3 * D], st[1 + 3 * D:] = rows.min(0), rows.max(0)
    else:
        st[1:1 + 2 * D] = 0.0
        st[1 + 2 * D:1 + 3 * D], st[1 + 3 * D:] = np.inf, -np.inf
    return st, rows


def _stats_run(buf, D, ld, off, lens, n_utt, max_rows, state):
    """nnk_frame_stats over `buf` (host, flat rows of `ld` elements); returns the state vector."""
    import torch

    from nnmnkwii_b200 import _lib
    x = torch.from_numpy(buf).cuda()
    od = torch.from_numpy(np.asarray(off, np.int64)).cuda()
    ld_t = torch.from_numpy(np.asarray(lens, np.int32)).cuda() if lens is not None else None
    st = torch.from_numpy(state.copy()).cuda()
    ws = torch.empty(int(_lib.lib.nnk_frame_stats_workspace_bytes(n_utt, max_rows, D)), dtype=torch.uint8, device="cuda")
    _lib.check(_lib.lib.nnk_frame_stats(x.data_ptr(), _code(buf.dtype), D, ld, od.data_ptr(),
                                        ld_t.data_ptr() if ld_t is not None else None, n_utt, max_rows, st.data_ptr(),
                                        ws.data_ptr(), ws.numel(), _stream()), "nnk_frame_stats")
    return st.cpu().numpy()


def _check_state(got, rows, D, what):
    rows = rows.astype(np.float64)
    mean = rows.mean(0)
    assert got[0] == len(rows), (what, got[0], len(rows))
    assert rel_err(got[1:1 + D], mean) <= 1e-12, what
    assert rel_err(got[1 + D:1 + 2 * D], np.square(rows - mean).sum(0)) <= 1e-12, what
    assert np.array_equal(got[1 + 2 * D:1 + 3 * D], rows.min(0)), what
    assert np.array_equal(got[1 + 3 * D:], rows.max(0)), what


def _padded_case(D, dt, seed):
    """(B, T, D + 5) padded batch, lengths at tile_rows - 1, tile_rows, tile_rows + 1, 0, 1, above T, 2 tiles + 1."""
    rng = np.random.default_rng(seed)
    tr = M.stats_shape(1, 1, D)["tile_rows"]
    T = 2 * tr + 1
    lens = np.array([tr - 1, tr, tr + 1, 0, 1, T + 50, 2 * tr + 1, int(rng.integers(1, T))], np.int64)
    B, W = len(lens), D + 5
    x = np.full((B, T, W), 1e6, dt)  # padding rows and columns: must not enter the statistics
    for b, n in enumerate(lens):
        x[b, :min(n, T), :D] = _columns(rng, min(n, T), D, dt)
    return x, lens, rng


@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("D", STATS_D)
def test_frame_stats_every_geometry(D, dt):
    x, lens, rng = _padded_case(D, dt, seed=D)
    B, T, W = x.shape
    valid = np.concatenate([x[b, :min(n, T), :D] for b, n in enumerate(lens)])
    # padded batch read in place (ld = D + 5), clipped lengths, and a non-empty incoming state
    state, prior = _incoming(rng, D, 7)
    got = _stats_run(x.reshape(-1), D, W, np.arange(B + 1) * T, lens, B, T, state)  # lengths above T clip
    _check_state(got, np.concatenate([prior, valid.astype(np.float64)]), D, "padded")
    # the same rows packed back to back (ld = D, no lengths), empty incoming state
    off = np.concatenate([[0], np.cumsum(np.minimum(lens, T))])
    got = _stats_run(np.ascontiguousarray(valid).reshape(-1), D, D, off, None, B, int(np.minimum(lens, T).max()),
                     _incoming(rng, D, 0)[0])
    _check_state(got, valid, D, "packed")


@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("D,n_utt", [(1, 1300), (769, 300)])
def test_frame_stats_many_tiles_per_block(D, n_utt, dt):
    """Three or more tiles per block: n_tiles >= 3 * grid."""
    rng = np.random.default_rng(D)
    tr = M.stats_shape(1, 1, D)["tile_rows"]
    s = M.stats_shape(n_utt, tr, D)
    assert s["n_tiles"] >= 3 * s["grid"], s
    lens = rng.integers(0, tr + 1, n_utt)
    x = _columns(rng, n_utt * tr, D, dt)
    got = _stats_run(x.reshape(-1), D, D, np.arange(n_utt + 1) * tr, lens, n_utt, tr, _incoming(rng, D, 0)[0])
    valid = np.concatenate([x[u * tr:u * tr + n] for u, n in enumerate(lens)])
    _check_state(got, valid, D, "many tiles")


@pytest.mark.parametrize("dt", ["float32", "float64"])
def test_column_slice_is_bit_identical(dt):
    """Form (c) on x[:, :, a:b] (read in place, ld > D) equals the contiguous copy bit for bit."""
    import torch

    from nnmnkwii_b200.preprocessing import normalize as P
    rng = np.random.default_rng(5)
    x = torch.from_numpy(_columns(rng, 6 * 300, 200, dt).reshape(6, 300, 200)).cuda()
    lens = [300, 0, 1, 129, 64, 257]
    for a, b in ((3, 160), (0, 1), (10, 43)):
        view = x[:, :, a:b]
        assert not view.is_contiguous()
        for f in (P.meanvar, P.minmax):
            for s, t in zip(f(view, lens), f(view.contiguous(), lens)):
                assert torch.equal(s, t), (dt, a, b, f.__name__)


# ---- column_affine_kernel ---------------------------------------------------------------------------------------------
AFFINE_D = [1, 3, 187, 256, 257, 425, 1024]
PASS_ELEMS = {1: 1_000_000, 2: 3_000_000, 3: 6_000_000}
# (x dtype, computed dtype): the three dtype instances of column_affine_kernel<Tin, T, FORM>
AFFINE_TYPES = [("float32", "float32"), ("float32", "float64"), ("float64", "float64")]


def affine_reference(x, a, b, form):
    """The reference's NumPy expression in the computed dtype: (x - a) / b or x * b + a."""
    xc = x.astype(a.dtype)
    return (xc - a) / b if form == 0 else xc * b + a


def _affine_run(x, a, b, form):
    import torch

    from nnmnkwii_b200 import _lib
    D = x.shape[-1]
    xd, ad, bd = (torch.from_numpy(v).cuda() for v in (x, a, b))
    out = torch.empty(x.shape, dtype=getattr(torch, a.dtype.name), device="cuda")
    _lib.check(_lib.lib.nnk_column_affine(xd.data_ptr(), _code(x.dtype), _code(a.dtype), x.size // D, D, ad.data_ptr(),
                                          bd.data_ptr(), form, out.data_ptr(), _stream()), "nnk_column_affine")
    return out


def _affine_case(D, passes, seed):
    rng = np.random.default_rng(seed)
    rows = -(-PASS_ELEMS[passes] // D)
    x = rng.standard_normal((rows, D)) * 7
    a, b = rng.standard_normal(D), rng.uniform(0.1, 3.0, D)
    return x, a, b


@pytest.mark.parametrize("D", AFFINE_D)
def test_column_affine_every_instance_and_pass_count(D):
    strides = set()
    for passes in (1, 2, 3):
        x64, a64, b64 = _affine_case(D, passes, seed=D + passes)
        got_passes, _, stride_c = M.affine_passes(x64.size, D)
        assert got_passes == passes, (D, passes, got_passes)
        strides.add(stride_c)
        for xdt, cdt in AFFINE_TYPES:
            x = x64.astype(xdt)
            a, b = a64.astype(cdt), b64.astype(cdt)
            for form in (0, 1):
                got = _affine_run(x, a, b, form).cpu().numpy()
                assert np.array_equal(got, affine_reference(x, a, b, form)), (D, passes, xdt, cdt, form)
    assert (0 in strides) == (D in (1, 3, 256, 1024)), strides  # both column steps between passes are covered


# ---- kernel names ---------------------------------------------------------------------------------------------------
def launch(kind, *args):
    if kind == "stats":
        D, dt = args
        x, lens, rng = _padded_case(D, dt, seed=D)
        B, T, W = x.shape
        _stats_run(x.reshape(-1), D, W, np.arange(B + 1) * T, np.minimum(lens, T), B, T, _incoming(rng, D, 0)[0])
    else:
        xdt, cdt, form = args
        x, a, b = _affine_case(257, 2, seed=1)
        _affine_run(x.astype(xdt), a.astype(cdt), b.astype(cdt), form)


def test_kernel_names_follow_the_mirror():
    cases, want = [], []
    for dt in ("float32", "float64"):
        cases.append([["stats", 257, dt], r"\bframe_stats_kernel<"])
        want.append("frame_stats_kernel<%s>" % ("float" if dt == "float32" else "double"))
    for xdt, cdt in AFFINE_TYPES:
        for form in (0, 1):
            cases.append([["affine", xdt, cdt, form], r"\bcolumn_affine_kernel<"])
            want.append("column_affine_kernel<%s, %s, %d>" % ("float" if xdt == "float32" else "double",
                                                               "float" if cdt == "float32" else "double", form))
    got = M.profiled_in_child("test_variants_stats_gpu", "launch", cases)
    for (case, _), w, (names, err) in zip(cases, want, got):
        assert err == "None", (case, err)
        assert names and all(w in n for n in names), (case, w, names)
