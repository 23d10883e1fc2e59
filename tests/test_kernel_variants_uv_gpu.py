"""Every sweep `UnitVarianceMLPG` can select, against the float64 dense product with the same R.

`_uvmlpg.band_of` reduces R to its band (half-width K) and picks, separately for the forward and the
backward table: the factored sweep (`nnk_uv_apply_factored`, one long filter plus 3- or 5-tap stencils,
KC = 1 or 2, K buckets 16 / 24 / 32), the shift-invariant sweep (`nnk_uv_apply_toeplitz`, K buckets
8 / 16 / 24 / 32 / 48 / 64, nw = 1..3) or the per-row table (`nnk_uv_apply`: K > 64, a shift-invariant run
shorter than 64 rows, or a float64 R).  Where a path begins depends on the float32 R the device builds, so
each case scans a short list of window sets (host-side K values in the comments, at T = 400) and takes the
first one whose band lands where the case wants; the kernel name is then asserted from the profiler.  The names
are collected in a child process (`variant_mirror.profiled_in_child`): late in a long pytest process,
torch.profiler has returned empty profiles for these calls on an H100."""
import numpy as np
import pytest

import variant_mirror as M
from conftest import rel_err, windows_set

pytestmark = pytest.mark.gpu

T_UV = 400
D1 = windows_set()[2][1]
D2 = windows_set()[2][2]
F1, F2 = windows_set()[3][1], windows_set()[3][2]
SEVEN_TAP = (3, 3, np.array([-3.0, -2.0, -1.0, 0.0, 1.0, 2.0, 3.0]) / 28.0)


def std_c(c):  # static coefficient c, delta, delta-delta: K = 11 (5.0), 15 (3.0), 20 (1.5), 23 (1.0), 26 (0.7), 39 (0.5), 71 (0.3)
    return [(0, 0, np.array([c])), D1, D2]


def five_c(c):  # 5-point windows of windows_set()[3]: K = 11 (8.0), 13 (5.0), 19 (2.0), 25 (1.0), 28 (0.7)
    return [(0, 0, np.array([c])), F1, F2]


def one_c(a):  # a single 3-tap window: K = 7 (0.05), 11 (0.15), 20 (0.3), 31 (0.4), 47 (0.45), 62 (0.47)
    return [(1, 1, np.array([a, 1.0, a]))]


def seven_c(c):  # static + 7-tap delta (does not factor): K = 18 (4.0), 23 (2.0), 32 (1.0), 49 (0.5)
    return [(0, 0, np.array([c])), SEVEN_TAP]


def seven3_c(c):  # static + delta + 7-tap window (does not factor): K = 15 (8.0), 24 (2.0), 28 (1.5), 36 (1.0), 53 (0.6)
    return [(0, 0, np.array([c])), D1, SEVEN_TAP]


def _kk(K, buckets):
    return next(b for b in buckets if K <= b)


def _paths(band):
    """(forward path, backward path): "fact<KK,KC>", "toep<KK,nw>" or "table", as `apply_forward` /
    `apply_backward` choose them."""
    out = []
    for toep, fact in ((band.toep, band.fact), (band.toepT, band.factT)):
        if toep is not None and fact is not None:
            out.append("fact<%d,%d>" % (_kk(band.K, (16, 24, 32)), fact[0]))
        elif toep is not None:
            out.append("toep<%d,%d>" % (_kk(band.K, (8, 16, 24, 32, 48, 64)), band.nw))
        else:
            out.append("table")
    return tuple(out)


def _band_for(want, family, cands, T=T_UV):
    import torch
    from nnmnkwii_b200 import _uvmlpg as uv
    from nnmnkwii_b200 import paramgen as G
    seen = []
    for c in cands:
        ws = family(c)
        Rt = torch.from_numpy(G.unit_variance_mlpg_matrix(ws, T)).cuda()
        band = uv.band_of(Rt, Rt.device)
        seen.append((c, band.K, _paths(band)))
        if _paths(band) == (want, want):
            return ws, Rt, band
    pytest.fail("no candidate lands on %s: %s" % (want, seen))


_NAME = {"fact": r"uv_fact_%s_kernel<%d, %d,", "toep": r"uv_(toeplitz2|%s_toeplitz)_kernel<%d, %d,"}


def _expect_kernel(names, path, direction, dtype):
    if path == "table":
        pat = r"uv_%s_kernel<%s, 4>" % (direction, dtype)
    else:
        kind, args = path.split("<")
        a, b = (int(s) for s in args.rstrip(">").split(","))
        pat = _NAME[kind] % (direction, a, b)
    assert M.launched(names, pat), (pat, [n for n in names if "uv_" in n])


def _dense_ref(R64, x, go, nw, reshaped):
    """float64 y = R x and g = R^T go per batch item, in the layout of x."""
    B = x.shape[0]
    T = R64.shape[0]
    xr = x if reshaped else x.reshape(B, T, nw, -1).transpose(0, 2, 1, 3).reshape(B, nw * T, -1)
    y = np.einsum("ts,bsd->btd", R64, xr)
    g = np.einsum("st,bsd->btd", R64, go)  # (B, nw*T, sd)
    if not reshaped:
        g = g.reshape(B, nw, T, -1).transpose(0, 2, 1, 3).reshape(B, T, -1)
    return y, g


def _inputs(band, dtype, sd, reshaped):
    nw, T = band.nw, band.T
    rng = np.random.default_rng(band.K + 10 * sd + reshaped)
    shape = (2, nw * T, sd) if reshaped else (2, T, nw * sd)
    xh = rng.standard_normal(shape).astype(np.float32 if dtype == "float" else np.float64)
    goh = rng.standard_normal((2, T, sd)).astype(xh.dtype)
    return xh, goh


COMBOS = [(sd, reshaped) for sd in (5, 6) for reshaped in (False, True)]


FACT = [
    ("fact<16,1>", std_c, (5.0, 4.0, 3.0)),
    ("fact<24,1>", std_c, (1.5, 2.0, 1.0)),
    ("fact<32,1>", std_c, (0.7, 0.6, 0.8)),
    ("fact<16,2>", five_c, (5.0, 8.0, 3.0)),
    ("fact<24,2>", five_c, (2.0, 1.5, 3.0)),
    ("fact<32,2>", five_c, (1.0, 0.7)),
]
TOEP = [
    ("toep<8,1>", one_c, (0.05, 0.02)),
    ("toep<16,1>", one_c, (0.15, 0.1, 0.2)),
    ("toep<24,1>", one_c, (0.3, 0.25, 0.33)),
    ("toep<32,1>", one_c, (0.4, 0.38)),
    ("toep<48,1>", one_c, (0.45, 0.44, 0.43)),
    ("toep<64,1>", one_c, (0.47, 0.465, 0.475)),
    ("toep<24,2>", seven_c, (2.0, 4.0, 3.0)),
    ("toep<32,2>", seven_c, (1.0, 1.2, 0.9)),
    ("toep<64,2>", seven_c, (0.5, 0.45)),
    ("toep<16,3>", seven3_c, (8.0, 10.0, 12.0)),
    ("toep<48,3>", seven3_c, (1.0, 0.9)),
    ("toep<64,3>", seven3_c, (0.6, 0.55)),
]
# every case of `_run_and_check`, as `_case` rebuilds it
CASES = ([("band", want, family.__name__, cands) for want, family, cands in FACT + TOEP]
         + [("band", "table", "std_c", (0.3, 0.25)), ("short", 0), ("short", 1), ("f64", 0), ("f64", 1)])


def _key(case):
    return tuple(tuple(c) if isinstance(c, (list, tuple)) else c for c in case)


@pytest.fixture(scope="module")
def uv_names():
    """(case, sd, reshaped, direction) -> names of the UV kernels of that call, all profiled in one child."""
    cases = [([list(c) if isinstance(c, tuple) else c for c in case], sd, reshaped, d)
             for case in CASES for sd, reshaped in COMBOS for d in ("fwd", "bwd")]
    res = M.profiled_in_child("test_kernel_variants_uv_gpu", "launch", [(list(c), r"\buv_\w*kernel\b") for c in cases])
    out = {}
    for (case, sd, reshaped, d), (names, err) in zip(cases, res):
        assert err == "None", (case, err)
        out[(_key(case), sd, reshaped, d)] = names
    return out


def _run_and_check(names_of, case, Rt, band, bound_kind):
    """Forward and backward, plain and reshaped layouts, odd and even static_dim; ``names_of`` (the `uv_names`
    fixture) names the kernel of each call."""
    import torch
    from nnmnkwii_b200.autograd import UnitVarianceMLPG
    fwd_path, bwd_path = _paths(band)
    T, nw = band.T, band.nw
    R64 = Rt.double().cpu().numpy()
    dtype = "double" if Rt.dtype == torch.float64 else "float"
    for sd, reshaped in COMBOS:
        for direction, path in (("fwd", fwd_path), ("bwd", bwd_path)):
            _expect_kernel(names_of[(_key(case), sd, reshaped, direction)], path, direction, dtype)
        xh, goh = _inputs(band, dtype, sd, reshaped)
        x = torch.from_numpy(xh).cuda().requires_grad_(True)
        y = UnitVarianceMLPG.apply(x, Rt)
        g = torch.autograd.grad(y, x, torch.from_numpy(goh).cuda(), retain_graph=True)[0]
        y_ref, g_ref = _dense_ref(R64, xh.astype(np.float64), goh.astype(np.float64), nw, reshaped)
        got_y, got_g = y.detach().cpu().numpy(), g.cpu().numpy()
        assert got_y.shape == y_ref.shape and got_g.shape == g_ref.shape
        if bound_kind == "table":
            tol = 2e-6 if dtype == "float" else 1e-13
            assert rel_err(got_y, y_ref) < tol and rel_err(got_g, g_ref) < tol, (sd, reshaped)
        else:
            # shift-invariant rows: the bound _uvmlpg.py documents, (2K+1) nw 2^-23 max|R| max|x| per output
            peak = np.abs(R64).max()
            scale = (2 * band.K + 1) * nw * 2.0 ** -23 * peak
            assert np.abs(got_y - y_ref).max() <= scale * np.abs(xh).max(), (sd, reshaped)
            assert np.abs(got_g - g_ref).max() <= scale * np.abs(goh).max(), (sd, reshaped)


FAMILIES = {"std_c": std_c, "five_c": five_c, "one_c": one_c, "seven_c": seven_c, "seven3_c": seven3_c}
_launched = {}


def _case(case):
    """(R, band) of a case: ("band", want, family, cands), ("short", dT) or ("f64", i)."""
    import torch
    from nnmnkwii_b200 import _uvmlpg as uv
    from nnmnkwii_b200 import paramgen as G
    if case[0] == "band":
        _, Rt, band = _band_for(case[1], FAMILIES[case[2]], case[3])
        return Rt, band
    if case[0] == "short":
        return _short_run_bands()[case[1]]
    ws = (windows_set()[2], five_c(1.0))[case[1]]
    Rt = torch.from_numpy(G.unit_variance_mlpg_matrix(ws, 300)).cuda().double()
    return Rt, uv.band_of(Rt, Rt.device)


def launch(case, sd, reshaped, direction):
    """One call of `_run_and_check` in a child process: the forward of (case, sd, reshaped), or the backward of
    the forward made before."""
    import torch
    from nnmnkwii_b200.autograd import UnitVarianceMLPG
    key = (_key(case), sd, reshaped)
    if direction == "fwd":
        Rt, band = _launched.get(key[0]) or _case(case)
        _launched[key[0]] = (Rt, band)
        xh, goh = _inputs(band, "double" if Rt.dtype == torch.float64 else "float", sd, reshaped)
        x = torch.from_numpy(xh).cuda().requires_grad_(True)
        go = torch.from_numpy(goh).cuda()
        torch.cuda.synchronize()
        _launched[key] = (x, go, UnitVarianceMLPG.apply(x, Rt))
    else:
        x, go, y = _launched[key]
        torch.autograd.grad(y, x, go, retain_graph=True)
    torch.cuda.synchronize()


@pytest.mark.parametrize("want,family,cands", FACT, ids=lambda v: v if isinstance(v, str) else None)
def test_factored_buckets(want, family, cands, uv_names):
    ws, Rt, band = _band_for(want, family, cands)
    _run_and_check(uv_names, ("band", want, family.__name__, cands), Rt, band, "bound")


@pytest.mark.parametrize("want,family,cands", TOEP, ids=lambda v: v if isinstance(v, str) else None)
def test_toeplitz_buckets(want, family, cands, uv_names):
    ws, Rt, band = _band_for(want, family, cands)
    _run_and_check(uv_names, ("band", want, family.__name__, cands), Rt, band, "bound")


def test_table_path_wide_band_float32(uv_names):
    """Static coefficient 0.3: K > 64, beyond every shift-invariant kernel."""
    ws, Rt, band = _band_for("table", std_c, (0.3, 0.25))
    assert band.K > 64
    _run_and_check(uv_names, ("band", "table", "std_c", (0.3, 0.25)), Rt, band, "table")


def _short_run_bands():
    """Standard windows: (R, band) at the largest T in 80..129 whose bands both take the per-row table, and one
    frame more."""
    import torch
    from nnmnkwii_b200 import _uvmlpg as uv
    from nnmnkwii_b200 import paramgen as G
    ws = windows_set()[2]
    bands = {}
    for T in range(80, 130):
        Rt = torch.from_numpy(G.unit_variance_mlpg_matrix(ws, T)).cuda()
        bands[T] = (Rt, uv.band_of(Rt, Rt.device))
    T_last = max(T for T, (_, b) in bands.items() if _paths(b) == ("table", "table"))
    assert T_last + 1 in bands
    return bands[T_last], bands[T_last + 1]


def test_table_path_short_shift_invariant_run_float32(uv_names):
    """Standard windows at the largest T whose shift-invariant run is still shorter than 64 rows (K < 64):
    the per-row table; one frame more reaches 64 rows and leaves the table on at least one side."""
    from nnmnkwii_b200 import _uvmlpg as uv
    (Rt, band), nxt = _short_run_bands()
    assert _paths(nxt[1]) != ("table", "table")
    assert band.K <= 64 and band.T >= uv.TOEPLITZ_MIN_ROWS
    _run_and_check(uv_names, ("short", 0), Rt, band, "table")
    _run_and_check(uv_names, ("short", 1), *nxt, "bound")


def test_table_path_float64(uv_names):
    import torch
    from nnmnkwii_b200 import _uvmlpg as uv
    from nnmnkwii_b200 import paramgen as G
    for i, ws in enumerate((windows_set()[2], five_c(1.0))):
        Rt = torch.from_numpy(G.unit_variance_mlpg_matrix(ws, 300)).cuda().double()
        band = uv.band_of(Rt, Rt.device)
        assert _paths(band) == ("table", "table")
        _run_and_check(uv_names, ("f64", i), Rt, band, "table")
