"""Every `mlpg_kernel` instance in the global-variance (MODE_GV) and solve (MODE_SOLVE) modes, GV batches split
into workspace waves, and `nnk_segment_moments` at every grid shape, against the float64 restatements.

`pick_instance` (csrc/nnk_mlpg.cu) serves a window set with one of four template instances; the standard sets
only reach instances 0-2, so instance 3 (NW = 4, L = U = 4, band depth 8) is driven here by a four-window set
and a three-window set with a half-width-3 window.  Each case names the kernel it expects and the profiler
confirms it ran; the names are collected in a child process (`variant_mirror.profiled_in_child`) so that the
profiles do not disturb the later variant modules' own.

GV comparisons guard against tie flips: a trial whose objective is within rounding of the current one can be
kept by the kernel and dropped by the oracle, or the other way round, without either being wrong.  Every trial
of every chain compared here clears a relative gap of 1e-9, so a mismatch is a kernel bug."""
import ctypes

import numpy as np
import pytest

import oracle
import oracle.gv as ogv
import variant_mirror as M
from conftest import rel_err, windows_set
from test_kernel_variants_mlpg_gpu import WIN_NW2_HW2, WIN_NW3_HW3, WIN_NW4

pytestmark = pytest.mark.gpu

MODE_SOLVE, MODE_GV = 2, 3
SETS = {
    "w0": windows_set()[0], "w1": windows_set()[1], "w2": windows_set()[2], "w3": windows_set()[3],
    "nw2_halfwidth2": WIN_NW2_HW2, "nw3_halfwidth3": WIN_NW3_HW3, "nw4": WIN_NW4,
}
# window set -> (instance, NW, L, U) of the mlpg_kernel that serves it
INSTANCE = {
    "w0": (0, 1, 0, 0),
    "w1": (1, 3, 1, 1), "w2": (1, 3, 1, 1),
    "w3": (2, 3, 2, 2), "nw2_halfwidth2": (2, 3, 2, 2),
    "nw3_halfwidth3": (3, 4, 4, 4), "nw4": (3, 4, 4, 4),
}
DT = {"f32": np.float32, "f64": np.float64}
LENS = [257, 1, 9, 2, 17, 8]  # T <= 2 m_edge zeroes every dynamic precision: 1 and 2 always, 8 on instance 3
GAP = 1e-9
# Trials per chain.  Kept trials bring c towards the optimum, where a trial changes F by less than rounding;
# with five, the draws of data stay clear of that (see `_draw`) and every case both keeps and rejects trials.
N_ITER = 5
TOL32, TOL64, TOL_F = 1e-5, 1e-8, 1e-10  # as tests/test_gv_gpu.py


def kernel_name(name, dtype, mode):
    """`mlpg_kernel<Tin, NW, L, U, MODE, PF>` of window set `name`: PF = 4 when L + U <= 2, otherwise 2."""
    _, NW, L, U = INSTANCE[name]
    tin = "float" if np.dtype(dtype) == np.float32 else "double"
    return "mlpg_kernel<%s, %d, %d, %d, %d, %d>" % (tin, NW, L, U, mode, 4 if L + U <= 2 else 2)


def gv_cap(lens, n_chain, windows, k):
    """A workspace cap worth `k` utterances of this batch's GV scratch (which has four more columns per frame
    than the forward solve's)."""
    from nnmnkwii_b200 import _lib
    need = _lib.lib.nnk_mlpg_gv_workspace_bytes(len(lens), n_chain, int(max(lens)), ctypes.byref(_lib.make_windows(windows)))
    assert need % len(lens) == 0
    return k * (need // len(lens))


def _G():
    from nnmnkwii_b200 import paramgen as G
    return G


def _offsets(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)


def _data(rng, lens, D, dtype, var_global):
    n = int(np.sum(lens))
    m = np.cumsum(rng.standard_normal((n, D)), axis=0) * 0.05 + rng.standard_normal((n, D)) * 0.3
    v = (rng.random(D) + 0.5) if var_global else (rng.random((n, D)) + 0.5)
    return m.astype(dtype), v.astype(dtype)


def _gv_params(rng, m, v, w, lens, sd):
    """gv_mean a few times the c_m variance of the longest utterance, gv_var about gv_mean squared: from the
    rescaled start point the first full step overshoots on some chains and is kept on others."""
    u = int(np.argmax(lens))
    a, b = _offsets(lens)[u:u + 2]
    cm = ogv.mlpg(m[a:b], v if v.ndim == 1 else v[a:b], w)
    gm = cm.var(axis=0) * (1.5 + 2.5 * rng.random(sd)) + 1e-3
    gvv = gm ** 2 * (0.5 + rng.random(sd))
    return gm, gvv


class Tie(AssertionError):
    """A trial of the oracle within rounding of a tie."""


def _reference(m, v, w, gm, gvv, n_iter, step=1.0, weight=None, trials=None):
    """oracle.gv.mlpg_gv of one utterance, chain by chain with a trace.  Raises `Tie` if a trial's objective is
    within a relative 1e-9 of the current one; counts the rejected / kept trials of chains of two or more frames
    into ``trials``."""
    T = m.shape[0]
    sd = m.shape[1] // len(w)
    ref = np.zeros((T, sd))
    for d in range(sd):
        mm, vv = ogv.chain_system(m, v, w, d)
        trace = []
        ref[:, d] = ogv.mlpg_gv_chain(mm, vv, w, gm[d], gvv[d], n_iter, step, weight, trace)
        f = trace[0][0]
        for i, (f2, ok) in enumerate(trace[1:]):
            if T == 1:  # v(c) == 0 for every c: the GV gradient vanishes, every trial is c' == c
                assert f2 == f, (d, i, f2, f)
            elif not abs(f2 - f) > GAP * abs(f):
                raise Tie("trial %d of chain %d (T = %d) is within rounding of a tie: %r, %r" % (i, d, T, f2, f))
            elif trials is not None:
                trials[bool(ok)] += 1
            if ok:
                f = f2
    return ref


def _compare(y, ref, m, v, w, gm, gvv, weight=None):
    """The bars of tests/test_gv_gpu.py: float64 trajectories within 1e-8 and their objective within 1e-10 of
    the oracle's, float32 within 1e-5."""
    err = np.abs(np.asarray(y, np.float64) - ref).max() / max(1e-300, np.abs(ref).max())
    if y.dtype == np.float32:
        assert err <= TOL32, err
        return
    assert err <= TOL64, err
    for d in range(ref.shape[1]):
        fr = ogv.chain_objective(m, v, w, d, ref[:, d], gm[d], gvv[d], weight)
        fy = ogv.chain_objective(m, v, w, d, y[:, d], gm[d], gvv[d], weight)
        assert abs(fy - fr) <= TOL_F * max(abs(fr), 1e-300), (d, fy, fr)


def _check(y, m, v, w, gm, gvv, n_iter):
    _compare(y, _reference(m, v, w, gm, gvv, n_iter), m, v, w, gm, gvv)


def _draw(name, dt, var_global, sd):
    """Data of one case of `test_gv_every_instance` and the oracle's trajectories, utterance by utterance.  The
    data is drawn again (from the next seed) while a trial of the oracle is within rounding of a tie."""
    w, dtype = SETS[name], DT[dt]
    off = _offsets(LENS)
    for attempt in range(8):
        rng = np.random.default_rng([list(SETS).index(name), dt == "f32", var_global, sd, attempt])
        m, v = _data(rng, LENS, len(w) * sd, dtype, var_global)
        gm, gvv = _gv_params(rng, m, v, w, LENS, sd)
        trials = [0, 0]
        try:
            refs = [_reference(m[a:b], v if var_global else v[a:b], w, gm, gvv, N_ITER, trials=trials)
                    for a, b in zip(off[:-1], off[1:])]
        except Tie:
            continue
        return m, v, gm, gvv, refs, trials
    raise AssertionError("no draw of %s clear of ties" % ((name, dt, var_global, sd),))


def _wave_batch(name, dtype):
    """Eleven utterances, not sorted by length, of window set `name` (seven static dimensions)."""
    w = SETS[name]
    rng = np.random.default_rng(31 + INSTANCE[name][0])
    lens = np.array([23, 70, 5, 41, 1, 66, 12, 58, 9, 33, 47])
    m, v = _data(rng, lens, 7 * len(w), dtype, False)
    gm, gvv = _gv_params(rng, m, v, w, lens, 7)
    return m, v, lens, gm, gvv


def _many_utterances():
    """65 537 utterances of 1-3 frames, D = 3: one more grid row than two launches of 65 535 minus one."""
    rng = np.random.default_rng(65537)
    lens = rng.integers(1, 4, size=65537)
    lens[-2:] = 3  # the second launch's utterances have a non-zero variance
    x = (rng.standard_normal((int(lens.sum()), 3)) * 2.0 + 1e4).astype(np.float32)
    return x, lens


def launch(kind, *args):
    """One call of each case whose kernels the profiler names (in a child process, see `kernels`)."""
    import torch

    from nnmnkwii_b200 import _device as dev
    G = _G()
    if kind == "gv":
        name, dt, var_global = args
        w = SETS[name]
        m, v = _data(np.random.default_rng(1), [17, 9], 5 * len(w), DT[dt], var_global)
        G.mlpg_gv_batch(m, v, w, np.full(5, 0.5), np.full(5, 0.1), lengths=[17, 9])
    elif kind == "solve":
        G.unit_variance_mlpg_matrix(SETS[args[0]], args[1])
    elif kind == "waves":
        name, dt, k = args
        m, v, lens, gm, gvv = _wave_batch(name, DT[dt])
        old = dev.WORKSPACE_CAP_BYTES
        if k:
            dev.WORKSPACE_CAP_BYTES = gv_cap(lens, m.shape[1] // len(SETS[name]), SETS[name], k)
        try:
            G.mlpg_gv_batch(m, v, SETS[name], gm, gvv, lengths=lens, n_iter=N_ITER)
        finally:
            dev.WORKSPACE_CAP_BYTES = old
    elif kind == "moments":
        x, lens = _many_utterances()
        G.global_variance(x, lengths=lens)
    else:
        raise ValueError(kind)
    torch.cuda.synchronize()


MLPG_FAMILY = r"\bmlpg_(fwd_as_)?kernel<"
WAVE_SETS, WAVE_KS = ("w2", "nw4"), (0, 1, 3, 6)  # k = 0: the default cap, one launch


@pytest.fixture(scope="module")
def kernels():
    """case -> names of the kernels of its family, one per launch."""
    cases = [(["gv", n, dt, vg], MLPG_FAMILY) for n in SETS for dt in DT for vg in (False, True)]
    cases += [(["solve", n, 40], MLPG_FAMILY) for n in ("nw2_halfwidth2", "nw3_halfwidth3", "nw4")]
    cases += [(["waves", n, dt, k], MLPG_FAMILY) for n in WAVE_SETS for dt in DT for k in WAVE_KS]
    cases += [(["moments"], r"\bsegment_moments_kernel<")]
    res = M.profiled_in_child("test_kernel_variants_gv_gpu", "launch", cases, repeats=True)
    out = {}
    for (case, _), (names, err) in zip(cases, res):
        assert err == "None", (case, err)
        out[tuple(case)] = names
    return out


def _assert_only(names, kernel):
    """`kernel` ran, and no other MLPG kernel did."""
    assert names and all(kernel in n for n in names), (kernel, names)


# ---- 1. GV on every instance ------------------------------------------------------------------------------------
@pytest.mark.parametrize("var_global", [False, True], ids=["var_frame", "var_global"])
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("name", list(SETS))
def test_gv_every_instance(name, dt, var_global, kernels):
    G = _G()
    w, dtype = SETS[name], DT[dt]
    inst = INSTANCE[name]
    assert M.pick_instance(w) == inst[1:]
    _assert_only(kernels[("gv", name, dt, var_global)], kernel_name(name, dtype, MODE_GV))
    off = _offsets(LENS)
    kept = rejected = 0
    for sd in (5, 33):  # 33: a partial second chain group
        m, v, gm, gvv, refs, trials = _draw(name, dt, var_global, sd)
        rejected, kept = rejected + trials[0], kept + trials[1]
        y = G.mlpg_gv_batch(m, v, w, gm, gvv, lengths=LENS, n_iter=N_ITER)
        assert y.dtype == dtype and y.shape == (sum(LENS), sd)
        for u, (a, b) in enumerate(zip(off[:-1], off[1:])):
            _compare(y[a:b], refs[u], m[a:b], v if var_global else v[a:b], w, gm, gvv)
    assert kept and rejected, (kept, rejected)  # both outcomes of a trial ran


@pytest.mark.parametrize("name", ["w1", "nw4"])
def test_gv_mean_zero_starts_from_the_constant_mean(name):
    G = _G()
    w = SETS[name]
    rng = np.random.default_rng(41)
    lens, sd = [40, 9, 17], 5
    m, v = _data(rng, lens, len(w) * sd, np.float64, False)
    gm, gvv = np.zeros(sd), np.full(sd, 0.05)
    off = _offsets(lens)
    y0 = G.mlpg_gv_batch(m, v, w, gm, gvv, lengths=lens, n_iter=0)
    y = G.mlpg_gv_batch(m, v, w, gm, gvv, lengths=lens, n_iter=N_ITER)
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        assert np.all(y0[a:b] == y0[a]), u  # every frame is the mean of c_m
        cm = ogv.mlpg(m[a:b], v[a:b], w)
        assert np.abs(y0[a] - cm.mean(axis=0)).max() <= 1e-12 * np.abs(cm).max()
        _check(y0[a:b], m[a:b], v[a:b], w, gm, gvv, 0)
        _check(y[a:b], m[a:b], v[a:b], w, gm, gvv, N_ITER)


@pytest.mark.parametrize("name,T", [("w0", 49), ("w0", 98), ("w0", 257), ("w2", 2), ("nw3_halfwidth3", 6),
                                    ("nw4", 8)])
def test_constant_cm_is_its_own_start_point(name, T):
    """Static means 0.75 under static variance 0.5, and T <= 2 m_edge where there are dynamic windows: c_m has
    one value (0.75 up to the solve's rounding) at every frame, v(c_m) == 0, and the start point is c_m itself.  At T = 49 and 98,
    (0.75 T) * (1 / T) is not 0.75: a mean taken that way leaves v(c_m) at an ulp squared."""
    G = _G()
    w = SETS[name]
    sd = 3
    rng = np.random.default_rng(T)
    m = rng.standard_normal((T, len(w) * sd))
    m[:, :sd] = 0.75
    v = np.full(len(w) * sd, 0.5)
    gm, gvv = np.full(sd, 2.0), np.full(sd, 0.1)
    for dtype in (np.float32, np.float64):
        md, vd = m.astype(dtype), v.astype(dtype)
        cm = ogv.mlpg(md, vd, w)
        assert ogv.variance(cm[:, 0]) == 0.0 and np.array_equal(ogv.mlpg_gv(md, vd, w, gm, gvv, n_iter=0), cm)
        y0 = G.mlpg_gv(md, vd, w, gm, gvv, n_iter=0)
        assert y0.dtype == dtype and np.all(y0 == y0[0]) and np.abs(y0 - 0.75).max() <= 2.0 ** -52, (dtype, y0)
        y = G.mlpg_gv(md, vd, w, gm, gvv)
        assert np.abs(y - ogv.mlpg_gv(md, vd, w, gm, gvv)).max() <= 1e-12, (dtype, y)


@pytest.mark.parametrize("name", ["nw3_halfwidth3", "nw4"])
def test_zero_iterations_on_instance_3(name):
    G = _G()
    w = SETS[name]
    lens, sd = [257, 17, 9], 5
    off = _offsets(lens)
    for dtype in (np.float32, np.float64):
        rng = np.random.default_rng(5 + (dtype == np.float32))
        m, v = _data(rng, lens, len(w) * sd, dtype, False)
        gm, gvv = _gv_params(rng, m, v, w, lens, sd)
        y = G.mlpg_gv_batch(m, v, w, gm, gvv, lengths=lens, n_iter=0)
        for u in range(len(lens)):
            a, b = off[u], off[u + 1]
            _check(y[a:b], m[a:b], v[a:b], w, gm, gvv, 0)


# ---- 2. solve mode (unit_variance_mlpg_matrix) on the wider instances -------------------------------------------
@pytest.mark.parametrize("name", ["nw2_halfwidth2", "nw3_halfwidth3", "nw4"])
def test_solve_mode_on_the_wider_instances(name, kernels):
    G = _G()
    w = SETS[name]
    _assert_only(kernels[("solve", name, 40)], kernel_name(name, np.float64, MODE_SOLVE))
    sd = 4
    for T in (1, 9, 40, 200):
        R = G.unit_variance_mlpg_matrix(w, T)
        assert R.dtype == np.float32 and R.shape == (T, len(w) * T)
        assert np.abs(R - oracle.unit_variance_mlpg_matrix(w, T)).max() < 2e-7, T
        # R @ reshape_means(mu) == mlpg(mu, ones)  (the reference's tests/test_paramgen.py)
        mu = np.random.default_rng(T).random((T, sd * len(w)))
        y = G.mlpg(mu, np.ones(sd * len(w)), w)
        assert np.allclose(R @ G.reshape_means(mu, sd), y, rtol=1e-5, atol=1e-6), T


# ---- 3. GV across workspace waves -------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("name", WAVE_SETS)
def test_gv_wave_split_is_bit_identical(name, dt, kernels, monkeypatch):
    import torch

    from nnmnkwii_b200 import _device as dev
    from nnmnkwii_b200 import _lib
    G = _G()
    w, dtype = SETS[name], DT[dt]
    m, v, lens, gm, gvv = _wave_batch(name, dtype)
    assert not np.all(np.diff(lens) <= 0) and not np.all(np.diff(lens) >= 0)
    n, sd = len(lens), m.shape[1] // len(w)
    Tmax = int(lens.max())
    pm = torch.zeros((n, Tmax, m.shape[1]), dtype=torch.float64 if dt == "f64" else torch.float32, device="cuda")
    pv = torch.ones_like(pm)
    off = _offsets(lens)
    for u, T in enumerate(lens):
        pm[u, :T] = torch.from_numpy(m[off[u]:off[u + 1]])
        pv[u, :T] = torch.from_numpy(v[off[u]:off[u + 1]])

    def run():
        c0 = _lib.launch_count()
        flat = G.mlpg_gv_batch(m, v, w, gm, gvv, lengths=lens, n_iter=N_ITER)
        c1 = _lib.launch_count()
        padded = G.mlpg_gv_batch(pm, pv, w, gm, gvv, lengths=lens, n_iter=N_ITER)
        c2 = _lib.launch_count()
        return flat, padded.cpu().numpy(), c1 - c0, c2 - c1

    flat1, pad1, nf, npd = run()
    assert (nf, npd) == (1, 1)
    for u, T in enumerate(lens):
        assert np.array_equal(pad1[u, :T], flat1[off[u]:off[u + 1]]) and not pad1[u, T:].any()
    kern = kernel_name(name, dtype, MODE_GV)
    _assert_only(kernels[("waves", name, dt, 0)], kern)
    assert len(kernels[("waves", name, dt, 0)]) == 1
    for k in WAVE_KS[1:]:
        waves = -(-n // k)
        monkeypatch.setattr(dev, "WORKSPACE_CAP_BYTES", gv_cap(lens, sd, w, k))
        flat2, pad2, nf, npd = run()
        assert (nf, npd) == (waves, waves), (k, nf, npd)
        names = kernels[("waves", name, dt, k)]
        _assert_only(names, kern)
        assert len(names) == waves, (k, names)
        assert np.array_equal(flat1, flat2) and np.array_equal(pad1, pad2), k
    for u in (0, 4, 7):  # and the split batch still matches the oracle
        a, b = off[u], off[u + 1]
        _check(flat2[a:b], m[a:b], v[a:b], w, gm, gvv, N_ITER)


@pytest.mark.parametrize("name", WAVE_SETS)
def test_gv_wave_split_reports_the_first_failure_in_reference_order(name, monkeypatch):
    """Longest-first waves of two: utterance 6 (35 frames) runs in the second wave, utterance 3 (20 frames) in
    the third.  Both fail; GV reports utterance 3, as the forward solve does under a cap of the same kind."""
    import torch

    from nnmnkwii_b200 import _device as dev
    from nnmnkwii_b200 import _lib
    from test_kernel_variants_mlpg_gpu import _cap_for
    G = _G()
    w = SETS[name]
    rng = np.random.default_rng(72)
    lens = np.array([50, 40, 30, 20, 10, 45, 35])
    sd = 4
    off = _offsets(lens)
    m = rng.random((int(lens.sum()), len(w) * sd))
    v = rng.random((int(lens.sum()), len(w) * sd)) + 0.1
    v[off[3]:off[4], 2] = -1.0  # utterance 3, chain 2
    v[off[6]:off[7], 0] = -1.0  # utterance 6, chain 0
    gm, gvv = np.full(sd, 0.1), np.full(sd, 0.01)
    for dt in (torch.float32, torch.float64):
        mt, vt = torch.from_numpy(m).to("cuda", dt), torch.from_numpy(v).to("cuda", dt)
        monkeypatch.setattr(dev, "WORKSPACE_CAP_BYTES", _cap_for(lens, G.StreamLayout.single(len(w) * sd, len(w)), w, 2))
        with pytest.raises(np.linalg.LinAlgError) as e_fwd:
            G.mlpg_batch(mt, vt, w, lengths=lens)
        monkeypatch.setattr(dev, "WORKSPACE_CAP_BYTES", gv_cap(lens, sd, w, 2))
        c0 = _lib.launch_count()
        with pytest.raises(np.linalg.LinAlgError) as e_gv:
            G.mlpg_gv_batch(mt, vt, w, gm, gvv, lengths=lens)
        assert _lib.launch_count() - c0 == 4
        assert str(e_gv.value) == str(e_fwd.value), (str(e_gv.value), str(e_fwd.value))
        assert "(utterance 3, chain 2)" in str(e_gv.value)


# ---- 4. padding, streams and the segment-moments grid -----------------------------------------------------------
def _padded(m, v, lens, fill_m, fill_v):
    import torch
    B, Tmax, D = len(lens), int(max(lens)), m.shape[1]
    pm = np.full((B, Tmax, D), fill_m, m.dtype)
    pv = np.full((B, Tmax, D), fill_v, v.dtype)
    off = _offsets(lens)
    for u, T in enumerate(lens):
        pm[u, :T], pv[u, :T] = m[off[u]:off[u + 1]], v[off[u]:off[u + 1]]
    return torch.from_numpy(pm).cuda(), torch.from_numpy(pv).cuda()


@pytest.mark.parametrize("name,dtype", [("w2", np.float32), ("nw4", np.float64)])
def test_gv_padding_rows_are_never_read(name, dtype):
    """Padding rows hold NaN means and -1 variances: read, they would poison or fail the solve."""
    import torch
    G = _G()
    w = SETS[name]
    rng = np.random.default_rng(77)
    lens, sd = [60, 3, 1, 121, 33, 9], 6
    m, v = _data(rng, lens, len(w) * sd, dtype, False)
    gm, gvv = _gv_params(rng, m, v, w, lens, sd)
    flat = G.mlpg_gv_batch(m, v, w, gm, gvv, lengths=lens)
    pm, pv = _padded(m, v, lens, np.nan, -1.0)
    y = G.mlpg_gv_batch(pm, pv, w, gm, gvv, lengths=lens)
    assert y.is_cuda and y.dtype == pm.dtype and y.shape == (len(lens), max(lens), sd)
    yh = y.cpu().numpy()
    off = _offsets(lens)
    for u, T in enumerate(lens):
        assert np.array_equal(yh[u, :T], flat[off[u]:off[u + 1]]), u
        assert np.all(yh[u, T:] == 0), u
    # the same call on a stream of its own
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ys = G.mlpg_gv_batch(pm, pv, w, gm, gvv, lengths=lens)
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(ys, y)


def _two_pass(x, lens):
    """Per-utterance population variance, float64, mean first and then the squared deviations."""
    x = np.asarray(x, np.float64)
    off = _offsets(lens)[:-1]
    mean = np.add.reduceat(x, off, axis=0) / np.asarray(lens)[:, None]
    dev = x - np.repeat(mean, lens, axis=0)
    return np.add.reduceat(dev * dev, off, axis=0) / np.asarray(lens)[:, None]


@pytest.mark.parametrize("D", [1, 31, 32, 33, 187, 513])
def test_global_variance_every_column_block(D):
    """Columns in blocks of 32; float32 frames offset by 1e4 (a one-pass sum of squares would lose about
    eight digits to cancellation); padded rows of NaN."""
    import torch
    G = _G()
    rng = np.random.default_rng(D)
    lens = [33, 1, 200, 7, 64]
    n = sum(lens)
    scale = 0.5 + 2.5 * rng.random(D)
    for dtype in (np.float32, np.float64):
        x = (rng.standard_normal((n, D)) * scale + 1e4).astype(dtype)
        ref = _two_pass(x, lens)
        bar = 1e-12 * np.abs(ref).max()
        got = G.global_variance(x, lengths=lens)
        assert got.dtype == np.float64 and got.shape == (len(lens), D)
        assert np.abs(got - ref).max() <= bar, (dtype, np.abs(got - ref).max() / np.abs(ref).max())
        assert np.all(got[1] == 0)  # one frame
        pad = np.full((len(lens), max(lens), D), np.nan, dtype)
        off = _offsets(lens)
        for u, T in enumerate(lens):
            pad[u, :T] = x[off[u]:off[u + 1]]
        pg = G.global_variance(torch.from_numpy(pad).cuda(), lengths=lens)
        assert pg.is_cuda and np.abs(pg.cpu().numpy() - ref).max() <= bar, dtype
        gm, gvv = G.gv_statistics(x, lengths=lens)
        assert np.abs(gm - ref.mean(axis=0)).max() <= bar
        assert np.abs(gvv - ref.var(axis=0)).max() <= 1e-12 * np.abs(ref.var(axis=0)).max()


def test_global_variance_of_more_utterances_than_one_grid(kernels):
    """65 537 utterances: grid.y holds 65 535, so the launcher makes a second launch from utterance 65 535."""
    from nnmnkwii_b200 import _lib
    G = _G()
    x, lens = _many_utterances()
    assert len(kernels[("moments",)]) == 2 and all("segment_moments_kernel<float>" in k for k in kernels[("moments",)])
    c0 = _lib.launch_count()
    got = G.global_variance(x, lengths=lens)
    assert _lib.launch_count() - c0 == 2
    ref = _two_pass(x, lens)
    assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
    assert rel_err(got[-2:], ref[-2:]) <= 1e-12 and np.all(ref[-2:] > 0)
