"""Every DTW kernel and instance `nnk_dtw_align` can select, against the oracle, bit for bit.

Exact mode: the fused kernel for 8 <= D < 40 while the padded Y series fits the opt-in shared memory
(`dtw_fused_kernel<T, D/8>`), otherwise the two-pass path (`dtw_cost_kernel` + `dtw_dp_kernel<MC>`,
MC = 4 / 8 / 16 for Tx up to 1024 / 2048 / 4096), in chunks of at most 2 GiB of cost matrices, and a clean
NotImplementedError beyond 4096 frames.  FastDTW: one kernel, whose back-pointers spill to global memory
when a level's window exceeds the shared-memory budget, and whose wavefront takes a slower loop when more
than FD_MAXW rows are active on one anti-diagonal.  Shapes come from `variant_mirror`; paths, distances
and cell counts must equal `oracle.fastdtw` exactly, for both cost kinds."""
import numpy as np
import pytest

import oracle
import variant_mirror as M

pytestmark = pytest.mark.gpu

KINDS = ((0, "euclid"), (1, "melcd"))
DTW_KERNELS = r"\b(dtw_fused|dtw_cost|dtw_dp|fastdtw)_kernel\b"


def _series(T, D, seed, dtype=np.float32):
    r = np.random.default_rng(seed)
    return (np.cumsum(r.standard_normal((T, D)), 0) * 0.3).astype(dtype)


def _pad(seqs, T, dtype):
    out = np.zeros((len(seqs), T, seqs[0].shape[1]), dtype=dtype)
    for i, s in enumerate(seqs):
        out[i, :len(s)] = s
    return out


def _align(X, Y, kind, radius):
    import torch
    from nnmnkwii_b200.preprocessing import alignment as A

    def run():
        res = A._align_batch(torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda(), kind, radius)
        return tuple(t.cpu().numpy() for t in (res.path_i, res.path_j, res.path_len, res.dist, res.cells))

    out, err, names = M.profiled(run)
    assert err is None, err
    return out, M.launched(names, DTW_KERNELS)


def _check(out, xs, ys, kname, radius, pairs=None):
    pi, pj, L, d, cells = out
    for n in range(len(xs)) if pairs is None else pairs:
        d0, oi, oj, c0 = oracle.fastdtw(xs[n], ys[n], radius=radius, kind=kname)
        assert L[n] == len(oi), (n, radius, kname)
        assert np.array_equal(pi[n, :L[n]], oi) and np.array_equal(pj[n, :L[n]], oj), (n, radius, kname)
        assert d[n] == d0 and cells[n] == c0, (n, radius, kname)


def _pairs(lx, ly, D, dtype, seed):
    xs = [_series(int(t), D, seed + i, dtype) for i, t in enumerate(lx)]
    ys = [_series(int(t), D, seed + 500 + i, dtype) for i, t in enumerate(ly)]
    return xs, ys


# ---- exact: fused ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [8, 15, 16, 23, 32, 39])
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
def test_exact_fused_instances(D, dt):
    ms = M.max_smem_optin()
    Tx, Ty = 125, 121
    assert M.dtw_fused_ok(Tx, Ty, D, ms)
    xs, ys = _pairs([1, 37, 120, 64, 2, 125], [121, 1, 99, 64, 3, 118], D, dt, 40 + D)
    X, Y = _pad(xs, Tx, dt), _pad(ys, Ty, dt)
    tname = "float" if dt == np.float32 else "double"
    for kind, kname in KINDS:
        out, kern = _align(X, Y, kind, -1)
        assert len(kern) == 1 and "dtw_fused_kernel<%s, %d>" % (tname, D // 8) in kern[0], kern
        _check(out, xs, ys, kname, -1)


# ---- exact: two-pass ---------------------------------------------------------------------------------------
def _assert_two_pass(kern, D, mc, n_chunks=1, tname="float"):
    cost = M.launched(kern, r"dtw_cost_kernel<%s, %d>" % (tname, D // 8 if 8 <= D < 40 else 0))
    dp = M.launched(kern, r"dtw_dp_kernel<%d>" % mc)
    assert len(cost) == n_chunks and len(dp) == n_chunks and len(kern) == 2 * n_chunks, kern


@pytest.mark.parametrize("D", [12, 25])
def test_exact_fused_limit_in_y(D):
    """Padded Ty at the fused kernel's shared-memory limit runs fused; one frame more runs two-pass.
    (At D = 12 and Tx = 300, Ty = 1919 asks for 232 440 bytes: within the H100's 232 448-byte opt-in, but
    not once the kernel's 16 static bytes are counted.  The launcher used to pick the fused kernel there
    and fail in cudaFuncSetAttribute.)"""
    ms = M.max_smem_optin()
    Tx = 300
    ty_lim = M.dtw_fused_ty_limit(Tx, D, ms)
    assert M.dtw_fused_ok(Tx, ty_lim, D, ms) and not M.dtw_fused_ok(Tx, ty_lim + 1, D, ms)
    for Ty, fused in ((ty_lim, True), (ty_lim + 1, False)):
        xs, ys = _pairs([Tx, 211, 5], [Ty, Ty - 300, 777], D, np.float32, 7 * D)
        X, Y = _pad(xs, Tx, np.float32), _pad(ys, Ty, np.float32)
        for kind, kname in KINDS:
            out, kern = _align(X, Y, kind, -1)
            if fused:
                assert len(kern) == 1 and "dtw_fused_kernel<float, %d>" % (D // 8) in kern[0], kern
            else:
                _assert_two_pass(kern, D, M.dtw_dp_bucket(Tx))
            _check(out, xs, ys, kname, -1)


@pytest.mark.parametrize("D", [3, 40, 64, 130])
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
def test_exact_two_pass_outside_the_fused_range(D, dt):
    """D = 130 takes pairwise_sumsq's split of frames wider than 128 dims."""
    ms = M.max_smem_optin()
    Tx, Ty = 130, 140
    assert not M.dtw_fused_ok(Tx, Ty, D, ms)
    xs, ys = _pairs([1, 130, 77, 20], [140, 1, 90, 133], D, dt, 90 + D)
    X, Y = _pad(xs, Tx, dt), _pad(ys, Ty, dt)
    for kind, kname in KINDS:
        out, kern = _align(X, Y, kind, -1)
        _assert_two_pass(kern, D, 4, tname="float" if dt == np.float32 else "double")
        _check(out, xs, ys, kname, -1)


@pytest.mark.parametrize("Tx", [1024, 1025, 2048, 2049, 4096])
def test_exact_two_pass_row_buckets(Tx):
    """Each `dtw_dp_kernel<MC>` bucket, with the bucket edges on both sides."""
    D, Ty = 3, 150
    mc = M.dtw_dp_bucket(Tx)
    assert mc == {1024: 4, 1025: 8, 2048: 8, 2049: 16, 4096: 16}[Tx]
    xs, ys = _pairs([Tx, Tx - 400], [Ty, 61], D, np.float32, Tx)
    X, Y = _pad(xs, Tx, np.float32), _pad(ys, Ty, np.float32)
    for kind, kname in KINDS:
        out, kern = _align(X, Y, kind, -1)
        _assert_two_pass(kern, D, mc)
        _check(out, xs, ys, kname, -1)


def test_exact_two_pass_in_two_chunks():
    """One pair more than fit 2 GiB of cost matrices: two chunks.  Pairs run longest first, so the chunk
    boundary falls between order[chunk - 1] and order[chunk]; both are checked against the oracle."""
    D, T = 3, 2048
    ch = M.dtw_exact_chunk(10 ** 6, T, T)
    n = ch + 1
    lx = T - np.arange(n)  # distinct lengths: the longest-first order is unambiguous
    ly = np.full(n, T)
    xs, ys = _pairs(lx, ly, D, np.float32, 3)
    X, Y = _pad(xs, T, np.float32), _pad(ys, T, np.float32)
    order = np.argsort(-(lx * ly), kind="stable")
    out, kern = _align(X, Y, 1, -1)
    _assert_two_pass(kern, D, M.dtw_dp_bucket(T), n_chunks=2)
    _check(out, xs, ys, "melcd", -1, pairs=[order[0], order[ch - 1], order[ch]])


def test_exact_beyond_4096_frames_raises_before_any_dtw_kernel():
    D = 3
    xs, ys = _pairs([4097], [50], D, np.float32, 11)
    X, Y = _pad(xs, 4097, np.float32), _pad(ys, 50, np.float32)
    import torch
    from nnmnkwii_b200.preprocessing import alignment as A
    _, err, names = M.profiled(lambda: A._align_batch(torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda(), 1, -1))
    assert isinstance(err, NotImplementedError) and "4096" in str(err), err
    assert not M.launched(names, DTW_KERNELS), names


# ---- FastDTW -----------------------------------------------------------------------------------------------
def _fastdtw_case(lx, ly, D, radius, seed):
    xs, ys = _pairs(lx, ly, D, np.float32, seed)
    Tx, Ty = max(lx), max(ly)
    X, Y = _pad(xs, Tx, np.float32), _pad(ys, Ty, np.float32)
    levels = [M.fastdtw_levels(x.astype(np.float64), y.astype(np.float64), radius, "melcd") for x, y in zip(xs, ys)]
    for kind, kname in KINDS:
        out, kern = _align(X, Y, kind, radius)
        assert kern and all("fastdtw_kernel" in k for k in kern), kern
        _check(out, xs, ys, kname, radius)
        if kname == "melcd":  # the mirror's windows are the kernel's: same cell count
            assert [sum(c for c, _ in lv) for lv in levels] == list(out[4]), (levels, out[4])
    return levels, M.fastdtw_caps(Tx, Ty, radius, M.max_smem_optin())


@pytest.mark.parametrize("D", [5, 25, 40, 130])
@pytest.mark.parametrize("radius", [3, 10, 30, 60])
def test_fastdtw_radius(radius, D):
    """Radius 3 keeps every level within FD_MAXW = 24 rows per anti-diagonal (about 2r + 8 rows): the
    lane-per-row wavefront.  Radius 10 and up widens the windows (about 4r + 2 rows) past it: the
    loop-over-cells wavefront.  D = 25 uses the batched cost loads (8 <= D <= 32), 5, 40 and 130 do not;
    130 takes pairwise_sumsq's split of frames wider than 128 dims."""
    levels, (bp_cap, cost_cap) = _fastdtw_case([700, 523, 9], [690, 700, 64], D, radius, 17 * radius + D)
    widest = max(w for lv in levels for _, w in lv)
    if radius == 3:
        assert widest <= M.FD_MAXW, widest
    else:
        assert widest > M.FD_MAXW, widest


@pytest.mark.parametrize("T,radius", [(3000, 1), (2000, 4)])
def test_fastdtw_back_pointers_in_global_memory(T, radius):
    """Long series: the shared-memory back-pointer budget is cut to keep four CTAs per SM, and the finest
    level's window exceeds it, so its back-pointers go to global scratch (`bp_in_smem == false`); the
    partner, radius 3 at 700 frames in test_fastdtw_radius, keeps every level in shared memory."""
    levels, (bp_cap, _) = _fastdtw_case([T, T - 211], [T - 57, T], 25, radius, T + radius)
    assert all(lv[0][0] > bp_cap for lv in levels), (levels, bp_cap)
    assert all(w <= M.FD_MAXW for lv in levels for _, w in lv)


def test_fastdtw_back_pointers_in_shared_memory():
    levels, (bp_cap, _) = _fastdtw_case([700, 523], [690, 700], 25, 3, 5)
    assert all(c <= bp_cap for lv in levels for c, _ in lv), (levels, bp_cap)
