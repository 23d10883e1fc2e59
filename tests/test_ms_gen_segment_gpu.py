"""Parameter generation considering the segment-level modulation spectrum on the GPU
(paramgen.mlpg_ms_batch(segment=L), csrc/nnk_ms_gen.cu ms_gen_segment_kernel) against the float64 restatement
tests/ms_gen_segment_oracle.py.

* every `ms_gen_segment_kernel<LOGN, TRIAL>` instance (n = 32 .. 512), checked by kernel name; the launch count
  2 + 2 n_iter for different batches and lengths;
* float64 within 1e-9 (max abs over max abs) of the restatement for n_iter 1, 5 and 20, on every n with
  L = 4, n / 2 (rounded to even) and n and T = 1, 2, H - 1, H + 1 and 5000, a 20 000-frame utterance the
  utterance level refuses, window sets of half-width 0, 1, 2 and 4 and the Merlin layout with its copied
  column.  The device's accept decisions are read from calls with n_iter = 0 .. n_iter; every decision whose
  margin in the restatement is above 1e-9 must be the device's, and at a near-tie (F changes by less than
  rounding resolves, e.g. close to a fixed point late in n_iter = 20) the restatement follows the device.  Where
  the restatement's own result moves by more than 1e-9 / 30 when the means move by 1e-13 of their size
  (n_iter = 20 on 20 000 frames, L = 4 at n >= 128), the bar is 30 times that sensitivity;
* exact equalities: n_iter = 0 and all-inf ms_var give mlpg_batch's bits; padded, flat and per-utterance calls
  agree bit for bit; repeated calls too; float32 input gives the float64 result of the widened input, rounded;
* the objective never falls, and rises when the statistics are far from the trajectory's MS;
* a matrix that is not positive definite raises LinAlgError;
* baseline.gmm.MLPG(ms=..., ms_segment=L) is mlpg_ms_batch(segment=L) on its own E and D."""
import re

import numpy as np
import pytest

import ms_gen_segment_oracle as S
import oracle.gv as ogv
import oracle.ms_segment as oseg
import variant_mirror as M
from conftest import windows_set

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from nnmnkwii_b200 import paramgen as G  # noqa: E402

NS = (32, 64, 128, 256, 512)
FAMILY = r"\bms_gen_segment_kernel<"
STD = windows_set()[2]
WINDOWS = {0: windows_set()[0], 1: STD, 2: windows_set()[3],
           4: [(0, 0, np.array([1.0])), (4, 4, np.array([1.0, -2.0, 3.0, -4.0, 0.0, 4.0, -3.0, 2.0, -1.0]) / 20.0)]}
MARGIN = 1e-9
TOL = 1e-9


def _ls(n):
    return (4, max(4, (n // 2) & ~1), n)


def _data(rng, T, nw, sd):
    m = np.concatenate([np.cumsum(rng.standard_normal((T, sd)), 0) * 0.1,
                        0.05 * rng.standard_normal((T, (nw - 1) * sd))], 1)
    return m, rng.random((T, nw * sd)) + 0.5


def _stats(rng, n, sd, L, rough=0.3):
    """Segment-level statistics of rough trajectories: far from what MLPG gives, so the MS term pulls."""
    nat = rng.standard_normal((4, 4 * n, sd)) * rough + np.cumsum(rng.standard_normal((4, 4 * n, sd)), 1) * 0.05
    mean, var = oseg.statistics(list(nat), n, L)
    return mean, var + 0.5


def _err(y, ref):
    return np.abs(np.asarray(y, dtype=np.float64) - ref).max() / max(np.abs(ref).max(), 1e-300)


def _decisions(run, n_iter, chains):
    """Per chain (a list of row-index / column pairs), the accept decision the device took in each trial: trial i
    was accepted when the results of n_iter = i and i - 1 differ (``run(k)`` is the host result of n_iter = k;
    the first k trials of a call are the same whatever n_iter, only the last one skips the gradient)."""
    ys = [run(k) for k in range(n_iter + 1)]
    return [[not np.array_equal(ys[i][rows, col], ys[i - 1][rows, col]) for i in range(1, n_iter + 1)]
            for rows, col in chains]


def _oracle(m, v, w, mm, mv, L, n_iter, follow):
    """The restatement's result along the device's path: at every trial whose margin is below MARGIN (F changes
    by less than rounding resolves, e.g. close to a fixed point late in n_iter = 20) it takes the device's
    decision, which either way is valid; every other decision must be the device's."""
    traces = []
    ref = S.mlpg_ms(m, v, w, mm, mv, L, n_iter=n_iter, traces=traces, follow=follow)
    for d, tr in enumerate(traces):
        for i, (_, ok, margin) in enumerate(tr[1:]):
            # margin inf: the trial moves c by at most 1e-11 of its size, so its decision cannot be read back
            assert margin <= MARGIN or margin == np.inf or ok == follow[d][i], (d, i, margin)
    return ref


def _bar(m, v, w, mm, mv, L, n_iter, follow, ref):
    """TOL, or 30 times the restatement's own sensitivity where that is larger: the change of its result when
    the means move by 1e-13 of their size.  Twenty trials can amplify rounding: on 20 000 frames the step
    h / omega scales the gradient by 3 T, and L = 4 zero-padded to n >= 128 has near-null bins whose 1 / |Y|^2
    is huge (a 1e-13 perturbation moves the n = 512, L = 4, T = 5000 result by 2e-7)."""
    pert = S.mlpg_ms(m * (1 + 1e-13), v, w, mm, mv, L, n_iter=n_iter, follow=follow)
    return max(TOL, 30 * _err(pert, ref))


def _check(y, run, m, v, w, mm, mv, L, lens, n_iter):
    """Every utterance of a flat batch (single-stream layout) against the restatement."""
    off = np.concatenate([[0], np.cumsum(lens)])
    sd = y.shape[1]
    chains = [(slice(off[u], off[u + 1]), d) for u in range(len(lens)) for d in range(sd)]
    dec = _decisions(run, n_iter, chains)
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        follow = dec[u * sd:(u + 1) * sd]
        ref = _oracle(m[a:b], v[a:b], w, mm, mv, L, n_iter, follow)
        bar = _bar(m[a:b], v[a:b], w, mm, mv, L, n_iter, follow, ref)
        assert _err(y[a:b], ref) <= bar, (u, lens[u], bar)


# ---- 1. every instance, by name, and the launch count ------------------------------------------------------------
def launch(n):
    """One mlpg_ms call at DFT length n, L = n / 2, with two trials (in a child process, see `kernels`)."""
    rng = np.random.default_rng(n)
    m, v = _data(rng, 300, 3, 2)
    mm, mv = _stats(rng, n, 2, n // 2)
    G.mlpg_ms(torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda(), STD, mm, mv, n_iter=2, segment=n // 2)
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def kernels():
    cases = [([n], FAMILY) for n in NS]
    res = M.profiled_in_child("test_ms_gen_segment_gpu", "launch", cases, repeats=True)
    out = {}
    for (case, _), (names, err) in zip(cases, res):
        assert err == "None", (case, err)
        out[case[0]] = names
    return out


def test_every_instance_is_launched_by_name(kernels):
    seen = set()
    for n, names in kernels.items():
        got = [re.search(r"ms_gen_segment_kernel<[^>]*>", s).group(0) for s in names]
        logn = n.bit_length() - 1
        assert got == (["ms_gen_segment_kernel<%d, false>" % logn] +
                       ["ms_gen_segment_kernel<%d, true>" % logn] * 2), (n, names)
        seen.update(got)
    assert len(seen) == 10


def test_launch_count_does_not_depend_on_the_batch():
    from nnmnkwii_b200 import _lib
    rng = np.random.default_rng(3)
    mm, mv = _stats(rng, 64, 2, 50)
    counts = []
    for lens in ([40], [512, 1, 3000, 77], [20000]):
        m, v = _data(rng, int(sum(lens)), 3, 2)
        n0 = _lib.launch_count()
        G.mlpg_ms_batch(torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda(), STD, mm, mv, lengths=lens, n_iter=7,
                        segment=50)
        counts.append(_lib.launch_count() - n0)
    assert counts == [2 + 2 * 7] * 3, counts


# ---- 2. against the restatement ----------------------------------------------------------------------------------
@pytest.mark.parametrize("n_iter", [1, 5, 20])
@pytest.mark.parametrize("n", NS)
def test_every_n_segment_and_edge_length_matches_oracle(n, n_iter):
    for L in _ls(n):
        H = L // 2
        lens = sorted({1, 2, max(H - 1, 1), H + 1}) + [5000]
        rng = np.random.default_rng([n, L, n_iter])
        m, v = _data(rng, sum(lens), 3, 1)
        mm, mv = _stats(rng, n, 1, L)

        def run(k):
            return G.mlpg_ms_batch(m, v, STD, mm, mv, lengths=lens, n_iter=k, segment=L)
        _check(run(n_iter), run, m, v, STD, mm, mv, L, lens, n_iter)


@pytest.mark.parametrize("n_iter", [1, 5, 20])
def test_a_long_utterance_the_utterance_level_refuses(n_iter):
    rng = np.random.default_rng([20000, n_iter])
    m, v = _data(rng, 20000, 3, 2)
    mm, mv = _stats(rng, 64, 2, 50)
    md, vd = torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda()

    def run(k):
        return G.mlpg_ms_batch(md, vd, STD, mm, mv, lengths=[20000], n_iter=k, segment=50).cpu().numpy()
    _check(run(n_iter), run, m, v, STD, mm, mv, 50, [20000], n_iter)


@pytest.mark.parametrize("n_iter", [1, 5, 20])
@pytest.mark.parametrize("hw", sorted(WINDOWS))
def test_window_sets_match_oracle(hw, n_iter):
    w = WINDOWS[hw]
    sd, n, L = 2, 64, 4
    lens = [1, 2, 9, 300]
    rng = np.random.default_rng([hw, n_iter, 7])
    m, v = _data(rng, sum(lens), len(w), sd)
    mm, mv = _stats(rng, n, sd, L)
    md, vd = torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda()

    def run(k):
        return G.mlpg_ms_batch(md, vd, w, mm, mv, lengths=lens, n_iter=k, segment=L).cpu().numpy()
    _check(run(n_iter), run, m, v, w, mm, mv, L, lens, n_iter)


@pytest.mark.parametrize("n_iter", [1, 5, 20])
def test_merlin_layout_with_a_copied_column(n_iter):
    rng = np.random.default_rng([63, n_iter])
    layout = G.merlin_layout()
    n, L, lens = 64, 50, [600, 333, 2]
    T = sum(lens)
    m = rng.standard_normal((T, 187)) * 0.05
    m[:, :60] += np.cumsum(rng.standard_normal((T, 60)), 0) * 0.1
    m[:, 183] = rng.random(T) > 0.5
    v = rng.random((T, 187)) + 0.5
    mm, mv = _stats(rng, n, 63, L)
    mm[:, 61], mv[:, 61] = np.nan, np.nan  # the copied column's statistics are never read
    mv[:, 0] = np.inf                       # the power coefficient left alone

    def run(k):
        return G.mlpg_ms_batch(m, v, STD, mm, mv, lengths=lens, layout=layout, n_iter=k, segment=L)
    y = run(n_iter)
    off = np.concatenate([[0], np.cumsum(lens)])
    groups = (((0, 60), (0, 180)), ((60, 61), (180, 183)), ((62, 63), (184, 187)))
    chains = [(slice(off[u], off[u + 1]), c) for u in range(len(lens)) for c in (*range(61), 62)]
    dec = dict(zip([(u, c) for u in range(len(lens)) for c in (*range(61), 62)], _decisions(run, n_iter, chains)))
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        assert np.array_equal(y[a:b, 61], m[a:b, 183])
        for cols, ins in groups:
            args = (m[a:b, ins[0]:ins[1]], v[a:b, ins[0]:ins[1]], STD, mm[:, cols[0]:cols[1]], mv[:, cols[0]:cols[1]],
                    L, n_iter, [dec[(u, c)] for c in range(*cols)])
            ref = _oracle(*args)
            bar = _bar(*args, ref)
            assert _err(y[a:b, cols[0]:cols[1]], ref) <= bar, (u, cols, bar)


# ---- 3. exact equalities -----------------------------------------------------------------------------------------
def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_no_trial_and_exempt_bins_give_mlpg_bits():
    rng = np.random.default_rng(11)
    lens = [3000, 1, 512]
    m, v = _data(rng, sum(lens), 3, 4)
    mm, mv = _stats(rng, 128, 4, 100)
    for vg in (False, True):
        vv = _cuda(v[0] if vg else v)
        want = G.mlpg_batch(_cuda(m), vv, STD, lengths=lens)
        assert torch.equal(G.mlpg_ms_batch(_cuda(m), vv, STD, mm, mv, lengths=lens, n_iter=0, segment=100), want)
        inf = np.full_like(mv, np.inf)
        assert torch.equal(G.mlpg_ms_batch(_cuda(m), vv, STD, mm, inf, lengths=lens, n_iter=5, segment=100), want)


def test_padded_flat_and_per_utterance_agree_bit_for_bit():
    rng = np.random.default_rng(12)
    lens = np.array([700, 1, 0, 6000, 33])
    m, v = _data(rng, int(lens.sum()), 3, 5)
    mm, mv = _stats(rng, 64, 5, 50)
    flat = G.mlpg_ms_batch(_cuda(m), _cuda(v), STD, mm, mv, lengths=lens, n_iter=6, segment=50)
    off = np.concatenate([[0], np.cumsum(lens)])
    Tmax = int(lens.max()) + 3
    pm = torch.full((len(lens), Tmax, 15), float("nan"), dtype=torch.float64, device="cuda")
    pv = torch.full((len(lens), Tmax, 15), float("nan"), dtype=torch.float64, device="cuda")
    for b in range(len(lens)):
        pm[b, :lens[b]], pv[b, :lens[b]] = _cuda(m[off[b]:off[b + 1]]), _cuda(v[off[b]:off[b + 1]])
    padded = G.mlpg_ms_batch(pm, pv, STD, mm, mv, lengths=lens, n_iter=6, segment=50)
    for b in range(len(lens)):
        one = G.mlpg_ms(_cuda(m[off[b]:off[b + 1]]), _cuda(v[off[b]:off[b + 1]]), STD, mm, mv, n_iter=6, segment=50)
        assert torch.equal(flat[off[b]:off[b + 1]], one), b
        assert torch.equal(padded[b, :lens[b]], one) and not padded[b, lens[b]:].any(), b
    for _ in range(3):
        assert torch.equal(G.mlpg_ms_batch(_cuda(m), _cuda(v), STD, mm, mv, lengths=lens, n_iter=6, segment=50), flat)


def test_float32_is_the_widened_float64_result_rounded():
    rng = np.random.default_rng(13)
    lens = [4000, 256]
    m, v = _data(rng, sum(lens), 3, 3)
    m32, v32 = m.astype(np.float32), v.astype(np.float32)
    mm, mv = _stats(rng, 64, 3, 50)
    y64 = G.mlpg_ms_batch(m32.astype(np.float64), v32.astype(np.float64), STD, mm, mv, lengths=lens, segment=50)
    y32 = G.mlpg_ms_batch(m32, v32, STD, mm, mv, lengths=lens, segment=50)
    assert y32.dtype == np.float32 and np.array_equal(y32, y64.astype(np.float32))
    t32 = G.mlpg_ms_batch(_cuda(m32), _cuda(v32), STD, mm, mv, lengths=lens, segment=50)
    assert t32.dtype == torch.float32 and np.array_equal(t32.cpu().numpy(), y32)


# ---- 4. the objective --------------------------------------------------------------------------------------------
def test_objective_never_falls_and_rises_when_the_ms_is_far():
    rng = np.random.default_rng(14)
    T, sd, n, L = 3000, 3, 64, 50
    m, v = _data(rng, T, 3, sd)
    cm = G.mlpg_batch(m, v, STD, lengths=[T])
    assert _err(cm, ogv.mlpg(m, v, STD)) <= 1e-12
    for rough, strict in ((0.3, True), (0.0, False)):
        mm, mv = _stats(rng, n, sd, L, rough)
        y = G.mlpg_ms(m, v, STD, mm, mv, segment=L)
        for d in range(sd):
            f0 = S.chain_objective(m, v, STD, d, cm[:, d], mm[:, d], mv[:, d], L)
            f = S.chain_objective(m, v, STD, d, y[:, d], mm[:, d], mv[:, d], L)
            assert f >= f0 - 1e-12 * abs(f0), (rough, d, f, f0)
            if strict:
                assert f > f0 + 1e-3 * abs(f0), (d, f, f0)


# ---- 5. a singular system ----------------------------------------------------------------------------------------
def test_not_positive_definite_raises():
    m, v = _data(np.random.default_rng(16), 5000, 3, 2)
    v[2000, 0::2] = -1.0  # every window of static dimension 0
    mm, mv = _stats(np.random.default_rng(17), 64, 2, 50)
    with pytest.raises(np.linalg.LinAlgError):
        G.mlpg_ms(m, v, STD, mm, mv, n_iter=2, segment=50)


# ---- 6. baseline.gmm.MLPG(ms=..., ms_segment=L) ------------------------------------------------------------------
def test_gmm_mlpg_with_ms_segment_is_mlpg_ms_on_its_e_and_d():
    from sklearn.mixture import GaussianMixture

    from nnmnkwii_b200.baseline.gmm import MLPG
    w = windows_set()[1]
    rng = np.random.default_rng(18)
    sd = 3
    src = np.cumsum(rng.standard_normal((6000, 2 * sd)), axis=0) * 0.1
    tgt = src * 0.8 + rng.standard_normal((6000, 2 * sd)) * 0.1
    gmm = GaussianMixture(n_components=4, covariance_type="full", random_state=0).fit(np.hstack([src, tgt]))
    mm, mv = _stats(rng, 64, sd, 50)
    model = MLPG(gmm, windows=w, ms=(mm, mv), ms_segment=50)
    utts = [src[:80], src[80:5200], src[5200:5203]]
    batch = model.transform_batch(utts)
    for u, s in enumerate(utts):
        x, c = model._to_device(s)
        E, Dv = model._means_vars(x, c)
        want = G.mlpg_ms_batch(E, Dv, w, mm, mv, lengths=[len(s)], segment=50).cpu().numpy()
        y = model.transform(s)
        assert np.array_equal(y, want) and np.array_equal(batch[u], y), u
