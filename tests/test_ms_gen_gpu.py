"""Parameter generation considering the modulation spectrum on the GPU (paramgen.mlpg_ms / mlpg_ms_batch,
csrc/nnk_ms_gen.cu) against the float64 restatement oracle/ms_gen.py.

* every `ms_gen_kernel<LOGN, TRIAL>` instance (n = 256 .. 4096), checked by kernel name and launch count;
* float64 within 1e-9 (max abs over max abs) of the restatement for n_iter 1, 5 and 20, on every n with
  T = 1, 2, n - 1 and n, on window sets of half-width 0, 1, 2 and 4 and on the Merlin layout with its copied
  column.  The restatement reports the margin of every accept decision; the tests assert that each one is
  clear of rounding, so the bar is well posed;
* exact equalities: n_iter = 0 and all-inf ms_var give mlpg_batch's bits; padded, flat and per-utterance calls
  agree bit for bit; repeated calls too; float32 input gives the float64 result of the widened input, rounded;
* the objective never falls below F(c_m), and rises when the MS is far from the statistics;
* a matrix that is not positive definite raises LinAlgError, as for mlpg_batch;
* baseline.gmm.MLPG(ms=...) is mlpg_ms_batch on its own E and D."""
import re

import numpy as np
import pytest

import oracle.gv as ogv
import oracle.ms_gen as O
import variant_mirror as M
from conftest import windows_set

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from nnmnkwii_b200 import paramgen as G  # noqa: E402

NS = (256, 512, 1024, 2048, 4096)
FAMILY = r"\bms_gen_kernel<"
STD = windows_set()[2]
# window sets by half-width; half-width 4 is the widest the MLPG kernels take
WINDOWS = {0: windows_set()[0], 1: STD, 2: windows_set()[3],
           4: [(0, 0, np.array([1.0])), (4, 4, np.array([1.0, -2.0, 3.0, -4.0, 0.0, 4.0, -3.0, 2.0, -1.0]) / 20.0)]}
MARGIN = 1e-9  # an accept decision whose relative margin is below this could flip under rounding
TOL = 1e-9


def _data(rng, T, nw, sd):
    """Means (T, nw sd) whose static part is a smooth walk, per-frame variances."""
    m = np.concatenate([np.cumsum(rng.standard_normal((T, sd)), 0) * 0.1,
                        0.05 * rng.standard_normal((T, (nw - 1) * sd))], 1)
    return m, rng.random((T, nw * sd)) + 0.5


def _stats(rng, n, sd, rough=0.3):
    """MS statistics of rough trajectories: far from what MLPG gives, so the MS term pulls."""
    nat = rng.standard_normal((8, n, sd)) * rough + np.cumsum(rng.standard_normal((8, n, sd)), 1) * 0.05
    s = np.log(np.maximum(np.abs(np.fft.rfft(nat, n, axis=1)) ** 2, O.TINY))
    return s.mean(0), s.var(0) + 0.5


def _err(y, ref):
    return np.abs(np.asarray(y, dtype=np.float64) - ref).max() / max(np.abs(ref).max(), 1e-300)


def _oracle(m, v, w, mm, mv, n_iter, **kw):
    traces = []
    ref = O.mlpg_ms(m, v, w, mm, mv, n_iter=n_iter, traces=traces, **kw)
    worst = min(t[2] for tr in traces for t in tr)
    assert worst > MARGIN, worst  # the seed gives clear accept decisions
    return ref


# ---- 1. every instance, by name, and the launch count ------------------------------------------------------------
def launch(n):
    """One mlpg_ms call at DFT length n with two trials (in a child process, see `kernels`)."""
    rng = np.random.default_rng(n)
    m, v = _data(rng, 40, 3, 2)
    mm, mv = _stats(rng, n, 2)
    G.mlpg_ms(torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda(), STD, mm, mv, n_iter=2)
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def kernels():
    cases = [([n], FAMILY) for n in NS]
    res = M.profiled_in_child("test_ms_gen_gpu", "launch", cases, repeats=True)
    out = {}
    for (case, _), (names, err) in zip(cases, res):
        assert err == "None", (case, err)
        out[case[0]] = names
    return out


def test_every_instance_is_launched_by_name(kernels):
    seen = set()
    for n, names in kernels.items():
        got = [re.search(r"ms_gen_kernel<[^>]*>", s).group(0) for s in names]
        logn = n.bit_length() - 1
        assert got == ["ms_gen_kernel<%d, false>" % logn] + ["ms_gen_kernel<%d, true>" % logn] * 2, (n, names)
        seen.update(got)
    assert len(seen) == 10


def test_launch_count_does_not_depend_on_the_batch():
    from nnmnkwii_b200 import _lib
    rng = np.random.default_rng(3)
    mm, mv = _stats(rng, 512, 2)
    counts = []
    for lens in ([40], [512, 1, 300, 77]):
        m, v = _data(rng, int(sum(lens)), 3, 2)
        n0 = _lib.launch_count()
        G.mlpg_ms_batch(torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda(), STD, mm, mv, lengths=lens, n_iter=7)
        counts.append(_lib.launch_count() - n0)
    assert counts == [2 + 2 * 7] * 2, counts


# ---- 2. against the restatement ----------------------------------------------------------------------------------
@pytest.mark.parametrize("n_iter", [1, 5, 20])
@pytest.mark.parametrize("n", NS)
def test_every_n_and_edge_length_matches_oracle(n, n_iter):
    rng = np.random.default_rng([n, n_iter])
    sd = 2
    lens = [1, 2, n - 1, n]
    m, v = _data(rng, sum(lens), 3, sd)
    mm, mv = _stats(rng, n, sd)
    y = G.mlpg_ms_batch(m, v, STD, mm, mv, lengths=lens, n_iter=n_iter)
    off = np.concatenate([[0], np.cumsum(lens)])
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        assert _err(y[a:b], _oracle(m[a:b], v[a:b], STD, mm, mv, n_iter)) <= TOL, (u, lens[u])


@pytest.mark.parametrize("n_iter", [1, 5, 20])
@pytest.mark.parametrize("hw", sorted(WINDOWS))
def test_window_sets_match_oracle(hw, n_iter):
    w = WINDOWS[hw]
    rng = np.random.default_rng([hw, n_iter, 7])
    sd, n = 3, 256
    lens = [1, 2, 9, 255, 256]
    m, v = _data(rng, sum(lens), len(w), sd)
    mm, mv = _stats(rng, n, sd)
    y = G.mlpg_ms_batch(torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda(), w, mm, mv, lengths=lens,
                        n_iter=n_iter).cpu().numpy()
    off = np.concatenate([[0], np.cumsum(lens)])
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        assert _err(y[a:b], _oracle(m[a:b], v[a:b], w, mm, mv, n_iter)) <= TOL, (u, lens[u])


@pytest.mark.parametrize("n_iter", [1, 5, 20])
def test_merlin_layout_with_a_copied_column(n_iter):
    rng = np.random.default_rng([63, n_iter])
    layout = G.merlin_layout()
    n, lens = 1024, [600, 333, 2]
    T = sum(lens)
    m = rng.standard_normal((T, 187)) * 0.05
    m[:, :60] += np.cumsum(rng.standard_normal((T, 60)), 0) * 0.1
    m[:, 183] = rng.random(T) > 0.5
    v = rng.random((T, 187)) + 0.5
    mm, mv = _stats(rng, n, 63)
    mm[:, 61], mv[:, 61] = np.nan, np.nan  # the copied column's statistics are never read
    mv[:, 0] = np.inf                       # the power coefficient left alone
    y = G.mlpg_ms_batch(m, v, STD, mm, mv, lengths=lens, layout=layout, n_iter=n_iter)
    off = np.concatenate([[0], np.cumsum(lens)])
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        assert np.array_equal(y[a:b, 61], m[a:b, 183])
        for cols, ins in (((0, 60), (0, 180)), ((60, 61), (180, 183)), ((62, 63), (184, 187))):
            ref = _oracle(m[a:b, ins[0]:ins[1]], v[a:b, ins[0]:ins[1]], STD, mm[:, cols[0]:cols[1]],
                          mv[:, cols[0]:cols[1]], n_iter)
            assert _err(y[a:b, cols[0]:cols[1]], ref) <= TOL, (u, cols)


# ---- 3. exact equalities -----------------------------------------------------------------------------------------
def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_no_trial_and_exempt_bins_give_mlpg_bits():
    rng = np.random.default_rng(11)
    lens = [300, 1, 512]
    m, v = _data(rng, sum(lens), 3, 4)
    mm, mv = _stats(rng, 512, 4)
    for vg in (False, True):
        vv = _cuda(v[0] if vg else v)
        want = G.mlpg_batch(_cuda(m), vv, STD, lengths=lens)
        assert torch.equal(G.mlpg_ms_batch(_cuda(m), vv, STD, mm, mv, lengths=lens, n_iter=0), want)
        inf = np.full_like(mv, np.inf)
        assert torch.equal(G.mlpg_ms_batch(_cuda(m), vv, STD, mm, inf, lengths=lens, n_iter=5), want)


def test_padded_flat_and_per_utterance_agree_bit_for_bit():
    rng = np.random.default_rng(12)
    lens = np.array([700, 1, 0, 1024, 33])
    m, v = _data(rng, int(lens.sum()), 3, 5)
    mm, mv = _stats(rng, 1024, 5)
    flat = G.mlpg_ms_batch(_cuda(m), _cuda(v), STD, mm, mv, lengths=lens, n_iter=6)
    off = np.concatenate([[0], np.cumsum(lens)])
    Tmax = int(lens.max()) + 3
    pm = torch.full((len(lens), Tmax, 15), float("nan"), dtype=torch.float64, device="cuda")
    pv = torch.full((len(lens), Tmax, 15), float("nan"), dtype=torch.float64, device="cuda")
    for b in range(len(lens)):
        pm[b, :lens[b]], pv[b, :lens[b]] = _cuda(m[off[b]:off[b + 1]]), _cuda(v[off[b]:off[b + 1]])
    padded = G.mlpg_ms_batch(pm, pv, STD, mm, mv, lengths=lens, n_iter=6)
    for b in range(len(lens)):
        one = G.mlpg_ms(_cuda(m[off[b]:off[b + 1]]), _cuda(v[off[b]:off[b + 1]]), STD, mm, mv, n_iter=6)
        assert torch.equal(flat[off[b]:off[b + 1]], one), b
        assert torch.equal(padded[b, :lens[b]], one) and not padded[b, lens[b]:].any(), b
    for _ in range(3):
        assert torch.equal(G.mlpg_ms_batch(_cuda(m), _cuda(v), STD, mm, mv, lengths=lens, n_iter=6), flat)


def test_float32_is_the_widened_float64_result_rounded():
    rng = np.random.default_rng(13)
    lens = [400, 256]
    m, v = _data(rng, sum(lens), 3, 3)
    m32, v32 = m.astype(np.float32), v.astype(np.float32)
    mm, mv = _stats(rng, 512, 3)
    y64 = G.mlpg_ms_batch(m32.astype(np.float64), v32.astype(np.float64), STD, mm, mv, lengths=lens)
    y32 = G.mlpg_ms_batch(m32, v32, STD, mm, mv, lengths=lens)
    assert y32.dtype == np.float32 and np.array_equal(y32, y64.astype(np.float32))
    t32 = G.mlpg_ms_batch(_cuda(m32), _cuda(v32), STD, mm, mv, lengths=lens)
    assert t32.dtype == torch.float32 and np.array_equal(t32.cpu().numpy(), y32)


# ---- 4. the objective --------------------------------------------------------------------------------------------
def test_objective_never_falls_and_rises_when_the_ms_is_far():
    rng = np.random.default_rng(14)
    T, sd, n = 500, 4, 512
    m, v = _data(rng, T, 3, sd)
    cm = G.mlpg_batch(m, v, STD, lengths=[T])  # the device's own start point
    assert _err(cm, ogv.mlpg(m, v, STD)) <= 1e-12
    for rough, strict in ((0.3, True), (0.0, False)):
        mm, mv = _stats(rng, n, sd, rough)
        y = G.mlpg_ms(m, v, STD, mm, mv)
        for d in range(sd):
            f0 = O.chain_objective(m, v, STD, d, cm[:, d], mm[:, d], mv[:, d])
            f = O.chain_objective(m, v, STD, d, y[:, d], mm[:, d], mv[:, d])
            # the device accepts on its own evaluation of F, which differs from the oracle's by rounding
            assert f >= f0 - 1e-12 * abs(f0), (rough, d, f, f0)
            if strict:
                assert f > f0 + 1e-3 * abs(f0), (d, f, f0)


# ---- 5. a singular system ----------------------------------------------------------------------------------------
def test_not_positive_definite_raises():
    m, v = _data(np.random.default_rng(16), 50, 3, 2)
    v[20, 0::2] = -1.0  # every window of static dimension 0
    mm, mv = _stats(np.random.default_rng(17), 256, 2)
    with pytest.raises(np.linalg.LinAlgError):
        G.mlpg_ms(m, v, STD, mm, mv, n_iter=2)


# ---- 6. baseline.gmm.MLPG(ms=...) --------------------------------------------------------------------------------
def test_gmm_mlpg_with_ms_is_mlpg_ms_on_its_e_and_d():
    from sklearn.mixture import GaussianMixture

    from nnmnkwii_b200.baseline.gmm import MLPG
    w = windows_set()[1]
    rng = np.random.default_rng(18)
    sd = 3
    src = np.cumsum(rng.standard_normal((600, 2 * sd)), axis=0) * 0.1
    tgt = src * 0.8 + rng.standard_normal((600, 2 * sd)) * 0.1
    gmm = GaussianMixture(n_components=4, covariance_type="full", random_state=0).fit(np.hstack([src, tgt]))
    mm, mv = _stats(rng, 256, sd)
    model = MLPG(gmm, windows=w, ms=(mm, mv))
    utts = [src[:80], src[80:200], src[200:203]]
    batch = model.transform_batch(utts)
    for u, s in enumerate(utts):
        x, c = model._to_device(s)
        E, Dv = model._means_vars(x, c)
        want = G.mlpg_ms_batch(E, Dv, w, mm, mv, lengths=[len(s)]).cpu().numpy()
        y = model.transform(s)
        assert np.array_equal(y, want) and np.array_equal(batch[u], y), u
