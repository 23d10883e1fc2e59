"""Trajectory EM of GMM voice conversion (baseline.gmm.MLPG.transform_em, `gmm_traj_em_kernel<EPL, EM>` in
csrc/nnk_gmm_traj.cu) on every window set, kernel instance, batch layout and posterior regime the kernel takes,
against the float64 restatement oracle/gmm_traj_em.py.

The bars are those of tests/test_gmm_traj_em_gpu.py: trajectories within 1e-9 and the objective L within 1e-10
relative of the restatement, L never decreasing, n_iter = 0 equal to MLPG.transform bit for bit.

* Window sets (`MG.em_window_sets()`): half-widths 0 to 4, an asymmetric set whose H comes from `l` alone and
  four windows, at T = 1, H, 2H, 2H + 1 (all frames edge frames, or one interior frame), across the 32-frame
  tile (31, 32, 33, 95) and at 200 frames.  The half-width-3 / 4 and four-window sets run the M-step on
  `mlpg_kernel` instance 3.
* Every instance by name: D on both sides of each EPL = ceil(D / 32) step and at the D = 96 limit, with and
  without the objective-only launch; the profiler (in a child process, `variant_mirror.profiled_in_child`)
  must record all six `gmm_traj_em_kernel<EPL, EM>`.
* Batch layout: 287 utterances, with runs of empty ones at the start, in the middle and at the end, each
  equal to its own single call bit for bit (the tile-to-utterance search over `tile_off`).
* Posterior regimes: one-hot posteriors with the winning mixture first and last (the online log-sum-exp
  rescale), a permuted GMM, M = 1 (a fixed point), a zero-weight mixture (the `lw > -inf` skip), log-weights
  far below the float64 exp range, and M = 256.
* Long sums: T = 2000 against the banded path of the restatement."""
import importlib.util
import os
import re
import types

import numpy as np
import pytest

from conftest import ROOT

import oracle.gmm_traj_em as OT
import variant_mirror as VM

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location("make_gmm_traj_golden",
                                               os.path.join(ROOT, "tests", "golden", "make_gmm_traj_golden.py"))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
SETS = MG.em_window_sets()


def _rel(a, b):
    return float(np.abs(np.asarray(a) - b).max() / max(1e-300, np.abs(b).max()))


def _mlpg(g, w):
    from nnmnkwii_b200.baseline.gmm import MLPG
    return MLPG(g, windows=w)


def _gmm(M, D, seed):
    return MG.joint_gmm(np.random.default_rng(seed), M, D)


def _src(T, D, seed, scale=1.0):
    return scale * np.random.default_rng(seed + 1000).standard_normal((T, D))


def _check_parity(g, w, src, n_iters=(1, 3), banded=False, m=None):
    """The device against the restatement at each n_iter; returns the device (y, L) of the last one."""
    m = m or _mlpg(g, w)
    T, S = len(src), src.shape[1] // len(w)
    for n_iter in n_iters:
        y, L = m.transform_em(src, n_iter=n_iter, return_log_likelihood=True)
        assert y.dtype == np.float64 and y.shape == (T, S) and L.shape == (n_iter + 1,)
        if n_iter == 0:
            assert np.array_equal(y, m.transform(src))
        want, Lw = OT.transform_em(g, w, src, n_iter, banded=banded)
        assert _rel(y, want) <= 1e-9, (n_iter, _rel(y, want))
        assert np.all(np.abs(L - Lw) <= 1e-10 * np.abs(Lw)), (n_iter, L, Lw)
        assert np.all(np.diff(L) >= -1e-12 * np.abs(L[:-1])), (n_iter, L)
    return y, L


# ---- window sets -------------------------------------------------------------------------------------------------
def _set_cases():
    out = []
    for name, w in SETS.items():
        H = MG.half_width(w)
        for T in sorted({1, H, 2 * H, 2 * H + 1, 31, 32, 33, 95, 200} - {0}):
            out.append((name, T))
    return out


@pytest.mark.parametrize("name,T", _set_cases(), ids=lambda v: str(v))
def test_window_sets(name, T):
    w = SETS[name]
    S = 3
    if name in ("hw3", "hw4", "nw4"):  # the M-step solves on mlpg_kernel instance 3
        assert VM.pick_instance(w) == (4, 4, 4) and VM.mlpg_kernel_for("fwd", w, S * len(w), 8) == VM.DIRECT
    seed = 13 * T + len(name)
    _check_parity(_gmm(4, S * len(w), seed), w, _src(T, S * len(w), seed), n_iters=(0, 1, 5))


# ---- every instance, by name -------------------------------------------------------------------------------------
# (static_dim, window set): D = 30, 32 | 33, 64 | 66, 96 on both sides of each EPL step and at the limit
INSTANCES = [(10, "nw3"), (16, "nw2"), (11, "nw3"), (32, "nw2"), (22, "nw3"), (32, "nw3"), (48, "nw2"), (24, "nw4")]


def launch(S, name, ll):
    """One small conversion of D = S * nw features (run under the profiler by `profiled_in_child`)."""
    w = SETS[name]
    D = S * len(w)
    _mlpg(_gmm(3, D, D), w).transform_em(_src(40, D, D), n_iter=1, return_log_likelihood=ll)


def test_every_instance_is_launched_by_name():
    # each kernel the test asserts on is named, so that a profile that lost one of them is taken again
    cases = [([S, name, ll], [r"\bgmm_traj_em_kernel<", r"\bgmm_traj_em_kernel<\d, true>"]
              + ([r"\bgmm_traj_em_kernel<\d, false>"] if ll else [])) for S, name in INSTANCES for ll in (False, True)]
    res = VM.profiled_in_child("test_gmm_traj_em_variants_gpu", "launch", cases)
    seen = set()
    for (case, _), (names, err) in zip(cases, res):
        S, name, ll = case
        assert err == "None", (case, err)
        epl = VM.traj_epl(S * len(SETS[name]))
        want = {"gmm_traj_em_kernel<%d, true>" % epl} | ({"gmm_traj_em_kernel<%d, false>" % epl} if ll else set())
        got = {re.search(r"gmm_traj_em_kernel<\d, (true|false)>", n).group(0) for n in names}
        assert got == want, (case, names)
        seen |= got
    assert len(seen) == 2 * VM.TRAJ_MAX_EPL, seen


@pytest.mark.parametrize("S,name", INSTANCES, ids=lambda v: str(v))
def test_every_instance(S, name):
    w = SETS[name]
    D = S * len(w)
    g, src = _gmm(4, D, 7 * D), _src(70, D, D)
    m = _mlpg(g, w)
    y, _ = _check_parity(g, w, src, n_iters=(3,), m=m)
    assert np.array_equal(m.transform_em(src, n_iter=3), y)  # the objective launch changes nothing


# ---- batch layout ------------------------------------------------------------------------------------------------
def _batch_lengths():
    rng = np.random.default_rng(11)
    lens = list(rng.choice([0, 1, 2, 31, 32, 33, 64, 65, 100], size=280))
    lens[:5] = [0] * 5          # empties at the start
    lens[140:150] = [0] * 10    # a run in the middle
    return [int(n) for n in lens] + [0] * 7  # and at the end


def test_batch_layout():
    w = SETS["nw3"]
    S, n_iter = 4, 3
    g = _gmm(5, S * len(w), 21)
    m = _mlpg(g, w)
    lens = _batch_lengths()
    srcs = [_src(T, S * len(w), i) for i, T in enumerate(lens)]
    ys, L = m.transform_em_batch(srcs, n_iter=n_iter, return_log_likelihood=True)
    assert len(ys) == len(lens) and L.shape == (len(lens), n_iter + 1)
    for i, s in enumerate(srcs):
        if not len(s):
            assert ys[i].shape == (0, S) and not L[i].any(), i
            continue
        y1, L1 = m.transform_em(s, n_iter=n_iter, return_log_likelihood=True)
        assert np.array_equal(ys[i], y1) and np.array_equal(L[i], L1), (i, lens[i], _rel(ys[i], y1), L[i] - L1)
    for i in [lens.index(T) for T in (1, 2, 31, 32, 33, 64, 65, 100)]:
        want, Lw = OT.transform_em(g, w, srcs[i], n_iter)
        assert _rel(ys[i], want) <= 1e-9 and np.all(np.abs(L[i] - Lw) <= 1e-10 * np.abs(Lw)), (i, lens[i])


# ---- posterior regimes -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("winner", ["first", "last"])
def test_separated_mixtures(winner):
    """Means 30 times apart: every frame's posterior is one-hot, on mixture 0 or on the last one.  With the
    winner last the online log-sum-exp must rescale the accumulators of all earlier mixtures away."""
    w = SETS["nw3"]
    S, M, T = 2, 5, 70
    D = S * len(w)
    g = _gmm(M, D, 5)
    g.means_ = 30.0 * g.means_
    k = 0 if winner == "first" else M - 1
    src = g.means_[k, :D] + 0.3 * _src(T, D, 5)
    lp, _ = OT.Model(g, w).frame_terms(src)
    others = np.delete(lp, k, axis=1)
    assert np.all(lp[:, k] - others.max(axis=1) > 800)  # exp of the gap underflows: one-hot in float64
    _check_parity(g, w, src, n_iters=(1, 3))


def test_permuted_mixtures():
    w = SETS["hw2"]
    D = 3 * len(w)
    g, src = _gmm(6, D, 8), _src(90, D, 8)
    perm = np.random.default_rng(8).permutation(6)
    gp = types.SimpleNamespace(weights_=g.weights_[perm], means_=g.means_[perm], covariances_=g.covariances_[perm],
                                  covariance_type="full")
    y, L = _mlpg(g, w).transform_em(src, n_iter=5, return_log_likelihood=True)
    yp, Lp = _mlpg(gp, w).transform_em(src, n_iter=5, return_log_likelihood=True)
    assert _rel(yp, y) <= 1e-12 and np.all(np.abs(Lp - L) <= 1e-12 * np.abs(L)), (_rel(yp, y), Lp - L)


@pytest.mark.parametrize("name", ["nw3", "hw4"])
def test_one_mixture_is_a_fixed_point(name):
    w = SETS[name]
    D = 3 * len(w)
    g, src = _gmm(1, D, 4), _src(80, D, 4)
    m = _mlpg(g, w)
    y0 = m.transform(src)
    for n_iter in (1, 4):
        y, L = m.transform_em(src, n_iter=n_iter, return_log_likelihood=True)
        assert _rel(y, y0) <= 1e-12 and np.all(np.abs(L - L[0]) <= 1e-12 * np.abs(L[0])), (n_iter, _rel(y, y0), L)


@pytest.mark.parametrize("where", ["first", "last"])
def test_zero_weight_mixture_is_left_out(where):
    """A mixture of weight exactly 0 has lp = -inf on every frame: the GMM with it converts as the GMM without."""
    w = SETS["nw3"]
    D = 2 * len(w)
    g, src = _gmm(4, D, 6), _src(75, D, 6)
    extra = _gmm(1, D, 60)
    i = 0 if where == "first" else 4
    g0 = types.SimpleNamespace(weights_=np.insert(g.weights_, i, 0.0),
                                  means_=np.insert(g.means_, i, extra.means_[0], axis=0),
                                  covariances_=np.insert(g.covariances_, i, extra.covariances_[0], axis=0),
                                  covariance_type="full")
    for n_iter in (0, 3):
        y, L = _mlpg(g, w).transform_em(src, n_iter=n_iter, return_log_likelihood=True)
        with np.errstate(divide="ignore"):  # log 0 of the zero weight
            y0, L0 = _mlpg(g0, w).transform_em(src, n_iter=n_iter, return_log_likelihood=True)
        assert np.all(np.isfinite(y0)) and np.all(np.isfinite(L0))
        assert _rel(y0, y) <= 1e-12 and np.all(np.abs(L0 - L) <= 1e-12 * np.abs(L)), (n_iter, _rel(y0, y), L0 - L)


def test_log_weights_below_the_exp_range():
    """Source frames far from every mixture: every lw_{t,m} is below log of the smallest double, so only a
    log-sum-exp taken relative to the frame's maximum keeps the posteriors."""
    w = SETS["nw3"]
    D = 2 * len(w)
    g, src = _gmm(5, D, 9), 60.0 + _src(64, D, 9, scale=10.0)
    lp, _ = OT.Model(g, w).frame_terms(src)
    assert np.all(lp.max(axis=1) < -746)
    _check_parity(g, w, src, n_iters=(1, 3))


def test_many_mixtures():
    w = SETS["nw3"]
    D = 2 * len(w)
    _check_parity(_gmm(256, D, 10), w, _src(40, D, 10), n_iters=(1, 3))


# ---- long sums ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["nw3", "asym"])
def test_long_utterance(name):
    """63 tiles in one utterance: their partial objectives fold into L (restatement: the banded solve)."""
    w = SETS[name]
    D = 4 * len(w)
    _check_parity(_gmm(8, D, 12), w, _src(2000, D, 12), n_iters=(3,), banded=True)
