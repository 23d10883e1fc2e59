"""Trajectory EM of GMM voice conversion on the GPU: baseline.gmm.MLPG.transform_em / transform_em_batch.

* n_iter = 0 is MLPG.transform / transform_batch bit for bit;
* parity with the float64 restatement (oracle/gmm_traj_em.py): trajectories within 1e-9 and the objective
  within 1e-10 relative, for every EPL instance of gmm_traj_em_kernel, diff / swap, T off the tile and T < the
  window; the device objective never decreases;
* a batch equals its utterances one by one, two calls are bit-identical, the errors come before any launch
  and the launch count depends on n_iter only.

Dirty allocations, workspace reuse and a delayed side stream are checked for these entry points by the
buffers-and-streams catalogue (tests/test_buffers_and_streams_gpu.py), as for every other one.  A call returns
only after its work has finished, so no table it reads can be evicted while that work is pending."""
import importlib.util
import os

import numpy as np
import pytest

from conftest import ROOT

import oracle.gmm_traj_em as OT

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location("make_gmm_traj_golden",
                                               os.path.join(ROOT, "tests", "golden", "make_gmm_traj_golden.py"))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
W = MG.WINDOWS


def _rel(a, b):
    return float(np.abs(np.asarray(a) - b).max() / max(1e-300, np.abs(b).max()))


def _model(S, nw, M, seed, swap=False, diff=False):
    from nnmnkwii_b200.baseline.gmm import MLPG
    g = MG.joint_gmm(np.random.default_rng(seed), M, S * nw)
    return g, MLPG(g, windows=W[:nw], swap=swap, diff=diff)


def _src(T, D, seed):
    return np.random.default_rng(seed + 1000).standard_normal((T, D))


def test_zero_iterations_is_transform_bit_for_bit():
    g, m = _model(3, 3, 5, 1)
    srcs = [_src(T, 9, T) for T in (70, 1, 33, 2)]
    for s in srcs:
        y, L = m.transform_em(s, n_iter=0, return_log_likelihood=True)
        assert np.array_equal(y, m.transform(s)) and L.shape == (1,)
        assert np.array_equal(m.transform_em(s, n_iter=0), m.transform(s))
    for got, want in zip(m.transform_em_batch(srcs, n_iter=0), m.transform_batch(srcs)):
        assert np.array_equal(got, want)


# (T, static_dim, nw, M, swap, diff): D = 4, 48, 48 from the issue's shapes; D = 30 / 80 for EPL 1 / 3;
# T = 1, 2 shorter than the delta window; T = 200, 600, 800 are not multiples of the 32-frame tile
PARITY = [(200, 2, 2, 4, False, False), (800, 24, 2, 32, False, False), (600, 16, 3, 8, False, False),
          (90, 10, 3, 6, True, False), (75, 40, 2, 3, False, True), (64, 20, 3, 4, True, True),
          (1, 2, 2, 3, False, False), (2, 3, 3, 2, False, True)]


@pytest.mark.parametrize("case", PARITY, ids=lambda c: "T%d_S%d_nw%d_M%d%s%s" % (c[:4] + (
    "_swap" if c[4] else "", "_diff" if c[5] else "")))
def test_oracle_parity(case):
    T, S, nw, M, swap, diff = case
    seed = T + 7 * S + M
    g, m = _model(S, nw, M, seed, swap, diff)
    src = _src(T, S * nw, seed)
    for n_iter in (1, 3, 10):
        want, Lw = OT.transform_em(g, W[:nw], src, n_iter, swap=swap, diff=diff)
        y, L = m.transform_em(src, n_iter=n_iter, return_log_likelihood=True)
        assert y.dtype == np.float64 and y.shape == (T, S) and L.shape == (n_iter + 1,)
        assert _rel(y, want) <= 1e-9, (n_iter, _rel(y, want))
        assert np.all(np.abs(L - Lw) <= 1e-10 * np.abs(Lw)), (n_iter, L, Lw)
        # EM never lowers the objective
        assert np.all(np.diff(L) >= -1e-12 * np.abs(L[:-1])), L


def test_batch_equals_each_utterance_and_calls_repeat_bit_for_bit():
    g, m = _model(4, 3, 7, 5, swap=True)
    lens = [100, 1, 0, 33, 64, 2]
    srcs = [_src(T, 12, i) for i, T in enumerate(lens)]
    ys, L = m.transform_em_batch(srcs, n_iter=4, return_log_likelihood=True)
    assert L.shape == (len(lens), 5) and not L[2].any()
    for i, s in enumerate(srcs):
        if not len(s):
            assert ys[i].shape == (0, 4)
            continue
        y1, L1 = m.transform_em(s, n_iter=4, return_log_likelihood=True)
        assert _rel(ys[i], y1) <= 1e-12 and np.all(np.abs(L[i] - L1) <= 1e-12 * np.abs(L1)), i
    ys2, L2 = m.transform_em_batch(srcs, n_iter=4, return_log_likelihood=True)
    assert all(np.array_equal(a, b) for a, b in zip(ys, ys2)) and np.array_equal(L, L2)
    assert np.array_equal(m.transform_em_batch(srcs, n_iter=4)[0], ys[0])


def test_errors_come_before_any_launch_and_launches_depend_on_n_iter_only():
    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200.baseline.gmm import MLPG
    g, m = _model(2, 2, 3, 9)
    src = _src(20, 4, 9)
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match="non-negative"):
        m.transform_em(src, n_iter=-1)
    with pytest.raises(ValueError, match="static and dynamic"):
        m.transform_em(src[:, :2])
    with pytest.raises(ValueError, match="global variance"):
        MLPG(g, windows=W[:2], gv=(np.ones(2), np.ones(2))).transform_em(src)
    bad = MG.joint_gmm(np.random.default_rng(9), 3, 4)
    bad.covariances_[1, 4 + 1, 4 + 1] = -50.0  # covarYY: a negative Eq. 23 variance
    with pytest.raises(ValueError, match="D_m"):
        MLPG(bad, windows=W[:2]).transform_em(src)
    gbig = MG.joint_gmm(np.random.default_rng(1), 2, 98)
    with pytest.raises(NotImplementedError, match="96"):
        MLPG(gbig, windows=W[:2]).transform_em(_src(5, 98, 1))
    with pytest.raises(NotImplementedError, match="96"):  # the same error as the arg-max path
        MLPG(gbig, windows=W[:2]).transform(_src(5, 98, 1))
    assert _lib.launch_count() == n0

    def launches(T, n_iter, ll):
        k = _lib.launch_count()
        m.transform_em(_src(T, 4, T), n_iter=n_iter, return_log_likelihood=ll)
        return _lib.launch_count() - k
    for n_iter in (0, 1, 3):
        for ll in (False, True):
            counts = {launches(T, n_iter, ll) for T in (1, 31, 32, 500, 2000)}
            assert len(counts) == 1, (n_iter, ll, counts)
    assert launches(50, 3, False) - launches(50, 2, False) == launches(50, 2, False) - launches(50, 1, False)
    assert launches(50, 2, True) == launches(50, 2, False) + 1
