"""Without a GPU: the float64 restatement of the trajectory EM (oracle/gmm_traj_em.py) never lowers its
objective, starts from the reference's MLPG.transform and, on every window set the GPU tests use, from the C
restatement of mlpg; its banded path equals its dense one; the C entry point refuses bad arguments before
touching the device."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest

from conftest import ROOT

import oracle.gmm_traj_em as OT

_spec = importlib.util.spec_from_file_location("make_gmm_traj_golden",
                                               os.path.join(ROOT, "tests", "golden", "make_gmm_traj_golden.py"))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)


@pytest.mark.parametrize("swap,diff", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("S,nw,M", [(2, 2, 4), (3, 3, 3)])
def test_oracle_objective_never_decreases(S, nw, M, swap, diff):
    rng = np.random.default_rng(7 * S + nw + M)
    g = MG.joint_gmm(rng, M, S * nw)
    src = rng.standard_normal((40, S * nw))
    _, L = OT.transform_em(g, MG.WINDOWS[:nw], src, 20, swap=swap, diff=diff)
    assert L.shape == (21,) and np.all(np.isfinite(L))
    assert np.all(np.diff(L) >= -1e-12 * np.abs(L[:-1]))
    assert L[-1] > L[0]


def test_oracle_starts_from_the_reference_transform():
    golden = np.load(os.path.join(ROOT, "tests", "golden", "gmm_traj_reference_golden.npz"))
    import types
    for i, (T, S, nw, M, swap, diff) in enumerate(MG.cases()):
        g = types.SimpleNamespace(weights_=golden["weights_%d" % i], means_=golden["means_%d" % i],
                                  covariances_=golden["covariances_%d" % i], covariance_type="full")
        c, L = OT.transform_em(g, MG.WINDOWS[:nw], golden["src_%d" % i], 0, swap=swap, diff=diff)
        want = golden["y_%d" % i]
        assert c.shape == want.shape == (T, S) and L.shape == (1,)
        assert np.abs(c - want).max() <= 1e-10 * np.abs(want).max(), i


SETS = MG.em_window_sets()


@pytest.mark.parametrize("name", list(SETS))
def test_oracle_starts_from_mlpg_and_climbs_on_every_window_set(name):
    """c_0 is the C restatement's mlpg of the arg-max mixture's E and D_m on every window set (the edge rule is
    mlpg's, [-0:] included), and the objective never decreases over 20 iterations."""
    import oracle
    w = SETS[name]
    S, M = 3, 6
    rng = np.random.default_rng(sum(map(ord, name)))
    g = MG.joint_gmm(rng, M, S * len(w))
    model = OT.Model(g, w)
    for T in sorted({1, 2, MG.half_width(w), 2 * MG.half_width(w) + 1, 40} - {0}):
        src = rng.standard_normal((T, S * len(w)))
        lp, E = model.frame_terms(src)
        mix = np.argmax(lp, axis=1)
        want = oracle.mlpg(E[mix, np.arange(T)], model.Dm[mix], w)
        c, L = OT.transform_em(g, w, src, 20)
        assert np.abs(OT.transform_em(g, w, src, 0)[0] - want).max() <= 1e-12 * np.abs(want).max(), T
        assert L.shape == (21,) and np.all(np.isfinite(L))
        assert np.all(np.diff(L) >= -1e-12 * np.abs(L[:-1])), (T, np.diff(L).min())


@pytest.mark.parametrize("name", ["nw3", "asym", "hw4", "h0"])
def test_banded_restatement_equals_the_dense_one(name):
    """The banded path the long-utterance GPU tests use against the dense one, T around the window and beyond."""
    w = SETS[name]
    rng = np.random.default_rng(3)
    g = MG.joint_gmm(rng, 5, 2 * len(w))
    for T in (1, 2, 5, 150):
        src = rng.standard_normal((T, 2 * len(w)))
        cd, Ld = OT.transform_em(g, w, src, 3)
        cb, Lb = OT.transform_em(g, w, src, 3, banded=True)
        assert np.abs(cb - cd).max() <= 1e-11 * np.abs(cd).max(), T
        assert np.all(np.abs(Lb - Ld) <= 1e-12 * np.abs(Ld)), T


def _valid_args(_lib):
    """A filled argument block with distinct non-NULL dummy pointers; nothing behind them is ever read."""
    g = _lib.NnkGmm()
    g.src_means = g.tgt_means = g.prec_chol = g.log_const = g.A_t = g.Dm = 0x1000
    g.M, g.D = 4, 4
    a = _lib.NnkGmmTrajArgs()
    for k, name in enumerate(("x", "lp", "c", "utt_off", "tile_off", "inv_Dm", "log_norm", "E_bar", "V", "ll_part")):
        setattr(a, name, 0x2000 + 0x100 * k)
    a.x_ld, a.c_ld, a.T, a.n_utt, a.n_tiles, a.static_dim = 4, 2, 0, 1, 0, 2
    a.win = _lib.make_windows([(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5]))])
    a.mode = _lib.NNK_GMM_TRAJ_EM
    return g, a


def test_c_argument_checks():
    """Each bad argument gets NNK_ERR_ARG / NNK_ERR_UNSUPPORTED from the C entry point; T = 0 is a no-op."""
    from nnmnkwii_b200 import _lib
    fn = _lib.lib.nnk_gmm_traj_em
    g, a = _valid_args(_lib)
    assert fn(ctypes.byref(g), ctypes.byref(a), None) == _lib.NNK_OK
    assert fn(None, ctypes.byref(a), None) == _lib.NNK_ERR_ARG
    assert fn(ctypes.byref(g), None, None) == _lib.NNK_ERR_ARG

    def rc(**changes):
        g, a = _valid_args(_lib)
        for k, v in changes.items():
            if k.startswith("g_"):
                setattr(g, k[2:], v)
            elif k == "half":
                a.win.u[1] = v
            else:
                setattr(a, k, v)
        return fn(ctypes.byref(g), ctypes.byref(a), None)

    for bad in (dict(mode=2), dict(mode=-1), dict(T=-1), dict(n_utt=0), dict(n_tiles=-1), dict(static_dim=0),
                dict(static_dim=3), dict(g_D=5), dict(g_M=0), dict(x_ld=3), dict(c_ld=1), dict(x=None), dict(lp=None),
                dict(c=None), dict(utt_off=None), dict(tile_off=None), dict(inv_Dm=None), dict(log_norm=None),
                dict(E_bar=None), dict(V=None), dict(g_A_t=None), dict(g_src_means=None), dict(g_tgt_means=None),
                dict(mode=_lib.NNK_GMM_TRAJ_OBJECTIVE, ll_part=None), dict(half=_lib.NNK_MAX_HALF + 1)):
        assert rc(**bad) == _lib.NNK_ERR_ARG, bad
    # the objective mode needs no E_bar / V, the EM mode no ll_part
    assert rc(mode=_lib.NNK_GMM_TRAJ_OBJECTIVE, E_bar=None, V=None) == _lib.NNK_OK
    assert rc(ll_part=None) == _lib.NNK_OK
    # more than 96 features, more than 65535 mixtures
    assert rc(g_D=98, static_dim=49, x_ld=98, c_ld=49) == _lib.NNK_ERR_UNSUPPORTED
    assert rc(g_M=65536) == _lib.NNK_ERR_UNSUPPORTED
    assert "96" in _lib.last_error() or "65535" in _lib.last_error()
