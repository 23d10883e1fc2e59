"""Without a GPU: parameter generation from per-frame mixtures.  The float64 restatement the GPU tests compare
against (tests/mix_gen_oracle.py) never lowers its objective, is plain MLPG for one component and is the GMM
trajectory EM of oracle/gmm_traj_em.py when fed that model's per-frame terms; paramgen.mlpg_mixture /
mlpg_mixture_batch refuse bad arguments before any launch, and so does the C entry point."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest

import mix_gen_oracle as O
import oracle.gmm_traj_em as OT
from conftest import ROOT

_spec = importlib.util.spec_from_file_location("make_gmm_traj_golden",
                                               os.path.join(ROOT, "tests", "golden", "make_gmm_traj_golden.py"))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
SETS = MG.em_window_sets()


def mixture(rng, T, M, D, spread=1.0):
    """Random per-frame mixtures whose components are close enough in weight that the posteriors move."""
    lw = rng.standard_normal((T, M)) * 0.5
    mu = np.cumsum(rng.standard_normal((T, M, D)), axis=0) * 0.1 + spread * rng.standard_normal((1, M, D))
    s2 = rng.random((T, M, D)) * 0.5 + 0.1
    return lw, mu, s2


# ---- the restatement ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SETS))
def test_objective_never_decreases(name):
    w = SETS[name]
    H = MG.half_width(w)
    rng = np.random.default_rng(sum(map(ord, name)))
    S, M = 2, 4
    for T in sorted({1, 2, H, 2 * H + 1, 50} - {0}):
        lw, mu, s2 = mixture(rng, T, M, S * len(w))
        _, L = O.mlpg_mixture(lw, mu, s2, w, 20)
        assert L.shape == (21,) and np.all(np.isfinite(L))
        assert np.all(np.diff(L) >= -1e-12 * np.abs(L[:-1])), (T, np.diff(L).min())
        if T == 50:
            assert L[-1] > L[0]


@pytest.mark.parametrize("name", list(SETS))
def test_one_component_is_mlpg_at_every_iteration(name):
    import oracle
    w = SETS[name]
    rng = np.random.default_rng(5)
    lw, mu, s2 = mixture(rng, 37, 1, 3 * len(w))
    want = oracle.mlpg(mu[:, 0], s2[:, 0], w)
    trace = []
    O.mlpg_mixture(lw, mu, s2, w, 4, trace=trace)
    for c in trace:
        assert np.abs(c - want).max() <= 1e-12 * np.abs(want).max()


def test_merlin_streams_and_copied_column():
    """A copied column is its precision-weighted mean; the layout's streams solve independently."""
    w = SETS["nw3"]
    streams = [(0, 2), (6, 1), (9, 1, "copy"), (10, 1)]
    rng = np.random.default_rng(6)
    lw, mu, s2 = mixture(rng, 30, 3, 13)
    c, L = O.mlpg_mixture(lw, mu, s2, w, 10, streams=streams)
    assert c.shape == (30, 5) and np.all(np.diff(L) >= -1e-12 * np.abs(L[:-1]))
    p = O.Problem(lw, mu, s2, w, streams)
    c9 = O.mlpg_mixture(lw, mu, s2, w, 9, streams=streams)[0]
    gl = p.log_weights(c9)
    gamma = np.exp(gl - gl.max(1, keepdims=True))
    gamma /= gamma.sum(1, keepdims=True)
    want = (gamma * mu[:, :, 9] / s2[:, :, 9]).sum(1) / (gamma / s2[:, :, 9]).sum(1)
    assert np.abs(c[:, 3] - want).max() <= 1e-12 * np.abs(want).max()


@pytest.mark.parametrize("name", ["nw2", "nw3", "hw2", "asym", "h0"])
def test_gmm_per_frame_terms_give_the_gmm_trajectory_em(name):
    """lw = lp, mu = E_{m,t}, s2 = D_m of a joint GMM: the restatement is oracle/gmm_traj_em.transform_em."""
    w = SETS[name]
    S, M = 2, 4
    rng = np.random.default_rng(sum(map(ord, name)) + 1)
    g = MG.joint_gmm(rng, M, S * len(w))
    model = OT.Model(g, w, banded=True)
    for T in (1, 2, 5, 60):
        src = rng.standard_normal((T, S * len(w)))
        lp, E = model.frame_terms(src)
        c_want, L_want = OT.transform_em(g, w, src, 8, banded=True)
        c, L = O.mlpg_mixture(lp, E.transpose(1, 0, 2), np.broadcast_to(model.Dm, (T,) + model.Dm.shape), w, 8)
        assert np.abs(c - c_want).max() <= 1e-12 * np.abs(c_want).max(), T
        assert np.all(np.abs(L - L_want) <= 1e-12 * np.abs(L_want)), T


# ---- argument errors, before any launch --------------------------------------------------------------------------
STD = SETS["nw3"]


def _args(T=20, M=3, D=6):
    return mixture(np.random.default_rng(8), T, M, D)


@pytest.mark.parametrize("case", [
    "n_iter_neg", "n_iter_float", "n_iter_bool", "mu_2d", "s2_shape", "lw_shape", "lw_int", "mu_int", "M_65",
    "D_257", "M_0", "layout", "lengths_sum", "offsets", "padded_no_lengths", "padded_too_long", "mixed_forms",
    "layout_overlap", "layout_outside",
])
def test_argument_errors_raise_before_any_launch(case):
    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200 import paramgen as G
    lw, mu, s2 = _args()
    kw = {}
    if case == "n_iter_neg":
        kw["n_iter"] = -1
    elif case == "n_iter_float":
        kw["n_iter"] = 2.0
    elif case == "n_iter_bool":
        kw["n_iter"] = True
    elif case == "mu_2d":
        mu = mu[:, 0]
    elif case == "s2_shape":
        s2 = s2[:, :, :5]
    elif case == "lw_shape":
        lw = lw[:, :2]
    elif case == "lw_int":
        lw = lw.astype(np.int64)
    elif case == "mu_int":
        mu = mu.astype(np.int32)
    elif case == "M_65":
        lw, mu, s2 = _args(M=65)
    elif case == "D_257":
        lw, mu, s2 = _args(D=257)
        kw["layout"] = G.StreamLayout(257, [(0, 1)])
    elif case == "M_0":
        lw, mu, s2 = lw[:, :0], mu[:, :0], s2[:, :0]
    elif case == "layout":
        kw["layout"] = G.merlin_layout()
    elif case == "lengths_sum":
        kw["lengths"] = [10, 5]
    elif case == "offsets":
        kw["offsets"] = [0, 30]
    elif case == "padded_no_lengths":
        lw, mu, s2 = lw.reshape(2, 10, 3), mu.reshape(2, 10, 3, 6), s2.reshape(2, 10, 3, 6)
    elif case == "padded_too_long":
        lw, mu, s2 = lw.reshape(2, 10, 3), mu.reshape(2, 10, 3, 6), s2.reshape(2, 10, 3, 6)
        kw["lengths"] = [10, 11]
    elif case == "mixed_forms":
        import torch
        mu = torch.from_numpy(mu)
    elif case == "layout_overlap":
        kw["layout"] = G.StreamLayout(6, [(0, 2), (1, 1, "copy")])
    elif case == "layout_outside":
        kw["layout"] = G.StreamLayout(6, [(0, 2), (5, 1)])
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        G.mlpg_mixture_batch(lw, mu, s2, STD, **kw)
    if case not in ("lengths_sum", "offsets", "padded_no_lengths", "padded_too_long", "layout", "layout_overlap",
                    "layout_outside"):
        with pytest.raises(ValueError):
            G.mlpg_mixture(lw, mu, s2, STD, n_iter=kw.get("n_iter", 5))
    assert _lib.launch_count() == n0


def test_c_argument_checks():
    """Each bad argument gets NNK_ERR_ARG / NNK_ERR_UNSUPPORTED from the C entry point; no tiles is a no-op."""
    from nnmnkwii_b200 import _lib
    fn = _lib.lib.nnk_mix_gen

    def rc(**changes):
        a = _lib.NnkMixGenArgs()
        for k, name in enumerate(("log_weights", "means", "vars", "utt_off", "utt_len", "tile_off", "col_map",
                                  "c", "lnorm", "E", "V", "ll_part", "status_word")):
            setattr(a, name, 0x2000 + 0x100 * k)
        a.dtype, a.M, a.D, a.n_utt, a.n_tiles = _lib.NNK_F64, 4, 6, 1, 0
        a.win = _lib.make_windows(STD)
        a.mode, a.c_ld, a.c_cols = _lib.NNK_MIX_GEN_ESTEP, 2, 2
        for k, v in changes.items():
            if k == "half":
                a.win.u[1] = v
            else:
                setattr(a, k, v)
        return fn(ctypes.byref(a), None)

    assert rc() == _lib.NNK_OK
    assert fn(None, None) == _lib.NNK_ERR_ARG
    for bad in (dict(mode=3), dict(mode=-1), dict(dtype=2), dict(M=0), dict(D=0), dict(n_utt=0), dict(n_tiles=-1),
                dict(half=_lib.NNK_MAX_HALF + 1), dict(log_weights=None), dict(means=None), dict(vars=None),
                dict(utt_off=None), dict(utt_len=None), dict(tile_off=None), dict(col_map=None), dict(lnorm=None),
                dict(E=None), dict(V=None), dict(c=None), dict(c_cols=0), dict(c_ld=1),
                dict(mode=_lib.NNK_MIX_GEN_SELECT, status_word=None),
                dict(mode=_lib.NNK_MIX_GEN_OBJECTIVE, ll_part=None)):
        assert rc(**bad) == _lib.NNK_ERR_ARG, bad
    assert rc(mode=_lib.NNK_MIX_GEN_SELECT, c=None, c_cols=0, ll_part=None) == _lib.NNK_OK
    assert rc(mode=_lib.NNK_MIX_GEN_OBJECTIVE, E=None, V=None) == _lib.NNK_OK
    assert rc(ll_part=None, status_word=None) == _lib.NNK_OK
    assert rc(D=257) == _lib.NNK_ERR_UNSUPPORTED
    assert rc(M=65) == _lib.NNK_ERR_UNSUPPORTED

