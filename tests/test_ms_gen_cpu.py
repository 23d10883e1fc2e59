"""Without a GPU: parameter generation considering the modulation spectrum.  The float64 restatement
(oracle/ms_gen.py) the GPU tests compare against has the definition's properties (analytic gradient, an objective
that never decreases, plain MLPG for n_iter = 0 or exempt bins); paramgen.mlpg_ms / mlpg_ms_batch and
baseline.gmm.MLPG(ms=...) refuse bad arguments before any device work."""
import numpy as np
import pytest

import oracle.gv as ogv
import oracle.ms_gen as O
from conftest import windows_set

STD = windows_set()[2]


def _data(seed, T, sd, n, rough=0.3):
    rng = np.random.default_rng(seed)
    m = np.concatenate([np.cumsum(rng.standard_normal((T, sd)), 0) * 0.1, 0.05 * rng.standard_normal((T, 2 * sd))], 1)
    v = rng.random((T, 3 * sd)) + 0.5
    nat = rng.standard_normal((8, n, sd)) * rough + np.cumsum(rng.standard_normal((8, n, sd)), 1) * 0.05
    s = np.log(np.maximum(np.abs(np.fft.rfft(nat, n, axis=1)) ** 2, O.TINY))
    return m, v, s.mean(0), s.var(0) + 0.5


# ---- the restatement ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,n", [(1, 256), (37, 256), (256, 256), (300, 512)])
def test_gradient_matches_central_differences(T, n):
    _, _, mm, mv = _data(T, T, 1, n)
    rng = np.random.default_rng(T + 1)
    c = np.cumsum(rng.standard_normal(T)) * 0.2
    q = O._precisions(mv[:, 0])
    q[5] = 0.0  # an exempt bin
    g = O.ms_gradient(c, mm[:, 0], q, n)
    e = 1e-6
    eye = np.eye(T)
    fd = np.array([(O.ms_term(c + e * eye[t], mm[:, 0], q, n) - O.ms_term(c - e * eye[t], mm[:, 0], q, n)) / (2 * e)
                   for t in range(T)])
    assert np.abs(fd - g).max() <= 1e-6 * np.abs(g).max()


@pytest.mark.parametrize("wi", range(4))
def test_objective_never_decreases(wi):
    w = windows_set()[wi]
    rng = np.random.default_rng(wi)
    T, n = 200, 256
    m = np.cumsum(rng.standard_normal((T, len(w))), 0) * 0.1
    v = rng.random((T, len(w))) + 0.5
    _, _, mm, mv = _data(wi, 1, 1, n)
    tr = []
    O.mlpg_ms_chain(m, v, w, mm[:, 0], mv[:, 0], n, n_iter=20, trace=tr)
    kept = [f for f, ok, _ in tr if ok]
    assert all(b >= a for a, b in zip(kept, kept[1:]))
    assert kept[-1] > kept[0] and len(kept) > 1


def test_no_trial_or_exempt_bins_return_cm():
    m, v, mm, mv = _data(3, 120, 2, 256)
    cm = ogv.mlpg(m, v, STD)
    assert np.array_equal(O.mlpg_ms(m, v, STD, mm, mv, n_iter=0), cm)
    inf = np.full_like(mv, np.inf)
    nan = np.full_like(mm, np.nan)  # exempt bins never read their mean
    assert np.array_equal(O.mlpg_ms(m, v, STD, nan, inf, n_iter=10), cm)


def test_zero_power_bins_add_no_gradient():
    c = np.zeros(40)
    q = np.ones(129)
    assert not O.ms_gradient(c, np.zeros(129), q, 256).any()
    assert O.ms_term(c, np.full(129, np.log(O.TINY)), q, 256) == 0.0


# ---- argument errors, before any device work ---------------------------------------------------------------------
def _args(K=129, D=2):
    m, v, mm, mv = _data(4, 50, D, 2 * (K - 1))
    return m, v, mm, mv


@pytest.mark.parametrize("case", [
    "K", "cols", "shape_mismatch", "var_zero", "var_neg", "var_nan", "mean_nan", "mean_inf", "too_long",
    "n_iter_neg", "n_iter_float", "n_iter_bool", "step_zero", "step_nan", "weight_zero", "weight_inf", "text",
])
def test_mlpg_ms_argument_errors(case):
    from nnmnkwii_b200 import paramgen as G
    m, v, mm, mv = _args()
    kw = {}
    if case == "K":
        mm, mv = mm[:100], mv[:100]
    elif case == "cols":
        mm, mv = mm[:, :1], mv[:, :1]
    elif case == "shape_mismatch":
        mv = np.ones((257, 2))
    elif case == "var_zero":
        mv[3, 1] = 0.0
    elif case == "var_neg":
        mv[3, 1] = -1.0
    elif case == "var_nan":
        mv[7, 0] = np.nan
    elif case == "mean_nan":
        mm[7, 0] = np.nan
    elif case == "mean_inf":
        mm[0, 1] = np.inf
    elif case == "too_long":
        m, v = np.zeros((257, 6)), np.ones((257, 6))
    elif case == "n_iter_neg":
        kw["n_iter"] = -1
    elif case == "n_iter_float":
        kw["n_iter"] = 2.5
    elif case == "n_iter_bool":
        kw["n_iter"] = True
    elif case == "step_zero":
        kw["step"] = 0.0
    elif case == "step_nan":
        kw["step"] = float("nan")
    elif case == "weight_zero":
        kw["weight"] = 0.0
    elif case == "weight_inf":
        kw["weight"] = float("inf")
    elif case == "text":
        mm = "abc"
    with pytest.raises(ValueError):
        G.mlpg_ms(m, v, STD, mm, mv, **kw)
    with pytest.raises(ValueError):
        G.mlpg_ms_batch(m, v, STD, mm, mv, lengths=[len(m)], **kw)


def test_mlpg_ms_batch_layout_and_length_errors():
    from nnmnkwii_b200 import paramgen as G
    m, v, mm, mv = _args()
    with pytest.raises(ValueError, match="longer than the DFT length"):
        G.mlpg_ms_batch(np.zeros((300, 6)), np.ones((300, 6)), STD, mm, mv, lengths=[40, 260])
    with pytest.raises(ValueError, match="longer than the DFT length"):
        G.mlpg_ms_batch(np.zeros((2, 300, 6)), np.ones((2, 300, 6)), STD, mm, mv, lengths=[3, 257])
    with pytest.raises(ValueError, match="needs lengths"):
        G.mlpg_ms_batch(np.zeros((2, 30, 6)), np.ones((2, 30, 6)), STD, mm, mv)
    with pytest.raises(ValueError, match="lengths sum"):
        G.mlpg_ms_batch(m, v, STD, mm, mv, lengths=[10, 10])
    with pytest.raises(ValueError, match="offsets"):
        G.mlpg_ms_batch(m, v, STD, mm, mv, offsets=[0, 60])
    with pytest.raises(ValueError, match="layout covers"):
        G.mlpg_ms_batch(m, v, STD, mm, mv, layout=G.merlin_layout())
    # the copied column's statistics are neither used nor checked
    layout = G.merlin_layout()
    K = 129
    mm, mv = np.zeros((K, 63)), np.ones((K, 63))
    mm[:, 61], mv[:, 61] = np.nan, -1.0
    with pytest.raises(ValueError, match="DFT length"):  # gets past the statistics' checks
        G.mlpg_ms_batch(np.zeros((300, 187)), np.ones((300, 187)), STD, mm, mv, layout=layout)


def test_gmm_mlpg_ms_argument_errors():
    from sklearn.mixture import GaussianMixture

    from nnmnkwii_b200.baseline.gmm import MLPG
    rng = np.random.default_rng(0)
    X = rng.standard_normal((200, 8))
    gmm = GaussianMixture(n_components=2, covariance_type="full", random_state=0, max_iter=5).fit(X)
    good = (np.zeros((129, 2)), np.ones((129, 2)))
    with pytest.raises(ValueError, match="diff"):
        MLPG(gmm, ms=good, diff=True)
    with pytest.raises(ValueError, match="cannot be combined"):
        MLPG(gmm, ms=good, gv=(np.ones(2), np.ones(2)))
    with pytest.raises(ValueError):
        MLPG(gmm, ms=(np.zeros((129, 3)), np.ones((129, 3))))
    with pytest.raises(ValueError):
        MLPG(gmm, ms=(np.zeros((100, 2)), np.ones((100, 2))))
    with pytest.raises(ValueError):
        MLPG(gmm, ms=(np.zeros((129, 2)), np.zeros((129, 2))))
    model = MLPG(gmm, ms=good)
    assert MLPG(gmm).ms is None and model.ms is not None
    with pytest.raises(ValueError, match="modulation spectrum"):
        model.transform_em(rng.standard_normal((20, 4)))
