"""Parameter generation considering global variance: properties of the float64 restatement
(oracle/gv.py) and the argument checks of the public API, which all run before any launch."""
import numpy as np
import pytest

from conftest import windows_set

import oracle.gv as ogv

WIN3 = windows_set()[2]


def _chain(rng, T, windows, smooth=True):
    """(mean, var) (T, nw) of one chain; smooth=True gives an over-smoothed trajectory (large static variances
    and small dynamic ones pull c_m towards a flat line)."""
    nw = len(windows)
    mean = rng.standard_normal((T, nw))
    var = rng.random((T, nw)) + 0.5
    if smooth:
        mean[:, 0] = np.sin(np.arange(T) / 7.0) * 2.0 + rng.standard_normal(T)
        mean[:, 1:] *= 0.05
        var[:, 0] *= 20.0
        var[:, 1:] *= 0.02
    return mean, var


@pytest.mark.parametrize("wi", range(4))
def test_mu_equal_to_cm_variance_returns_cm(wi):
    rng = np.random.default_rng(wi)
    w = windows_set()[wi]
    mean, var = _chain(rng, 120, w)
    cm = ogv.solve(*ogv.build_system(mean, var, w))
    out = ogv.mlpg_gv_chain(mean, var, w, ogv.variance(cm), 1.0, n_iter=20)
    assert np.abs(out - cm).max() <= 1e-12 * np.abs(cm).max()


def test_huge_gv_var_returns_cm():
    rng = np.random.default_rng(1)
    mean, var = _chain(rng, 200, WIN3)
    cm = ogv.solve(*ogv.build_system(mean, var, WIN3))
    # a huge gv_var leaves only the MLPG term of F: the first full step goes from the rescaled start back to c_m
    out = ogv.mlpg_gv_chain(mean, var, WIN3, 1.5 * ogv.variance(cm), 1e30, n_iter=20)
    assert np.abs(out - cm).max() <= 1e-12 * np.abs(cm).max()


@pytest.mark.parametrize("wi", range(4))
def test_objective_never_decreases_over_accepted_trials(wi):
    rng = np.random.default_rng(10 + wi)
    w = windows_set()[wi]
    mean, var = _chain(rng, 300, w)
    trace = []
    ogv.mlpg_gv_chain(mean, var, w, 2.0, 0.01, n_iter=30, trace=trace)
    accepted = [f for f, ok in trace if ok]
    assert len(accepted) >= 2
    assert all(b >= a for a, b in zip(accepted, accepted[1:]))


def test_gv_distance_shrinks_on_over_smoothed_data():
    rng = np.random.default_rng(3)
    mean, var = _chain(rng, 400, WIN3)
    cm = ogv.solve(*ogv.build_system(mean, var, WIN3))
    mu = 4.0 * ogv.variance(cm)
    out = ogv.mlpg_gv_chain(mean, var, WIN3, mu, 1e-3 * mu * mu, n_iter=20)
    assert abs(ogv.variance(out) - mu) < 0.5 * abs(ogv.variance(cm) - mu)


def test_zero_iterations_return_the_start_point():
    rng = np.random.default_rng(4)
    mean, var = _chain(rng, 150, WIN3)
    cm = ogv.solve(*ogv.build_system(mean, var, WIN3))
    mu = 3.0 * ogv.variance(cm)
    out = ogv.mlpg_gv_chain(mean, var, WIN3, mu, 0.1, n_iter=0)
    assert np.array_equal(out, np.mean(cm) + np.sqrt(mu / ogv.variance(cm)) * (cm - np.mean(cm)))
    flat = np.zeros((1, 3)), np.ones((1, 3))  # T = 1: v(c_m) == 0, c0 = c_m
    assert np.array_equal(ogv.mlpg_gv_chain(*flat, WIN3, 1.0, 1.0, n_iter=0), np.zeros(1))


def test_objective_from_the_factor_identity():
    """b^T c - c^T P c / 2 == -(c - c_m)^T P (c - c_m) / 2 + c_m^T P c_m / 2 (what the kernel's factor form relies on)."""
    rng = np.random.default_rng(5)
    mean, var = _chain(rng, 80, WIN3, smooth=False)
    Pu, b = ogv.build_system(mean, var, WIN3)
    cm = ogv.solve(Pu, b)
    c = rng.standard_normal(80)
    lhs = b @ c - 0.5 * c @ ogv.band_matvec(Pu, c)
    rhs = -0.5 * (c - cm) @ ogv.band_matvec(Pu, c - cm) + 0.5 * cm @ ogv.band_matvec(Pu, cm)
    assert abs(lhs - rhs) <= 1e-10 * abs(lhs)


@pytest.mark.skipif(not __import__("oracle").reference_available(), reason="oracle/_ref not built")
@pytest.mark.parametrize("wi", range(4))
@pytest.mark.parametrize("T", [1, 4, 157])
def test_oracle_cm_matches_reference_mlpg(wi, T):
    import oracle
    nn = oracle.import_reference()
    w = windows_set()[wi]
    rng = np.random.default_rng(T + wi)
    sd = 3
    m = rng.standard_normal((T, len(w) * sd))
    v = rng.random((T, len(w) * sd)) + 0.3
    ref = nn.paramgen.mlpg(m, v, w)
    ours = ogv.mlpg(m, v, w)
    assert np.abs(ours - ref).max() <= 1e-10 * max(1.0, np.abs(ref).max())


# ---- argument checks of the public API: raised before anything reaches a device -------------------------
def _args():
    rng = np.random.default_rng(0)
    m = rng.standard_normal((20, 6))
    v = rng.random((20, 6)) + 0.5
    return m, v, WIN3, np.ones(2), np.ones(2)


@pytest.mark.parametrize("bad", [
    dict(gv_var=np.array([1.0, 0.0])),
    dict(gv_var=np.array([1.0, -1.0])),
    dict(gv_var=np.array([1.0, np.nan])),
    dict(gv_mean=np.array([1.0, -0.5])),
    dict(gv_mean=np.array([1.0, np.inf])),
    dict(gv_mean=np.array([1.0, np.nan])),
    dict(gv_mean=np.ones(3)),
    dict(gv_var=np.ones(1)),
    dict(n_iter=-1),
    dict(n_iter=2.5),
    dict(step=0.0),
    dict(step=-1.0),
    dict(weight=0.0),
    dict(weight=-2.0),
])
def test_mlpg_gv_argument_errors(bad):
    from nnmnkwii_b200 import paramgen as G
    m, v, w, gm, gvv = _args()
    kw = dict(gv_mean=gm, gv_var=gvv, n_iter=5, step=1.0, weight=None)
    kw.update(bad)
    with pytest.raises(ValueError):
        G.mlpg_gv(m, v, w, **kw)
    with pytest.raises(ValueError):
        G.mlpg_gv_batch(m, v, w, lengths=[8, 12], **kw)


def test_mlpg_gv_batch_layout_and_padding_errors():
    from nnmnkwii_b200 import paramgen as G
    rng = np.random.default_rng(0)
    lay = G.merlin_layout()
    m = rng.standard_normal((30, 187))
    with pytest.raises(ValueError):  # one entry per OUTPUT column (63), not per static dim of one stream
        G.mlpg_gv_batch(m, m, WIN3, np.ones(60), np.ones(60), lengths=[30], layout=lay)
    with pytest.raises(ValueError):
        G.mlpg_gv_batch(m[None], m[None], WIN3, np.ones(63), np.ones(63), layout=lay)


def test_copied_columns_ignore_their_gv_entries():
    """Merlin's vuv column is copied: its gv entries are never read, so they are not checked either."""
    from nnmnkwii_b200 import paramgen as G
    lay = G.merlin_layout()
    gm, gvv = np.ones(63), np.ones(63)
    gm[61], gvv[61] = np.nan, 0.0
    out = G._gv_args(gm, gvv, lay, 3, 1.0, None)
    assert out[0][61] == 0.0 and out[1][61] == 1.0 and out[2:] == (3, 1.0, 0.0)


@pytest.mark.parametrize("case", ["zero_padded", "zero_flat", "no_lengths", "bad_offsets", "bad_sum"])
def test_global_variance_argument_errors(case):
    from nnmnkwii_b200 import paramgen as G
    x = np.ones((10, 4))
    with pytest.raises(ValueError):
        if case == "zero_padded":
            G.global_variance(np.ones((2, 5, 4)), lengths=[5, 0])
        elif case == "zero_flat":
            G.global_variance(x, offsets=[0, 4, 4, 10])
        elif case == "no_lengths":
            G.global_variance(np.ones((2, 5, 4)))
        elif case == "bad_offsets":
            G.global_variance(x, offsets=[0, 4, 9])
        else:
            G.gv_statistics(x, lengths=[3, 3])


def test_gmm_mlpg_gv_argument_errors():
    from sklearn.mixture import GaussianMixture

    from nnmnkwii_b200.baseline.gmm import MLPG
    rng = np.random.default_rng(0)
    X = rng.standard_normal((200, 8))
    gmm = GaussianMixture(n_components=2, covariance_type="full", random_state=0, max_iter=5).fit(X)
    with pytest.raises(ValueError):
        MLPG(gmm, gv=(np.ones(2), np.ones(2)), diff=True)
    with pytest.raises(ValueError):
        MLPG(gmm, gv=(np.ones(3), np.ones(2)))
    with pytest.raises(ValueError):
        MLPG(gmm, gv=(np.ones(2), np.zeros(2)))
    assert MLPG(gmm).gv is None and MLPG(gmm, gv=(np.ones(2), np.ones(2))).gv is not None
