"""Without a GPU: parameter generation considering the segment-level modulation spectrum.  The float64 restatement
(tests/ms_gen_segment_oracle.py) the GPU tests compare against has the definition's properties (its closed-form
gradient is the derivative of its MS term, checked by central differences and by torch autograd of the
definition; its objective never decreases; n_iter = 0 is plain MLPG); paramgen.mlpg_ms / mlpg_ms_batch with
``segment`` and baseline.gmm.MLPG(ms_segment=...) refuse bad arguments before any device work while
``segment=None`` keeps its refusals."""
import numpy as np
import pytest

import ms_gen_segment_oracle as S
import oracle.gv as ogv
import oracle.ms_segment as oseg
from conftest import windows_set

STD = windows_set()[2]


def _stats(seed, n, sd, L, rough=0.3):
    rng = np.random.default_rng(seed)
    nat = rng.standard_normal((4, 3 * n, sd)) * rough + np.cumsum(rng.standard_normal((4, 3 * n, sd)), 1) * 0.05
    mean, var = oseg.statistics(list(nat), n, L)
    return mean, var + 0.5


def _data(seed, T, sd):
    rng = np.random.default_rng(seed)
    m = np.concatenate([np.cumsum(rng.standard_normal((T, sd)), 0) * 0.1, 0.05 * rng.standard_normal((T, 2 * sd))], 1)
    return m, rng.random((T, 3 * sd)) + 0.5


# ---- the restatement ---------------------------------------------------------------------------------------------
def _gradient_cases():
    cases = []
    for n in (64, 128):
        for L in (4, 50, n):
            H = L // 2
            for T in sorted({1, 2, max(H - 1, 1), H, H + 1, 300}):
                cases.append((T, n, L))
    return cases


@pytest.mark.parametrize("T,n,L", _gradient_cases())
def test_gradient_matches_central_differences_and_autograd(T, n, L):
    torch = pytest.importorskip("torch")
    mm, mv = _stats(T + L, n, 1, L)
    rng = np.random.default_rng([T, n, L])
    c = np.cumsum(rng.standard_normal(T)) * 0.2 + 0.3
    q = S._precisions(mv[:, 0])
    q[3] = 0.0  # an exempt bin
    nu = mm[:, 0]
    g = S.ms_gradient(c, nu, q, n, L)
    # central differences on a subset of frames (all of them for short chains); the log of a short segment's
    # small powers curves fast, so the differences carry a truncation error of ~1e-5 at this step
    e = 1e-6
    ts = np.unique(np.linspace(0, T - 1, min(T, 40)).astype(int))
    for t in ts:
        d = np.zeros(T)
        d[t] = e
        fd = (S.ms_term(c + d, nu, q, n, L) - S.ms_term(c - d, nu, q, n, L)) / (2 * e)
        assert abs(fd - g[t]) <= 1e-4 * max(np.abs(g).max(), 1e-12), (t, fd, g[t])
    # torch autograd of the definition, float64
    H = L // 2
    J = S.count(T, L)
    ct = torch.tensor(c, dtype=torch.float64, requires_grad=True)
    pad = torch.cat([torch.zeros(H, dtype=torch.float64), ct, torch.zeros(J * H + L, dtype=torch.float64)])
    segs = torch.stack([pad[j * H:j * H + L] for j in range(J)]) * torch.tensor(S.window(L))
    P = torch.fft.rfft(segs, n, dim=1).abs() ** 2
    s = torch.log(torch.clamp(P, min=S.TINY))
    on = torch.tensor(q > 0)
    on[0] = False
    qt, nut = torch.tensor(q), torch.tensor(nu)
    F = -0.5 * (qt[on] * (s[:, on] - nut[on]) ** 2).sum() / J
    F.backward()
    assert abs(F.item() - S.ms_term(c, nu, q, n, L)) <= 1e-12 * abs(F.item())
    assert np.abs(ct.grad.numpy() - g).max() <= 1e-10 * np.abs(g).max()


def test_zero_power_segments_add_no_gradient():
    c = np.zeros(40)
    q = np.ones(33)
    assert not S.ms_gradient(c, np.zeros(33), q, 64, 20).any()
    assert S.ms_term(c, np.full(33, np.log(S.TINY)), q, 64, 20) == 0.0
    # one nonzero frame: the segments that miss it have zero power everywhere and add nothing
    c[0] = 1.0
    g = S.ms_gradient(c, np.zeros(33), q, 64, 20)
    assert np.isfinite(g).all() and not g[20:].any()


@pytest.mark.parametrize("wi", range(4))
def test_objective_never_decreases(wi):
    w = windows_set()[wi]
    rng = np.random.default_rng(wi)
    T, n, L = 700, 64, 50
    m = np.cumsum(rng.standard_normal((T, len(w))), 0) * 0.1
    v = rng.random((T, len(w))) + 0.5
    mm, mv = _stats(wi, n, 1, L)
    tr = []
    S.mlpg_ms_chain(m, v, w, mm[:, 0], mv[:, 0], n, L, n_iter=20, trace=tr)
    kept = [f for f, ok, _ in tr if ok]
    assert all(b >= a for a, b in zip(kept, kept[1:]))
    assert kept[-1] > kept[0] and len(kept) > 1


def test_no_trial_or_exempt_bins_return_cm():
    m, v = _data(3, 500, 2)
    mm, mv = _stats(3, 64, 2, 50)
    cm = ogv.mlpg(m, v, STD)
    assert np.array_equal(S.mlpg_ms(m, v, STD, mm, mv, 50, n_iter=0), cm)
    inf = np.full_like(mv, np.inf)
    nan = np.full_like(mm, np.nan)  # exempt bins never read their mean
    assert np.array_equal(S.mlpg_ms(m, v, STD, nan, inf, 50, n_iter=10), cm)


def test_a_long_utterance_takes_seconds():
    import time
    m, v = _data(5, 20000, 1)
    mm, mv = _stats(5, 64, 1, 50)
    t0 = time.perf_counter()
    y = S.mlpg_ms(m, v, STD, mm, mv, 50, n_iter=20)
    assert np.isfinite(y).all() and time.perf_counter() - t0 < 60


# ---- argument errors, before any device work ---------------------------------------------------------------------
def _args(n=64, L=50, D=2, T=50):
    m, v = _data(4, T, D)
    mm, mv = _stats(4, n, D, min(L, n))
    return m, v, mm, mv


@pytest.mark.parametrize("case", [
    "n_big", "n_small", "n_odd_bins", "L_odd", "L_small", "L_big", "L_float", "L_str", "L_bool", "var_zero",
    "mean_nan", "n_iter_neg", "step_zero", "weight_inf", "cols",
])
def test_segment_argument_errors(case):
    from nnmnkwii_b200 import paramgen as G
    m, v, mm, mv = _args()
    L = 50
    exc = ValueError
    if case == "n_big":
        mm, mv = np.zeros((513, 2)), np.ones((513, 2))
    elif case == "n_small":
        mm, mv = np.zeros((9, 2)), np.ones((9, 2))
    elif case == "n_odd_bins":
        mm, mv = mm[:30], mv[:30]
    elif case == "L_odd":
        L = 49
    elif case == "L_small":
        L = 2
    elif case == "L_big":
        L = 66
    elif case in ("L_float", "L_str", "L_bool"):
        L, exc = {"L_float": 50.0, "L_str": "50", "L_bool": True}[case], TypeError
    elif case == "var_zero":
        mv[3, 1] = 0.0
    elif case == "mean_nan":
        mm[7, 0] = np.nan
    elif case == "cols":
        mm, mv = mm[:, :1], mv[:, :1]
    kw = {"n_iter_neg": {"n_iter": -1}, "step_zero": {"step": 0.0}, "weight_inf": {"weight": float("inf")}}.get(case, {})
    with pytest.raises(exc):
        G.mlpg_ms(m, v, STD, mm, mv, segment=L, **kw)
    with pytest.raises(exc):
        G.mlpg_ms_batch(m, v, STD, mm, mv, lengths=[len(m)], segment=L, **kw)
    with pytest.raises(exc):
        G.mlpg_ms_batch(np.zeros((2, 50, 6)), np.ones((2, 50, 6)), STD, mm, mv, lengths=[50, 0], segment=L, **kw)


def test_segment_none_keeps_its_refusals():
    from nnmnkwii_b200 import paramgen as G
    m, v, mm, mv = _args(n=256, L=50, T=300)
    with pytest.raises(ValueError, match="longer than the DFT length"):
        G.mlpg_ms(m, v, STD, mm, mv)
    with pytest.raises(ValueError, match="longer than the DFT length"):
        G.mlpg_ms_batch(m, v, STD, mm, mv, lengths=[len(m)], segment=None)
    _, _, mm128, mv128 = _args(n=128)
    with pytest.raises(ValueError, match="must be one of 256"):
        G.mlpg_ms(m[:100], v[:100], STD, mm128, mv128)
    # the same statistics pass the checks with a segment (and get as far as the device)
    import nnmnkwii_b200._device as dev
    calls = []
    orig = dev.require_cuda

    def stop():
        calls.append(1)
        raise RuntimeError("stop before the device")
    dev.require_cuda = stop
    try:
        with pytest.raises(RuntimeError, match="stop before the device"):
            G.mlpg_ms(m, v, STD, mm128, mv128, segment=128)
    finally:
        dev.require_cuda = orig
    assert calls


def test_gmm_mlpg_ms_segment_argument_errors():
    from sklearn.mixture import GaussianMixture

    from nnmnkwii_b200.baseline.gmm import MLPG
    rng = np.random.default_rng(0)
    X = rng.standard_normal((200, 8))
    gmm = GaussianMixture(n_components=2, covariance_type="full", random_state=0, max_iter=5).fit(X)
    good = (np.zeros((33, 2)), np.ones((33, 2)))
    with pytest.raises(ValueError, match="ms_segment needs ms"):
        MLPG(gmm, ms_segment=20)
    with pytest.raises(ValueError):
        MLPG(gmm, ms=good)  # n = 64 is not an utterance-level length
    with pytest.raises(ValueError):
        MLPG(gmm, ms=good, ms_segment=66)
    with pytest.raises(ValueError):
        MLPG(gmm, ms=good, ms_segment=21)
    with pytest.raises(TypeError):
        MLPG(gmm, ms=good, ms_segment=20.0)
    with pytest.raises(ValueError, match="diff"):
        MLPG(gmm, ms=good, ms_segment=20, diff=True)
    with pytest.raises(ValueError, match="cannot be combined"):
        MLPG(gmm, ms=good, ms_segment=20, gv=(np.ones(2), np.ones(2)))
    model = MLPG(gmm, ms=good, ms_segment=20)
    assert model.ms_segment == 20 and MLPG(gmm).ms_segment is None
    with pytest.raises(ValueError, match="modulation spectrum"):
        model.transform_em(rng.standard_normal((20, 4)))
