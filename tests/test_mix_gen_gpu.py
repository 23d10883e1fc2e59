"""Parameter generation from per-frame mixtures on the GPU (paramgen.mlpg_mixture / mlpg_mixture_batch,
`mix_gen_kernel<EPL, MODE, T>` in csrc/nnk_mix_gen.cu) against the float64 restatement tests/mix_gen_oracle.py.

* every instance (EPL 1, 2, 4, 8 x SELECT / ESTEP / OBJECTIVE x float / double) by kernel name, and the launch
  count 2 + 2 n_iter (+1 for the objective) whatever the batch;
* float64 trajectories within 1e-9 and L within 1e-10 relative of the restatement for n_iter 1, 3 and 10, on
  window sets of half-width 0 to 4, M = 1, 2, 8 and 64, T = 1, 2, H, 2H + 1, across the 32-frame tile and at
  2000 frames, single-stream and Merlin layouts, flat and padded, with zero-weight components;
* exact equalities: n_iter = 0 gives mlpg_batch of the arg-max rows (ties included) bit for bit; float32 input
  gives the float64 result of the widened input, rounded; padded = flat; repeated calls agree;
* the GMM trajectory EM (baseline.gmm.MLPG.transform_em_batch) fed through its per-frame terms;
* the objective never falls; data errors raise and never come back as NaN."""
import importlib.util
import os
import re

import numpy as np
import pytest

import mix_gen_oracle as O
import oracle.gmm_traj_em as OT
import variant_mirror as VM
from conftest import ROOT

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from nnmnkwii_b200 import _lib  # noqa: E402
from nnmnkwii_b200 import paramgen as G  # noqa: E402

_spec = importlib.util.spec_from_file_location("make_gmm_traj_golden",
                                               os.path.join(ROOT, "tests", "golden", "make_gmm_traj_golden.py"))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
SETS = MG.em_window_sets()
STD = SETS["nw3"]
BY_HALF_WIDTH = {"h0": 0, "nw2": 1, "hw2": 2, "hw3": 3, "hw4": 4, "asym": 2, "nw4": 2}
MERLIN = [(0, 60), (180, 1), (183, 1, "copy"), (184, 1)]
FAMILY = r"\bmix_gen_kernel<"


def mixture(rng, T, M, D, spread=1.0):
    lw = rng.standard_normal((T, M)) * 0.5
    mu = np.cumsum(rng.standard_normal((T, M, D)), axis=0) * 0.1 + spread * rng.standard_normal((1, M, D))
    s2 = rng.random((T, M, D)) * 0.5 + 0.1
    return lw, mu, s2


def _rel(a, b):
    a = a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)
    return float(np.abs(a.astype(np.float64) - b).max() / max(1e-300, np.abs(b).max()))


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _pad(a, lens, fill=np.nan):
    off = np.concatenate([[0], np.cumsum(lens)])
    out = np.full((len(lens), max(int(max(lens)), 1)) + a.shape[1:], fill)
    for b in range(len(lens)):
        out[b, :lens[b]] = a[off[b]:off[b + 1]]
    return out


def _check(lw, mu, s2, w, lens, n_iter, streams=None, y=None, L=None):
    """Every utterance of the flat batch against the restatement."""
    off = np.concatenate([[0], np.cumsum(lens)])
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        if a == b:
            assert not np.asarray(y[a:b]).size and np.all(L[u] == 0.0)
            continue
        want, Lw = O.mlpg_mixture(lw[a:b], mu[a:b], s2[a:b], w, n_iter, streams=streams)
        assert _rel(y[a:b], want) <= 1e-9, (u, lens[u], _rel(y[a:b], want))
        assert np.all(np.abs(L[u] - Lw) <= 1e-10 * np.abs(Lw)), (u, lens[u], L[u], Lw)


# ---- 1. every instance, by name, and the launch count ------------------------------------------------------------
def launch(D, dtype):
    """One float call with n_iter = 1 and the objective: SELECT, ESTEP, OBJECTIVE (in a child process)."""
    rng = np.random.default_rng(D)
    lw, mu, s2 = (a.astype(dtype) for a in mixture(rng, 40, 3, D))
    G.mlpg_mixture_batch(_cuda(lw), _cuda(mu), _cuda(s2), STD, n_iter=1, return_log_likelihood=True,
                         layout=G.StreamLayout(D, [(0, D // 3)]))
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def kernels():
    cases = [([D, dt], FAMILY) for D in (6, 40, 100, 187) for dt in ("float32", "float64")]
    res = VM.profiled_in_child("test_mix_gen_gpu", "launch", cases, repeats=True)
    out = {}
    for (case, _), (names, err) in zip(cases, res):
        assert err == "None", (case, err)
        out[tuple(case)] = names
    return out


def test_every_instance_is_launched_by_name(kernels):
    seen = set()
    for (D, dt), names in kernels.items():
        epl = {6: 1, 40: 2, 100: 4, 187: 8}[D]
        T = {"float32": "float", "float64": "double"}[dt]
        got = sorted(re.search(r"mix_gen_kernel<[^>]*>", s).group(0) for s in names)
        assert got == ["mix_gen_kernel<%d, %d, %s>" % (epl, mode, T) for mode in range(3)], (D, dt, names)
        seen.update(got)
    assert len(seen) == 24


@pytest.mark.parametrize("n_iter", [0, 1, 4])
@pytest.mark.parametrize("want_ll", [False, True])
def test_launch_count_does_not_depend_on_length_or_batch(n_iter, want_ll):
    rng = np.random.default_rng(n_iter)
    counts = []
    for lens in ([1], [40], [700, 0, 3, 65, 1]):
        lw, mu, s2 = mixture(rng, int(sum(lens)), 4, 9)
        n0 = _lib.launch_count()
        G.mlpg_mixture_batch(_cuda(lw), _cuda(mu), _cuda(s2), STD, lengths=lens, n_iter=n_iter,
                             return_log_likelihood=want_ll)
        counts.append(_lib.launch_count() - n0)
    assert counts == [2 + 2 * n_iter + int(want_ll)] * 3, counts


# ---- 2. against the restatement ----------------------------------------------------------------------------------
@pytest.mark.parametrize("n_iter", [1, 3, 10])
@pytest.mark.parametrize("name", list(BY_HALF_WIDTH))
def test_window_sets_and_edge_lengths_match_oracle(name, n_iter):
    w = SETS[name]
    H = BY_HALF_WIDTH[name]
    assert MG.half_width(w) == H
    rng = np.random.default_rng([sum(map(ord, name)), n_iter])
    lens = sorted({1, 2, H, 2 * H + 1, 31, 33, 95} - {0})
    lw, mu, s2 = mixture(rng, sum(lens), 8, 2 * len(w))
    lw[rng.random(lw.shape) < 0.2] = -np.inf  # zero-weight components
    lw[:, 0] = np.maximum(lw[:, 0], 0.0)
    y, L = G.mlpg_mixture_batch(lw, mu, s2, w, lengths=lens, n_iter=n_iter, return_log_likelihood=True)
    assert y.dtype == np.float64 and y.shape == (sum(lens), 2) and L.shape == (len(lens), n_iter + 1)
    _check(lw, mu, s2, w, lens, n_iter, y=y, L=L)


@pytest.mark.parametrize("n_iter", [1, 3, 10])
@pytest.mark.parametrize("M", [1, 2, 8, 64])
def test_component_counts_padded_match_oracle(M, n_iter):
    rng = np.random.default_rng([M, n_iter, 1])
    lens = [1, 5, 0, 70]
    lw, mu, s2 = mixture(rng, sum(lens), M, 9)
    y, L = G.mlpg_mixture_batch(_cuda(_pad(lw, lens)), _cuda(_pad(mu, lens)), _cuda(_pad(s2, lens)), STD,
                                lengths=lens, n_iter=n_iter, return_log_likelihood=True)
    off = np.concatenate([[0], np.cumsum(lens)])
    flat = np.concatenate([y[b, :lens[b]].cpu().numpy() for b in range(len(lens))])
    for b in range(len(lens)):
        assert not y[b, lens[b]:].any()
    _check(lw, mu, s2, STD, lens, n_iter, y=flat, L=L)
    assert off[-1] == len(flat)


def test_long_utterance_matches_oracle():
    w = SETS["hw4"]
    rng = np.random.default_rng(2000)
    lw, mu, s2 = mixture(rng, 2000, 4, 3 * len(w))
    y, L = G.mlpg_mixture_batch(_cuda(lw), _cuda(mu), _cuda(s2), w, lengths=[2000], n_iter=10,
                                return_log_likelihood=True)
    _check(lw, mu, s2, w, [2000], 10, y=y.cpu().numpy(), L=L)


@pytest.mark.parametrize("n_iter", [1, 3, 10])
def test_merlin_layout_matches_oracle(n_iter):
    rng = np.random.default_rng([187, n_iter])
    lens = [150, 3, 40]
    lw, mu, s2 = mixture(rng, sum(lens), 4, 187)
    mu[:, :, 183] = rng.random((sum(lens), 4)) > 0.5  # a vuv-like copied column
    layout = G.merlin_layout()
    y, L = G.mlpg_mixture_batch(lw, mu, s2, STD, lengths=lens, layout=layout, n_iter=n_iter,
                                return_log_likelihood=True)
    assert y.shape == (sum(lens), 63)
    _check(lw, mu, s2, STD, lens, n_iter, streams=MERLIN, y=y, L=L)
    yp, Lp = G.mlpg_mixture_batch(_pad(lw, lens), _pad(mu, lens), _pad(s2, lens), STD, lengths=lens,
                                  layout=layout, n_iter=n_iter, return_log_likelihood=True)
    off = np.concatenate([[0], np.cumsum(lens)])
    for b in range(len(lens)):
        assert np.array_equal(yp[b, :lens[b]], y[off[b]:off[b + 1]]) and not yp[b, lens[b]:].any()
    assert np.array_equal(Lp, L)


# ---- 3. exact equalities -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("merlin", [False, True])
def test_no_iteration_is_mlpg_of_the_arg_max_rows(merlin):
    rng = np.random.default_rng(30 + merlin)
    lens = [300, 1, 77]
    D = 187 if merlin else 9
    layout = G.merlin_layout() if merlin else None
    lw, mu, s2 = mixture(rng, sum(lens), 5, D)
    lw[::3, 3] = lw[::3, 1] = lw[::3].max(axis=1) + 1.0  # ties: the lower index wins
    lw[1::7, :] = 0.0                                    # every component tied
    t = np.arange(sum(lens))
    mix = np.argmax(lw, axis=1)
    want = G.mlpg_batch(_cuda(mu[t, mix]), _cuda(s2[t, mix]), STD, lengths=lens, layout=layout)
    got = G.mlpg_mixture_batch(_cuda(lw), _cuda(mu), _cuda(s2), STD, lengths=lens, layout=layout, n_iter=0)
    assert torch.equal(got, want)
    pw = G.mlpg_batch(_cuda(_pad(mu[t, mix], lens, 0.0)), _cuda(_pad(s2[t, mix], lens, 1.0)), STD, lengths=lens,
                      layout=layout)
    pg = G.mlpg_mixture_batch(_cuda(_pad(lw, lens)), _cuda(_pad(mu, lens)), _cuda(_pad(s2, lens)), STD,
                              lengths=lens, layout=layout, n_iter=0)
    assert torch.equal(pg, pw)


def test_float32_is_the_widened_float64_result_rounded():
    rng = np.random.default_rng(32)
    lens = [400, 33]
    lw, mu, s2 = (a.astype(np.float32) for a in mixture(rng, sum(lens), 6, 187))
    wide = [a.astype(np.float64) for a in (lw, mu, s2)]
    kw = dict(lengths=lens, layout=G.merlin_layout(), n_iter=5, return_log_likelihood=True)
    y64, L64 = G.mlpg_mixture_batch(*wide, STD, **kw)
    y32, L32 = G.mlpg_mixture_batch(lw, mu, s2, STD, **kw)
    assert y32.dtype == np.float32 and np.array_equal(y32, y64.astype(np.float32)) and np.array_equal(L32, L64)
    t32, Lt = G.mlpg_mixture_batch(_cuda(lw), _cuda(mu), _cuda(s2), STD, **kw)
    assert t32.dtype == torch.float32 and t32.is_cuda and np.array_equal(t32.cpu().numpy(), y32)
    assert np.array_equal(Lt, L64)


def test_batch_padded_and_repeated_calls_agree():
    rng = np.random.default_rng(33)
    lens = np.array([700, 1, 0, 64, 33, 2])
    lw, mu, s2 = mixture(rng, int(lens.sum()), 8, 12)
    args = [_cuda(a) for a in (lw, mu, s2)]
    flat, L = G.mlpg_mixture_batch(*args, SETS["nw4"], lengths=lens, n_iter=6, return_log_likelihood=True)
    padded, Lp = G.mlpg_mixture_batch(*[_cuda(_pad(a, lens)) for a in (lw, mu, s2)], SETS["nw4"], lengths=lens,
                                      n_iter=6, return_log_likelihood=True)
    off = np.concatenate([[0], np.cumsum(lens)])
    for b in range(len(lens)):
        a, e = off[b], off[b + 1]
        assert torch.equal(padded[b, :lens[b]], flat[a:e]) and not padded[b, lens[b]:].any(), b
        if lens[b]:
            one, L1 = G.mlpg_mixture(*[x[a:e] for x in args], SETS["nw4"], n_iter=6, return_log_likelihood=True)
            assert _rel(flat[a:e], one.cpu().numpy()) <= 1e-12, b
            assert np.all(np.abs(L[b] - L1) <= 1e-12 * np.abs(L1)), b
    assert np.array_equal(Lp, L)
    for _ in range(3):
        again, La = G.mlpg_mixture_batch(*args, SETS["nw4"], lengths=lens, n_iter=6, return_log_likelihood=True)
        assert torch.equal(again, flat) and np.array_equal(La, L)


# ---- 4. the GMM trajectory EM through its per-frame terms --------------------------------------------------------
@pytest.mark.parametrize("name", ["nw2", "nw3", "h0"])
def test_gmm_terms_give_transform_em(name):
    from nnmnkwii_b200.baseline.gmm import MLPG
    w = SETS[name]
    S, M = 3, 6
    rng = np.random.default_rng(sum(map(ord, name)) + 2)
    g = MG.joint_gmm(rng, M, S * len(w))
    model = OT.Model(g, w)
    srcs = [rng.standard_normal((T, S * len(w))) for T in (60, 1, 200)]
    want, Lw = MLPG(g, windows=w).transform_em_batch(srcs, n_iter=5, return_log_likelihood=True)
    terms = [model.frame_terms(s) for s in srcs]
    lw = np.concatenate([lp for lp, _ in terms])
    mu = np.concatenate([E.transpose(1, 0, 2) for _, E in terms])
    s2 = np.broadcast_to(model.Dm, mu.shape)
    y, L = G.mlpg_mixture_batch(lw, mu, s2, w, lengths=[len(s) for s in srcs], n_iter=5,
                                return_log_likelihood=True)
    off = np.concatenate([[0], np.cumsum([len(s) for s in srcs])])
    for u in range(len(srcs)):
        assert _rel(y[off[u]:off[u + 1]], want[u]) <= 1e-9, u
        assert np.all(np.abs(L[u] - Lw[u]) <= 1e-9 * np.abs(Lw[u])), u


# ---- 5. the objective and data errors ----------------------------------------------------------------------------
def test_objective_never_decreases():
    rng = np.random.default_rng(34)
    lens = [500, 37]
    lw, mu, s2 = mixture(rng, sum(lens), 8, 9, spread=0.3)
    _, L = G.mlpg_mixture_batch(lw, mu, s2, STD, lengths=lens, n_iter=20, return_log_likelihood=True)
    # the device sums 32-frame partials in a fixed order: a converged step may round below the last value by a
    # few units in the last place of the partial sums
    assert np.all(np.diff(L, axis=1) >= -1e-13 * np.abs(L[:, :-1])), np.diff(L, axis=1).min()
    assert np.all(L[:, -1] > L[:, 0])


@pytest.mark.parametrize("case", ["lw_nan", "lw_posinf", "lw_all_neginf", "s2_zero", "s2_neg", "s2_nan", "s2_inf",
                                  "s2_zero_unused_component"])
def test_data_errors_raise(case):
    rng = np.random.default_rng(35)
    lens = [50, 20]
    lw, mu, s2 = mixture(rng, 70, 4, 9)
    row = 57
    if case == "lw_nan":
        lw[row, 2] = np.nan
    elif case == "lw_posinf":
        lw[row, 0] = np.inf
    elif case == "lw_all_neginf":
        lw[row] = -np.inf
    elif case == "s2_zero":
        s2[row, 1, 4] = 0.0
    elif case == "s2_neg":
        s2[row, 3, 0] = -1.0
    elif case == "s2_nan":
        s2[row, 0, 8] = np.nan
    elif case == "s2_inf":
        s2[row, 2, 3] = np.inf
    elif case == "s2_zero_unused_component":
        lw[row, 1] = -np.inf
        s2[row, 1, 2] = 0.0
    for n_iter in (0, 3):
        with pytest.raises(ValueError, match="frame 7 of utterance 1"):
            G.mlpg_mixture_batch(_cuda(lw), _cuda(mu), _cuda(s2), STD, lengths=lens, n_iter=n_iter,
                                 return_log_likelihood=True)


def test_columns_no_chain_reads_are_not_checked():
    rng = np.random.default_rng(36)
    lw, mu, s2 = mixture(rng, 40, 3, 10)  # three windows of 3 static columns: column 9 takes no part
    y = G.mlpg_mixture(lw, mu, s2, STD, n_iter=3)
    mu[:, :, 9], s2[:, :, 9] = np.nan, -1.0
    assert np.array_equal(G.mlpg_mixture(lw, mu, s2, STD, n_iter=3), y)
    _check(lw, mu[:, :, :9], s2[:, :, :9], STD, [40], 3, y=y, L=G.mlpg_mixture(lw, mu, s2, STD, n_iter=3,
                                                                                   return_log_likelihood=True)[1][None])
