"""Every kernel instance the GMM EM launchers (csrc/nnk_gmm_em.cu) and the GMM mapping launchers
(csrc/nnk_gmm.cu) can select, against float64 references.

EM: `estep_d` picks `em_estep_kernel<EPL, T>` with EPL = ceil(D / 32) and `mstep_d` picks
`em_cov_kernel<TI, T>` with TI = ceil(D / 16); T is the dtype of X.  A whole fit compounds last-bit
differences over iterations and through label ties, so each case drives `baseline.gmm._EmState` (the object
`fit_predict` uses) one kernel step at a time from given responsibilities and parameters, and compares every
step with scikit-learn 1.9's own float64 helpers (`_estimate_gaussian_parameters`,
`_compute_precision_cholesky`, `_estimate_log_gaussian_prob`, `_logsumexp`), called live.  Shapes come from
`variant_mirror` and each case asserts, from the profiler, the instance the mirror predicts.

Mapping: `gmm_logprob_kernel`, `gmm_select_kernel` (mode 0) and `gmm_posterior_kernel` (mode 1) against
the reference's per-frame algebra written out in NumPy float64 (`gmm_map_reference`)."""
import ctypes
import types
import warnings

import numpy as np
import pytest

import variant_mirror as M
from conftest import rel_err

pytestmark = pytest.mark.gpu

REG_COVAR = 1e-6
# above this condition number a float64 Cholesky (LAPACK's or the kernel's) carries more than ~1e-10 of
# rounding whatever the order of its sums; such cases are judged against a long-double factorisation
ILL_CONDITIONED = 1e5


def _rel(a, b):
    """max |a - b| / max |a| (the one-step bar of tests/test_gmm_fit_gpu.py)."""
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(1e-300, np.abs(np.asarray(a)).max()))


def _host(t):
    return t.detach().cpu().numpy().astype(np.float64)


# ---- references ------------------------------------------------------------------------------------------------
def em_mstep_reference(X, resp, reg_covar):
    """(nk, weights after mstep(0), weights after mstep(1), means, covariances, precisions_cholesky)."""
    from sklearn.mixture._gaussian_mixture import _compute_precision_cholesky, _estimate_gaussian_parameters
    nk, means, cov = _estimate_gaussian_parameters(X, resp, reg_covar, "full")
    return nk, nk / X.shape[0], nk / np.sum(nk), means, cov, _compute_precision_cholesky(cov, "full")


def em_estep_reference(X, weights, means, prec_chol):
    """(resp, lower_bound) of sklearn's _e_step on the given parameters."""
    from sklearn.mixture._gaussian_mixture import _estimate_log_gaussian_prob
    from sklearn.utils._array_api import _logsumexp
    lp = _estimate_log_gaussian_prob(X, means, prec_chol, "full") + np.log(weights)
    lse = _logsumexp(lp, axis=1)
    return np.exp(lp - lse[:, np.newaxis]), float(np.mean(lse))


def prec_chol_longdouble(cov):
    """L^-T with C = L L^T per component, in long double (right-looking Cholesky, forward substitution)."""
    C = np.asarray(cov, dtype=np.longdouble)
    K, D, _ = C.shape
    L = np.zeros_like(C)
    for j in range(D):
        L[:, j, j] = np.sqrt(C[:, j, j] - np.einsum("kc,kc->k", L[:, j, :j], L[:, j, :j]))
        L[:, j + 1:, j] = ((C[:, j + 1:, j] - np.einsum("krc,kc->kr", L[:, j + 1:, :j], L[:, j, :j]))
                           / L[:, j, j][:, None])
    Z = np.zeros_like(C)
    eye = np.eye(D, dtype=np.longdouble)
    for r in range(D):
        Z[:, r, :] = (eye[r] - np.einsum("kc,kcj->kj", L[:, r, :r], Z[:, :r, :])) / L[:, r, r][:, None]
    return Z.transpose(0, 2, 1)


def gmm_map_reference(base, src):
    """The reference's per-frame algebra (gmm.py:97-121, 219-244) in NumPy float64, one `solve` per
    mixture: (lp (T, M), Em (T, M, D) the per-mixture means, post-mean E (T, D), Dm (M, D))."""
    from scipy.special import logsumexp
    T, dim = src.shape
    Mx = base.num_mixtures
    lp = np.empty((T, Mx))
    Em = np.empty((T, Mx, dim))
    for m in range(Mx):
        d = src - base.src_means[m]
        sol = np.linalg.solve(base.covarXX[m], d.T).T
        lp[:, m] = (np.log(base.weights[m]) - 0.5 * (d * sol).sum(1) - 0.5 * np.linalg.slogdet(base.covarXX[m])[1]
                    - 0.5 * dim * np.log(2 * np.pi))
        Em[:, m] = base.tgt_means[m] + sol @ base.covarYX[m].T
    post = np.exp(lp - logsumexp(lp, axis=1, keepdims=True))
    E = np.einsum("tm,tmi->ti", post, Em)
    Dm = np.stack([np.diag(base.covarYY[m]) - np.diag(base.covarYX[m]) / np.diag(base.covarXX[m]) * np.diag(base.covarXY[m])
                   for m in range(Mx)])
    return lp, Em, E, Dm


# ---- EM: one kernel step at a time -------------------------------------------------------------------------------
def _em_data(N, D, K, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, D)) * rng.uniform(0.5, 2.0, D) + rng.standard_normal(D)
    X[:, 0] += 20.0  # an energy-like dimension with |mu| >> sigma
    resp = rng.dirichlet(np.ones(K), size=N)
    if K > 1:
        resp[:, K // 2] *= 1e-9  # a component with almost no mass
    return X, resp


def _frames(X, dtype, pad=0):
    """X on the device in `dtype`; with pad > 0 a column slice of a wider tensor (x_ld = D + pad)."""
    import torch
    N, D = X.shape
    wide = torch.full((N, D + pad), 7.0, dtype=dtype, device="cuda")
    wide[:, :D] = torch.from_numpy(X).to(dtype)
    return wide[:, :D]


def _type(dtype):
    import torch
    return "float" if dtype == torch.float32 else "double"


def _expect(fn, instance, family):
    """``fn()`` (repeatable) ran `instance`, and no other kernel of `family`.  The profile is taken with
    `family` itself, so a profile that lost the records of that kernel is repeated (`M.profiled`)."""
    _, err, names = M.profiled(fn, family)
    assert err is None, err
    got = set(M.launched(names, family))
    assert got and all(instance in n for n in got), (instance, sorted(got))


def _check_estep(st, X64):
    resp, lb = em_estep_reference(X64, _host(st.weights), _host(st.means), _host(st.prec_chol))
    assert np.abs(_host(st.resp) - resp).max() < 1e-10
    assert abs(float(st.lower_bound.item()) - lb) <= 1e-12 * abs(lb), (float(st.lower_bound.item()), lb)


def _check_factor(st, cov, pc):
    """precisions_cholesky of `cov` (sklearn's covariances) against sklearn's `pc`."""
    cond = np.linalg.cond(cov)
    if cond.max() <= ILL_CONDITIONED:
        assert _rel(pc, _host(st.prec_chol)) < 1e-10, _rel(pc, _host(st.prec_chol))
        return
    # fewer frames than features: the factors of both are rounding-bound (cond ~ 1e7 - 1e8).  Factor sklearn's own
    # covariances on the device and judge both factorisations against long double, on the worst components
    st.put("covariances", cov)
    st.factor(True)
    st.check_status()
    worst = np.argsort(cond)[-8:]
    truth = prec_chol_longdouble(cov[worst])
    e_dev = _rel(truth, _host(st.prec_chol)[worst])
    e_lapack = _rel(truth, pc[worst])
    assert e_dev <= max(1e-10, 4 * e_lapack), (e_dev, e_lapack, cond.max())


def _em_step_case(N, D, K, dtype, pad=0):
    """mstep(0), mstep(1), factor(True), estep(), then factor(False) + estep() from given parameters,
    each against sklearn; asserts the predicted em_cov / em_estep instances.  Returns the _EmState."""
    from nnmnkwii_b200.baseline.gmm import _EmState
    X, resp = _em_data(N, D, K, seed=N * 1009 + D * 31 + K)
    Xd = _frames(X, dtype, pad)
    X64 = _host(Xd)  # float32 frames widened, as the kernels read them
    T = _type(dtype)
    st = _EmState(Xd, K, REG_COVAR)
    assert st.args.x_ld == D + pad
    st.put("resp", resp)
    nk, w0, w1, means, cov, pc = em_mstep_reference(X64, resp, REG_COVAR)

    _expect(lambda: st.mstep(0), "em_cov_kernel<%d, %s>" % (M.em_cov_ti(D), T), r"\bem_cov_kernel<")
    _expect(lambda: st.mstep(0), "em_stats_kernel<%s>" % T, r"\bem_stats_kernel<")
    assert _rel(w0, _host(st.weights)) < 1e-10
    st.mstep(1)
    for name, want in (("weights", w1), ("means", means), ("covariances", cov)):
        assert _rel(want, _host(getattr(st, name))) < 1e-10, (name, _rel(want, _host(getattr(st, name))))
    st.factor(True)
    st.check_status()
    _check_factor(st, cov, pc)

    _expect(st.estep, "em_estep_kernel<%d, %s>" % (M.em_estep_epl(D), T), r"\bem_estep_kernel<")
    _check_estep(st, X64)

    # factor(False): the E-step constants from given precisions, means and weights
    rng = np.random.default_rng(K)
    st.put("prec_chol", pc * rng.uniform(0.8, 1.25, (K, 1, 1)))
    st.put("means", means + 0.1 * rng.standard_normal(means.shape))
    st.put("weights", rng.dirichlet(np.ones(K)))
    st.factor(False)
    st.estep()
    _check_estep(st, X64)
    return st


_D_EDGES = [1, 16, 17, 32, 33, 48, 49, 64, 65, 80, 81, 96, 97, 112, 113, 127, 128]
_K_EDGES = [1, 31, 32, 33, 64, 128]
_DK = [(D, _K_EDGES[i % len(_K_EDGES)]) for i, D in enumerate(_D_EDGES)]


def _dtypes():
    import torch
    return {"float64": torch.float64, "float32": torch.float32}


@pytest.mark.parametrize("dtype", ["float64", "float32"])
@pytest.mark.parametrize("D,K", _DK, ids=["D%d_K%d" % dk for dk in _DK])
def test_em_step_every_instance(D, K, dtype):
    """Both sides of every EPL (32, 64, 96) and TI (16, 32, ..., 112) boundary, every K edge."""
    _em_step_case(4 * D + 333, D, K, _dtypes()[dtype])


@pytest.mark.parametrize("dtype", ["float64", "float32"])
@pytest.mark.parametrize("N", [2000, 128, 20])
def test_em_step_at_the_size_limits(N, dtype):
    """D = K = 128: the largest dynamic shared memory of the statistics, E-step and factor kernels
    (opt-in on sm_90a: 227 KB); N = K and a single partial E-step tile (N < 32)."""
    D = K = 128
    assert M.em_stats_smem(D, K) == 197632 and M.em_factor_smem(D) == 133120
    assert max(M.em_estep_smem(D, K), M.em_cov_smem(D)) <= 232448
    _em_step_case(N, D, K, _dtypes()[dtype])


@pytest.mark.parametrize("N", [31, 32, 33, 1024, 1025])
def test_em_step_tile_and_chunk_tails(N):
    """E-step tiles of 32 frames, statistics chunks of 1024; D = 20 is TI = 2."""
    L = M.em_layout(N, 20, 3)
    assert L["n_tiles"] == (N + 31) // 32 and L["n_stat"] == (N + 1023) // 1024
    _em_step_case(N, 20, 3, _dtypes()["float64"])


def _cov_chunk_shapes(D, K):
    """The largest N with a single covariance chunk, and the smallest N >= 1000 with several chunks whose
    last one is short and ends inside a 32-frame sub-tile."""
    single = max(N for N in range(1, 2000) if M.em_layout(N, D, K)["n_cov"] == 1)
    for N in range(1000, 5000):
        L = M.em_layout(N, D, K)
        tail = N - (L["n_cov"] - 1) * L["cov_chunk"]
        if L["n_cov"] > 1 and tail < L["cov_chunk"] and tail % M.EM_CV_SUB:
            return single, N
    raise AssertionError("no shape with a covariance-chunk tail")


@pytest.mark.parametrize("D,K", [(20, 3), (40, 33)])
def test_em_step_covariance_chunks(D, K):
    single, several = _cov_chunk_shapes(D, K)
    assert M.em_layout(single + 1, D, K)["n_cov"] > 1
    for N in (single, several):
        _em_step_case(N, D, K, _dtypes()["float64"])


@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_em_strided_frames_are_bit_identical(dtype):
    """x_ld > D (a column slice of a wider tensor, which `_as_frames` keeps) gives the same bits as the
    same frames made contiguous: through `_EmState` and through a whole `GaussianMixture.fit`."""
    import torch

    from nnmnkwii_b200.baseline.gmm import GaussianMixture, _as_frames, _EmState
    N, D, K = 1025, 20, 4
    X, resp = _em_data(N, D, K, seed=11)
    Xs = _frames(X, _dtypes()[dtype], pad=9)
    Xc = Xs.contiguous()
    assert Xs.stride(0) == D + 9 and _as_frames(Xs)[0].data_ptr() == Xs.data_ptr()
    outs = []
    for Xd in (Xs, Xc):
        st = _EmState(Xd, K, REG_COVAR)
        st.put("resp", resp)
        st.mstep(0)
        st.mstep(1)
        st.factor(True)
        st.estep()
        torch.cuda.synchronize()
        outs.append([getattr(st, n).clone() for n in ("resp", "weights", "means", "covariances", "prec_chol",
                                                      "lower_bound")])
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    fits = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for Xd in (Xs, Xc):
            fits.append(GaussianMixture(n_components=K, random_state=0, max_iter=5, tol=0).fit(Xd))
    for name in ("weights_", "means_", "covariances_", "precisions_cholesky_", "lower_bounds_"):
        assert np.array_equal(getattr(fits[0], name), getattr(fits[1], name)), name


@pytest.mark.parametrize("N,D,K", [(20000, 72, 64), (8000, 100, 8)])
def test_em_fit_at_voice_conversion_size(N, D, K):
    """The VC workload of tools/bench_gmm.py (72 dims, 64 components, several components per lane) and a
    fit with EPL = 4 / TI = 7, whole fits against scikit-learn under the bar of tests/test_gmm_fit_gpu.py."""
    from test_gmm_fit_gpu import _assert_same_fit, _blobs, _fit_both
    X = _blobs(N, D, K, 12)
    _assert_same_fit(*_fit_both(X, n_components=K, init_params="kmeans", random_state=0, max_iter=10))


# ---- mapping kernels ------------------------------------------------------------------------------------------------
def _joint_gmm(Mx, dim, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((Mx, 2 * dim, 2 * dim)) / np.sqrt(2 * dim)
    cov = A @ A.transpose(0, 2, 1) + 0.5 * np.eye(2 * dim)
    w = rng.random(Mx) + 0.1
    return types.SimpleNamespace(means_=rng.standard_normal((Mx, 2 * dim)), covariances_=cov, weights_=w / w.sum(),
                                 covariance_type="full")


def _map_with_mix(base, x, mode):
    """`nnk_gmm_logprob` + `nnk_gmm_map` through ctypes with a `mix` buffer: (lp, E, Dv, mix) on the host."""
    import torch

    from nnmnkwii_b200 import _device as dev
    from nnmnkwii_b200 import _lib
    c = base._constants()
    T, D = x.shape
    f64 = dict(dtype=torch.float64, device=x.device)
    lp = base._weighted_log_prob(x, c)
    E = torch.empty((T, D), **f64)
    Dv = torch.empty((T, D), **f64) if mode == 0 else None
    mix = torch.full((T,), -1, dtype=torch.int32, device=x.device)
    _lib.check(_lib.lib.nnk_gmm_map(ctypes.byref(c["gmm"]), x.data_ptr(), x.stride(0), T, lp.data_ptr(), mode,
                                    E.data_ptr(), Dv.data_ptr() if Dv is not None else None, mix.data_ptr(),
                                    dev.current_stream_ptr(x.device)), "nnk_gmm_map")
    torch.cuda.synchronize()
    return (lp.cpu().numpy(), E.cpu().numpy(), Dv.cpu().numpy() if Dv is not None else None,
            mix.cpu().numpy().astype(np.int64))


def _check_mapping(base, src, pad=0):
    lp_ref, Em, E_ref, Dm = gmm_map_reference(base, src)
    T = src.shape[0]
    x = _frames(src, _dtypes()["float64"], pad)
    _, err, _ = M.profiled(lambda: base._weighted_log_prob(x, base._constants()), r"\bgmm_logprob_kernel\b")
    assert err is None, err
    (lp, E0, Dv, mix), err, _ = M.profiled(lambda: _map_with_mix(base, x, 0), r"\bgmm_select_kernel\b")
    assert err is None, err
    assert rel_err(lp, lp_ref) < 1e-9
    assert np.array_equal(mix, lp.argmax(1)) and np.array_equal(mix, lp_ref.argmax(1))
    assert rel_err(E0, Em[np.arange(T), mix]) < 1e-9
    assert np.array_equal(Dv, Dm[mix])
    (_, E1, _, mix1), err, _ = M.profiled(lambda: _map_with_mix(base, x, 1), r"\bgmm_posterior_kernel\b")
    assert err is None, err
    assert rel_err(E1, E_ref) < 1e-9
    assert np.all(mix1 == -1)  # mode 1 writes no mixture index
    return lp, E0, Dv, mix, E1


_MAP_M = [1, 31, 32, 33, 64, 65, 128]
_MAP_D = [1, 31, 32, 33, 64, 65, 95, 96]
_MAP_T = [1, 3, 4, 5, 15, 16, 17, 333]
_MAP_CASES = [(_MAP_M[i % len(_MAP_M)], _MAP_D[i], _MAP_T[(3 * i) % len(_MAP_T)]) for i in range(len(_MAP_D))]


@pytest.mark.parametrize("Mx,D,T", _MAP_CASES, ids=["M%d_D%d_T%d" % c for c in _MAP_CASES])
def test_mapping_kernels(Mx, D, T):
    """Every M edge (components per lane in the arg-max and the softmax), every D edge up to the 96 limit,
    tails of the 16-frame (log-prob, posterior) and 4-frame (select) tiles."""
    from nnmnkwii_b200.baseline.gmm import MLPGBase
    assert D <= M.GMM_MAX_D
    base = MLPGBase(_joint_gmm(Mx, D, Mx * 1000 + D))
    src = np.random.default_rng(T).standard_normal((T, D)) + base.src_means[T % Mx]
    _check_mapping(base, src)


def test_mapping_every_axis_value_is_covered():
    assert {c[0] for c in _MAP_CASES} == set(_MAP_M)
    assert {c[1] for c in _MAP_CASES} == set(_MAP_D)
    assert {c[2] for c in _MAP_CASES} == set(_MAP_T)


def test_mapping_arg_max_ties_take_the_first_index():
    """Duplicated components tie exactly: 8 / 40 sit on the same lane, 31 / 64 on different lanes with the
    larger index on the lower lane.  The kernel must return NumPy's first index."""
    from nnmnkwii_b200.baseline.gmm import MLPGBase
    Mx, dim = 70, 6
    g = _joint_gmm(Mx, dim, 5)
    w = np.full(Mx, 0.2 / Mx)
    for lo, hi in ((8, 40), (31, 64)):
        g.means_[hi] = g.means_[lo]
        g.covariances_[hi] = g.covariances_[lo]
        w[lo] = w[hi] = 0.2
    g.weights_ = w / w.sum()
    base = MLPGBase(g)
    rng = np.random.default_rng(6)
    src = np.concatenate([base.src_means[8] + 0.1 * rng.standard_normal((9, dim)),
                          base.src_means[31] + 0.1 * rng.standard_normal((10, dim))])
    lp, _, _, mix, _ = _check_mapping(base, src)
    assert np.array_equal(lp[:, 8], lp[:, 40]) and np.array_equal(lp[:, 31], lp[:, 64])
    assert np.array_equal(mix, np.array([8] * 9 + [31] * 10))


@pytest.mark.parametrize("pad", [1, 13])
def test_mapping_strided_frames_are_bit_identical(pad):
    """x_ld > D through the C ABI gives the same bits as contiguous frames."""
    from nnmnkwii_b200.baseline.gmm import MLPGBase
    base = MLPGBase(_joint_gmm(33, 40, 7))
    src = np.random.default_rng(8).standard_normal((37, 40)) + base.src_means[0]
    contiguous = _check_mapping(base, src)
    strided = _check_mapping(base, src, pad=pad)
    for a, b in zip(contiguous, strided):
        assert np.array_equal(a, b)


def test_mapping_beyond_96_dims_raises_before_any_launch():
    import torch

    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200.baseline.gmm import MLPG, MLPGBase
    g = _joint_gmm(2, M.GMM_MAX_D + 1, 9)
    src = np.zeros((5, M.GMM_MAX_D + 1))
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with pytest.raises(NotImplementedError, match="96"):
        MLPGBase(g).transform(src)
    conv = MLPG(g, windows=[(0, 0, np.array([1.0]))])
    conv.static_dim = 1  # the E / D (arg-max) path
    with pytest.raises(NotImplementedError, match="96"):
        conv.transform(src)
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0
