"""GPU: baseline.gmm.GaussianMixture (EM in csrc/nnk_gmm_em.cu) against scikit-learn's GaussianMixture run
live on the same float64 data."""
import pickle
import warnings

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _blobs(N, D, K, seed, zero_frac=0.0):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((K, D)) * 3.0
    scales = rng.uniform(0.3, 1.5, (K, D))
    lab = rng.integers(0, K, N)
    X = centres[lab] + rng.standard_normal((N, D)) * scales[lab]
    X[:, 0] += 20.0  # an energy-like dimension with |mu| >> sigma
    if zero_frac:
        X[rng.random(N) < zero_frac] = 0.0  # zero-padded frames, as the aligner's joint matrix has
    return X


def _fit_both(X, fit_X=None, **kw):
    from sklearn.mixture import GaussianMixture as Sk

    from nnmnkwii_b200.baseline.gmm import GaussianMixture
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        a = Sk(**kw)
        la = a.fit_predict(X)
        b = GaussianMixture(**kw)
        lb = b.fit_predict(X if fit_X is None else fit_X)
    return a, la, b, lb


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(1e-300, np.abs(np.asarray(a)).max()))


def _assert_same_fit(a, la, b, lb, tol=1e-8):
    assert b.n_iter_ == a.n_iter_ and b.converged_ == a.converged_
    assert np.array_equal(np.asarray(lb), la)
    assert len(b.lower_bounds_) == len(a.lower_bounds_)
    assert np.allclose(b.lower_bounds_, a.lower_bounds_, rtol=1e-10, atol=0)
    for name in ("weights_", "means_", "covariances_", "precisions_cholesky_", "precisions_"):
        got = getattr(b, name)
        assert isinstance(got, np.ndarray) and got.dtype == np.float64, name
        assert _rel(getattr(a, name), got) < tol, (name, _rel(getattr(a, name), got))


def test_one_em_step_from_given_parameters():
    from sklearn.mixture import GaussianMixture as Sk
    X = _blobs(3000, 6, 3, 1)
    ref = Sk(n_components=3, random_state=0, max_iter=5).fit(X)
    kw = dict(n_components=3, max_iter=1, weights_init=ref.weights_, means_init=ref.means_,
              precisions_init=ref.precisions_)
    a, la, b, lb = _fit_both(X, **kw)
    for name in ("weights_", "means_", "covariances_", "precisions_cholesky_"):
        assert _rel(getattr(a, name), getattr(b, name)) < 1e-10, name
    assert abs(a.lower_bound_ - b.lower_bound_) <= 1e-10 * abs(a.lower_bound_)
    assert np.array_equal(la, lb)


@pytest.mark.parametrize("N,D,K,zero_frac,max_iter", [(5000, 8, 4, 0.0, 100), (20000, 50, 16, 0.15, 20),
                                                       (8000, 72, 32, 0.0, 20)])
def test_full_fit_matches_sklearn(N, D, K, zero_frac, max_iter):
    X = _blobs(N, D, K, 2, zero_frac)
    _assert_same_fit(*_fit_both(X, n_components=K, init_params="kmeans", random_state=0, max_iter=max_iter))


@pytest.mark.parametrize("init", ["k-means++", "random", "random_from_data"])
def test_other_initialisers(init):
    X = _blobs(4000, 5, 4, 3)
    _assert_same_fit(*_fit_both(X, n_components=4, init_params=init, random_state=0, max_iter=30))


def test_n_init_and_warm_start():
    from sklearn.mixture import GaussianMixture as Sk

    from nnmnkwii_b200.baseline.gmm import GaussianMixture
    X = _blobs(4000, 5, 4, 4)
    _assert_same_fit(*_fit_both(X, n_components=4, n_init=3, random_state=0, max_iter=30))
    a = Sk(n_components=4, warm_start=True, max_iter=3, random_state=0)
    b = GaussianMixture(n_components=4, warm_start=True, max_iter=3, random_state=0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for _ in range(3):
            a.fit(X)
            b.fit(X)
            assert b.n_iter_ == a.n_iter_
            assert _rel(a.means_, b.means_) < 1e-9 and _rel(a.covariances_, b.covariances_) < 1e-9


def test_float32_and_cuda_tensor_inputs():
    import torch
    X = _blobs(4000, 6, 3, 5).astype(np.float32)
    X64 = X.astype(np.float64)
    a, la, b, lb = _fit_both(X64, fit_X=X, n_components=3, random_state=0)
    _assert_same_fit(a, la, b, lb)
    for t in (torch.from_numpy(X).cuda(), torch.from_numpy(X64).cuda()):
        _, _, c, lc = _fit_both(X64, fit_X=t, n_components=3, random_state=0)
        assert isinstance(lc, torch.Tensor) and lc.is_cuda
        assert np.array_equal(lc.cpu().numpy(), lb)
        for name in ("weights_", "means_", "covariances_", "precisions_cholesky_"):
            assert np.array_equal(getattr(c, name), getattr(b, name)), name


def test_fits_are_bit_identical():
    from nnmnkwii_b200.baseline.gmm import GaussianMixture
    X = _blobs(20000, 20, 8, 6)
    fits = [GaussianMixture(n_components=8, random_state=0, max_iter=10, tol=0).fit(X) for _ in range(2)]
    for name in ("weights_", "means_", "covariances_", "precisions_cholesky_", "lower_bounds_"):
        assert np.array_equal(getattr(fits[0], name), getattr(fits[1], name)), name


def test_collapsed_component_raises_sklearn_error():
    from nnmnkwii_b200.baseline.gmm import GaussianMixture
    X = np.repeat(_blobs(3, 4, 1, 7), 200, axis=0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(ValueError, match="ill-defined empirical covariance"):
            GaussianMixture(n_components=3, reg_covar=0.0, random_state=0).fit(X)
    # the library is still usable afterwards
    GaussianMixture(n_components=2, random_state=0).fit(_blobs(500, 4, 2, 8))


def test_size_limits_raise_before_any_launch():
    import torch

    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200.baseline.gmm import GaussianMixture
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match="at most 128 features"):
        GaussianMixture(n_components=2).fit(np.random.default_rng(0).standard_normal((300, 129)))
    with pytest.raises(ValueError, match="at most 128 components"):
        GaussianMixture(n_components=129).fit(np.random.default_rng(0).standard_normal((300, 3)))
    with pytest.raises(NotImplementedError):
        GaussianMixture(n_components=2, covariance_type="diag").fit(np.random.default_rng(0).standard_normal((300, 3)))
    with pytest.raises(ValueError, match="n_samples >= n_components"):
        GaussianMixture(n_components=5).fit(np.random.default_rng(0).standard_normal((4, 3)))
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0
    assert _lib.lib.nnk_gmm_em_workspace_bytes(1000, 129, 4) == 0


def test_fitted_object_in_use():
    from sklearn.mixture import GaussianMixture as Sk

    from nnmnkwii_b200.baseline.gmm import MLPG, GaussianMixture
    rng = np.random.default_rng(9)
    X = _blobs(6000, 8, 4, 9)  # joint static+delta source / target, 2 x (2 x 2)
    kw = dict(n_components=4, random_state=0)
    a = Sk(**kw).fit(X)
    b = GaussianMixture(**kw).fit(X)
    src = rng.standard_normal((50, 4)) + X[:50, :4]
    ya = MLPG(a).transform(src)
    yb = MLPG(b).transform(src)
    assert np.abs(ya - yb).max() <= 1e-9 * max(1.0, np.abs(ya).max())
    assert np.allclose(b.predict_proba(X[:100]), a.predict_proba(X[:100]), rtol=1e-8, atol=1e-12)
    assert abs(b.score(X) - a.score(X)) < 1e-9 * abs(a.score(X))
    assert np.isfinite(b.bic(X))
    assert b.sample(10)[0].shape == (10, 8)
    c = pickle.loads(pickle.dumps(b))
    assert np.array_equal(c.predict(X[:100]), b.predict(X[:100]))


def _aligner_pairs(n, T, D, seed):
    rng = np.random.default_rng(seed)
    X = np.zeros((n, T, D))
    Y = np.zeros((n, T, D))
    for i in range(n):
        tx, ty = rng.integers(T * 3 // 4, T + 1, 2)
        x = np.cumsum(rng.standard_normal((tx, D)), 0) * 0.3
        X[i, :tx] = x
        idx = np.minimum(np.arange(ty) * tx // ty, tx - 1)
        Y[i, :ty] = x[idx] + 0.05 * rng.standard_normal((ty, D))
    return X, Y


@pytest.mark.parametrize("n,T,D", [(3, 40, 4), (32, 800, 25)])
def test_iterative_aligner_device_gmm(n, T, D):
    from nnmnkwii_b200.preprocessing.alignment import IterativeDTWAligner
    X, Y = _aligner_pairs(n, T, D, 10)
    kw = dict(n_iter=2, n_components_gmm=4, random_state=0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        Xa, Ya = IterativeDTWAligner(**kw).transform((X, Y))
        Xb, Yb = IterativeDTWAligner(gmm="device", **kw).transform((X, Y))
    assert Xb.shape == Xa.shape and Xb.dtype == Xa.dtype
    assert np.allclose(Xb, Xa, rtol=1e-9, atol=1e-12) and np.allclose(Yb, Ya, rtol=1e-9, atol=1e-12)
    with pytest.raises(ValueError):
        IterativeDTWAligner(gmm="cpu")
