"""GPU: the device k-means initialisation of baseline.gmm.GaussianMixture (csrc/nnk_kmeans.cu) against
scikit-learn 1.9's KMeans / kmeans_plusplus run live on the same float64 data (float32 frames widened)."""
import warnings

import numpy as np
import pytest

from test_gmm_fit_gpu import _aligner_pairs, _assert_same_fit, _blobs, _fit_both, _rel
from test_gmm_kmeans_cpu import km_epl, km_layout

pytestmark = pytest.mark.gpu


def _frames(X, dtype=None, pad=0):
    import torch
    dtype = dtype or torch.float64
    N, D = X.shape
    wide = torch.full((N, D + pad), 7.0, dtype=dtype, device="cuda")
    wide[:, :D] = torch.from_numpy(X).to(dtype)
    return wide[:, :D]


def _host(t):
    return t.detach().cpu().numpy()


def _sk_kmeans(X, K, **kw):
    from sklearn.cluster import KMeans
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return KMeans(n_clusters=K, n_init=1, **kw).fit(X)


def _dev_kmeans(Xd, K, **kw):
    from nnmnkwii_b200.baseline.gmm import _device_kmeans
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return _device_kmeans(Xd, K, **kw)


def _assert_same_kmeans(ref, got, inertia_atol=0.0):
    labels, centers, inertia, n_iter = got
    assert n_iter == ref.n_iter_
    assert np.array_equal(_host(labels), ref.labels_)
    assert _rel(ref.cluster_centers_, _host(centers)) < 1e-10, _rel(ref.cluster_centers_, _host(centers))
    assert abs(inertia - ref.inertia_) <= 1e-10 * abs(ref.inertia_) + inertia_atol, (inertia, ref.inertia_)


# ---- seeding -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,D,K,zero_frac", [(3000, 8, 4, 0.0), (20000, 50, 16, 0.15), (8000, 72, 32, 0.0)])
def test_seeding_matches_kmeans_plusplus(N, D, K, zero_frac):
    import torch
    from sklearn.cluster import kmeans_plusplus

    from nnmnkwii_b200.baseline.gmm import _device_kmeans_plusplus
    X = _blobs(N, D, K, 11, zero_frac)
    for dtype in (torch.float64, torch.float32):
        Xd = _frames(X, dtype)
        X64 = _host(Xd).astype(np.float64)
        for seed in (0, 5):
            want_c, want_i = kmeans_plusplus(X64, K, random_state=seed)
            centers, indices = _device_kmeans_plusplus(Xd, K, seed)
            assert np.array_equal(_host(indices), want_i)
            assert np.array_equal(_host(centers), X64[want_i]) and np.array_equal(_host(centers), want_c)


# ---- Lloyd from given centres: the three stops --------------------------------------------------------------------
@pytest.mark.parametrize("stop,kw", [("strict", dict(max_iter=300, tol=0.0)), ("tol", dict(max_iter=300, tol=1e-2)),
                                     ("max_iter", dict(max_iter=3, tol=0.0))])
def test_lloyd_from_given_centres(stop, kw, capsys):
    X = _blobs(20000, 12, 10, 12, 0.05)
    init = X[np.random.default_rng(0).choice(len(X), 10, replace=False)] + 0.5
    capsys.readouterr()
    ref = _sk_kmeans(X, 10, init=init, verbose=1, **kw)
    printed = capsys.readouterr().out
    if stop == "strict":
        assert "strict convergence" in printed
    elif stop == "tol":
        assert "within tolerance" in printed
    else:
        assert "Converged" not in printed and ref.n_iter_ == kw["max_iter"]
    _assert_same_kmeans(ref, _dev_kmeans(_frames(X), 10, init=init, **kw))


# ---- whole k-means -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,D,K,zero_frac", [(5000, 8, 4, 0.0), (20000, 50, 16, 0.15), (8000, 72, 32, 0.0)])
def test_whole_kmeans_matches_sklearn(N, D, K, zero_frac):
    X = _blobs(N, D, K, 2, zero_frac)
    for seed in (0, 3):
        _assert_same_kmeans(_sk_kmeans(X, K, random_state=seed), _dev_kmeans(_frames(X), K, random_state=seed))


# ---- empty clusters and duplicate points ---------------------------------------------------------------------------
@pytest.mark.parametrize("n_far", [1, 3])
def test_empty_clusters_are_relocated_like_sklearn(n_far):
    X = _blobs(6000, 5, 6, 13)
    init = X[np.random.default_rng(1).choice(len(X), 8, replace=False)].copy()
    init[:n_far] = 1e4 + np.arange(n_far)[:, None]  # far from every frame: empty after the first assignment
    ref = _sk_kmeans(X, 8, init=init, max_iter=50)
    got = _dev_kmeans(_frames(X), 8, init=init, max_iter=50)
    _assert_same_kmeans(ref, got)
    first = _sk_kmeans(X, 8, init=init, max_iter=1)  # the relocated centres themselves
    _assert_same_kmeans(first, _dev_kmeans(_frames(X), 8, init=init, max_iter=1))


def test_duplicate_points_warn_about_distinct_clusters():
    from sklearn.exceptions import ConvergenceWarning

    from nnmnkwii_b200.baseline.gmm import _device_kmeans
    X = np.repeat(_blobs(3, 4, 3, 14), 100, axis=0)
    ref = _sk_kmeans(X, 5, random_state=0)
    with pytest.warns(ConvergenceWarning, match=r"Number of distinct clusters \(3\) found smaller than n_clusters \(5\)"):
        got = _device_kmeans(_frames(X), 5, random_state=0)
    # every frame sits on its centre: both inertias are rounding residue of the centring, ~1e-26
    _assert_same_kmeans(ref, got, inertia_atol=1e-12 * float(np.square(X).sum()))


# ---- every kernel instance ------------------------------------------------------------------------------------------
INSTANCE_SHAPES = [(4000, 32, 32), (4000, 33, 33), (3000, 64, 64), (3000, 65, 65), (3000, 96, 96), (3000, 97, 97),
                   (3000, 128, 128), (128, 128, 128), (37, 3, 37), (1, 1, 1), (17000, 7, 3), (16961, 20, 5)]

# The kernel names are collected in a child process: profiling this module's calls in the pytest process made
# torch.profiler lose the records of later modules' calls on an H100, which the other variant tests rely on.
_NAMES_SCRIPT = r"""
import json, sys
sys.path[:0] = sys.argv[1:3]
import numpy as np, torch
import variant_mirror as M
from nnmnkwii_b200.baseline import gmm as G
out = []
for N, D, K, dt in json.loads(sys.argv[3]):
    X = torch.from_numpy(np.random.default_rng(N + D + K).standard_normal((N, D))).to(getattr(torch, dt)).cuda()
    _, e1, a = M.profiled(lambda: G._device_kmeans_plusplus(X, 1, 0), r"\bkm_pp_dist_kernel<")
    st = G._KMeansState(X, K, centre=True)
    st.prepare()
    st.centers.copy_(X[:K].double() - st.mean)
    _, e2, b = M.profiled(lambda: st.lloyd(True), r"\bkm_assign_kernel<\d+, \w+, true>")
    out.append([sorted(set(M.launched(a, r"\bkm_pp_dist_kernel<"))),
                sorted(set(M.launched(b, r"\bkm_assign_kernel<\d+, \w+, true>"))), repr(e1), repr(e2)])
print(json.dumps(out))
"""


def test_kernel_names_follow_the_mirror():
    """km_pp_dist_kernel<ceil(D / 32), T> and km_assign_kernel<ceil(K / 32), T, true>, from the profiler."""
    import json
    import os
    import subprocess
    import sys

    from conftest import ROOT
    cases = [(N, D, K, dt) for N, D, K in INSTANCE_SHAPES for dt in ("float32", "float64")]
    res = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, os.path.join(ROOT, "tests"), ROOT, json.dumps(cases)],
                         capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0, res.stderr[-3000:]
    for (N, D, K, dt), (pp, assign, e1, e2) in zip(cases, json.loads(res.stdout.strip().splitlines()[-1])):
        T = "float" if dt == "float32" else "double"
        assert e1 == "None" and e2 == "None", (N, D, K, dt, e1, e2)
        want_pp, want_as = "km_pp_dist_kernel<%d, %s>" % (km_epl(D), T), "km_assign_kernel<%d, %s, true>" % (km_epl(K), T)
        assert pp and all(want_pp in n for n in pp), (want_pp, pp)
        assert assign and all(want_as in n for n in assign), (want_as, assign)


@pytest.mark.parametrize("N,D,K", INSTANCE_SHAPES)
def test_every_kernel_instance(N, D, K):
    """Each instance against sklearn; N % 64 != 0 ends in a partial frame tile, the others in a partial chunk."""
    import torch
    X = _blobs(N, D, min(K, 8), N + D + K)
    L = km_layout(N, D, K)
    assert (L["n_ll"] - 1) * L["ll_chunk"] < N <= L["n_ll"] * L["ll_chunk"]
    for dtype in (torch.float32, torch.float64):
        Xd = _frames(X, dtype)
        X64 = _host(Xd).astype(np.float64)
        _assert_same_kmeans(_sk_kmeans(X64, K, random_state=0, max_iter=30),
                            _dev_kmeans(Xd, K, random_state=0, max_iter=30))
        dense = _dev_kmeans(Xd, K, random_state=1, max_iter=5)
        strided = _dev_kmeans(_frames(X, dtype, pad=3), K, random_state=1, max_iter=5)
        assert np.array_equal(_host(dense[0]), _host(strided[0]))
        assert np.array_equal(_host(dense[1]), _host(strided[1])) and dense[2:] == strided[2:]


def test_runs_are_bit_identical():
    X = _blobs(30000, 24, 12, 15, 0.1)
    Xd = _frames(X)
    a = _dev_kmeans(Xd, 12, random_state=0)
    b = _dev_kmeans(Xd, 12, random_state=0)
    assert np.array_equal(_host(a[0]), _host(b[0])) and np.array_equal(_host(a[1]), _host(b[1])) and a[2:] == b[2:]


# ---- end to end ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("init", ["kmeans", "k-means++"])
def test_gmm_init_device_matches_host_init_and_sklearn(init):
    from nnmnkwii_b200.baseline.gmm import GaussianMixture
    X = _blobs(20000, 50, 16, 2, 0.15)
    kw = dict(n_components=16, init_params=init, random_state=0, max_iter=20)
    a, la, b, lb = _fit_both(X, **kw)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        c = GaussianMixture(init_device=True, **kw)
        lc = c.fit_predict(X)
    _assert_same_fit(a, la, c, lc)
    assert np.array_equal(lc, lb)
    for name in ("weights_", "means_", "covariances_", "precisions_cholesky_", "lower_bounds_"):
        assert np.array_equal(getattr(c, name), getattr(b, name)), name


def test_gmm_init_device_n_init_consumes_the_random_state_like_sklearn():
    from sklearn.mixture import GaussianMixture as Sk

    from nnmnkwii_b200.baseline.gmm import GaussianMixture
    X = _blobs(4000, 5, 4, 4)
    kw = dict(n_components=4, n_init=3, random_state=0, max_iter=30)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        a = Sk(**kw)
        la = a.fit_predict(X)
        b = GaussianMixture(init_device=True, **kw)
        lb = b.fit_predict(X)
    _assert_same_fit(a, la, b, lb)


def test_cuda_tensor_fit_never_downloads_the_frames(monkeypatch):
    import torch

    from nnmnkwii_b200.baseline import gmm as G
    X = _blobs(8000, 10, 6, 16).astype(np.float32)
    Xd = torch.from_numpy(X).cuda()
    seen = []
    real = G._host_f64

    def spy(t):
        seen.append(tuple(t.shape))
        return real(t)

    monkeypatch.setattr(G, "_host_f64", spy)
    for init in ("kmeans", "k-means++"):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            lc = G.GaussianMixture(n_components=6, init_params=init, init_device=True, random_state=0).fit_predict(Xd)
            ref = G.GaussianMixture(n_components=6, init_params=init, random_state=0).fit_predict(X)
        assert np.array_equal(lc.cpu().numpy(), ref)
    assert (8000, 10) not in seen


def test_iterative_aligner_device_init():
    from nnmnkwii_b200.preprocessing.alignment import IterativeDTWAligner
    X, Y = _aligner_pairs(4, 60, 5, 17)
    kw = dict(n_iter=2, n_components_gmm=4, random_state=0, gmm="device")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        Xa, Ya = IterativeDTWAligner(**kw).transform((X, Y))
        Xb, Yb = IterativeDTWAligner(gmm_init_device=True, **kw).transform((X, Y))
    assert np.array_equal(Xa, Xb) and np.array_equal(Ya, Yb)
