"""CPU: the host side of the device k-means initialisation of baseline.gmm.GaussianMixture (csrc/nnk_kmeans.cu).

The k-means++ random draws are made on the host with scikit-learn's own RandomState calls and uploaded; here
they are checked to leave a RandomState where `sklearn.cluster.kmeans_plusplus` leaves it, and a NumPy float64
restatement of the device seeding loop (`kmeans_plusplus_restated`, the step order of csrc/nnk_kmeans.cu) is
checked to pick scikit-learn's seeds from those draws.  The workspace layout is mirrored here (`km_layout`) and
compared with `nnk_kmeans_workspace_bytes`, and the size limits are checked to raise before any launch."""
import ctypes
import pickle

import numpy as np
import pytest

# ---- mirror of km_layout in csrc/nnk_kmeans.cu -----------------------------------------------------------------
KM_MAX_D = KM_MAX_K = 128
KM_KP = 128
KM_THREADS = 256
KM_COL_CHUNK = 1024
PP_CHUNK = 1024
LL_FT = 64             # Lloyd assignment: frames per tile (8 frames per warp x 8 warps)
K_NUM_SMS = 132
LL_TARGET_BLOCKS = 2 * K_NUM_SMS
IW_SLOTS = 16


def km_trials(K):
    return 2 + int(np.log(K))


def km_epl(n):
    """Template parameter of km_pp_dist_kernel (n = D) and km_assign_kernel (n = K): ceil(n / 32)."""
    return min(4, (n + 31) // 32)


def _r4(v):
    return (v + 3) // 4 * 4


def km_layout(N, D, K):
    t = km_trials(K)
    n_col = -(-N // KM_COL_CHUNK)
    n_pp = -(-N // PP_CHUNK)
    per = -(-N // LL_TARGET_BLOCKS)
    ll_chunk = -(-per // LL_FT) * LL_FT
    n_ll = -(-N // ll_chunk)
    n_in = -(-N // KM_THREADS)
    total = (IW_SLOTS + _r4(n_col * D) + 4 + _r4(t * n_pp) + _r4(t * N) + D * KM_KP + KM_KP
             + _r4(n_ll * (K * (D + 1) + 1)) + _r4(n_in) + _r4(K))
    return {"trials": t, "n_pp": n_pp, "ll_chunk": ll_chunk, "n_ll": n_ll, "total": total}


# ---- NumPy restatement of the device seeding ---------------------------------------------------------------------
def kmeans_plusplus_restated(X, K, first, u):
    """csrc/nnk_kmeans.cu's k-means++ in NumPy float64 from pre-drawn values: candidate distances as
    max(-2 x.c + |c|^2 + |x|^2, 0), min with closest_dist_sq, one potential per candidate, first argmin; the next
    candidates are the first rows whose inclusive prefix sum of closest_dist_sq reaches u * current_pot."""
    N = X.shape[0]
    xn = np.einsum("ij,ij->i", X, X)

    def dist(c):
        return np.maximum(-2.0 * (X @ X[c]) + xn[c] + xn, 0.0)

    indices = [first]
    closest = dist(first)
    pot = closest.sum()
    for c in range(1, K):
        cand = np.minimum(np.searchsorted(np.cumsum(closest), u[c - 1] * pot, side="left"), N - 1)
        d = np.minimum(closest[None, :], np.stack([dist(i) for i in cand]))
        pots = d.sum(axis=1)
        best = int(np.argmin(pots))
        pot, closest = pots[best], d[best]
        indices.append(int(cand[best]))
    return np.asarray(indices)


def _blobs(N, D, K, seed, zero_frac=0.0):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((K, D)) * 3.0
    lab = rng.integers(0, K, N)
    X = centres[lab] + rng.standard_normal((N, D)) * rng.uniform(0.3, 1.5, (K, D))[lab]
    X[:, 0] += 20.0
    if zero_frac:
        X[rng.random(N) < zero_frac] = 0.0
    return X


@pytest.mark.parametrize("N,K", [(10, 1), (500, 3), (2000, 16), (3000, 128)])
def test_draws_consume_the_random_state_like_sklearn(N, K):
    from sklearn.cluster import kmeans_plusplus

    from nnmnkwii_b200.baseline.gmm import _kmeans_plusplus_draws
    X = _blobs(N, 4, max(K, 2), 0)
    a, b = np.random.RandomState(7), np.random.RandomState(7)
    _, idx = kmeans_plusplus(X, K, random_state=a)
    first, u = _kmeans_plusplus_draws(N, K, b)
    assert u.shape == (K - 1, km_trials(K))
    assert first == idx[0]
    assert a.uniform() == b.uniform() and a.randint(1 << 30) == b.randint(1 << 30)


@pytest.mark.parametrize("N,D,K,zero_frac", [(50, 3, 1, 0.0), (1000, 2, 5, 0.0), (3000, 8, 16, 0.15),
                                             (4000, 50, 32, 0.0), (2000, 6, 128, 0.0)])
def test_restated_seeding_picks_sklearns_indices(N, D, K, zero_frac):
    from sklearn.cluster import kmeans_plusplus

    from nnmnkwii_b200.baseline.gmm import _kmeans_plusplus_draws
    X = _blobs(N, D, 8, N + D + K, zero_frac)
    for seed in (0, 1):
        _, want = kmeans_plusplus(X, K, random_state=seed)
        first, u = _kmeans_plusplus_draws(N, K, np.random.RandomState(seed))
        assert np.array_equal(kmeans_plusplus_restated(X, K, first, u), want)


@pytest.mark.parametrize("K", [1, 2, 7, 8, 20, 21, 54, 55, 128])
@pytest.mark.parametrize("D", [1, 31, 33, 128])
def test_workspace_mirror_matches_workspace_bytes(D, K):
    from nnmnkwii_b200 import _lib
    for N in (K, K + 1, 1023, 1024, 1025, 16895, 16896, 16897, 409600):
        if N < K:
            continue
        L = km_layout(N, D, K)
        assert L["total"] * 8 == _lib.lib.nnk_kmeans_workspace_bytes(N, D, K), (N, D, K)
        assert L["ll_chunk"] % LL_FT == 0 and (L["n_ll"] - 1) * L["ll_chunk"] < N <= L["n_ll"] * L["ll_chunk"]
        assert L["trials"] <= 8


def test_workspace_bytes_is_zero_outside_the_limits():
    from nnmnkwii_b200 import _lib
    ws = _lib.lib.nnk_kmeans_workspace_bytes
    assert ws(1000, KM_MAX_D, KM_MAX_K) > 0
    for N, D, K in ((1000, 0, 2), (1000, KM_MAX_D + 1, 2), (1000, 4, 0), (1000, 4, KM_MAX_K + 1), (3, 4, 4),
                    (1 << 31, 4, 2)):
        assert ws(N, D, K) == 0, (N, D, K)


def test_estimator_parameters_clone_and_pickle():
    from sklearn.base import clone

    from nnmnkwii_b200.baseline.gmm import GaussianMixture
    g = GaussianMixture(n_components=3, init_device=True, random_state=4)
    assert g.get_params()["init_device"] is True
    assert GaussianMixture().get_params()["init_device"] is False
    assert clone(g).get_params() == g.get_params()
    assert pickle.loads(pickle.dumps(g)).get_params() == g.get_params()
    with pytest.raises(ValueError, match="init_device"):
        GaussianMixture(init_device="yes")._validate_params()


def test_aligner_rejects_device_init_with_sklearn_gmm():
    from nnmnkwii_b200.preprocessing.alignment import IterativeDTWAligner
    with pytest.raises(ValueError, match="gmm_init_device"):
        IterativeDTWAligner(gmm="sklearn", gmm_init_device=True)
    assert IterativeDTWAligner(gmm="device", gmm_init_device=True).gmm_init_device


def _abi_call(name, N, D, K, x_ld=None):
    """An entry point with host dummies: the argument checks run, nothing is launched or dereferenced."""
    from nnmnkwii_b200 import _lib
    dummy = (ctypes.c_double * 16)()
    p = ctypes.cast(dummy, ctypes.c_void_p).value
    a = _lib.NnkKmeansArgs()
    a.X, a.N, a.x_ld, a.dtype, a.D, a.K = p, N, D if x_ld is None else x_ld, _lib.NNK_F64, D, K
    for f in ("centers", "sums", "weights", "labels", "indices", "mean", "dist", "out_centers", "status", "rand"):
        setattr(a, f, p)
    a.workspace, a.workspace_bytes = p, 0
    return getattr(_lib.lib, name)(ctypes.byref(a), None)


def test_bad_sizes_raise_before_any_launch():
    import torch

    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200.baseline.gmm import _device_kmeans, _device_kmeans_plusplus
    n0 = _lib.launch_count()
    for name in ("nnk_kmeans_prepare", "nnk_kmeans_seed", "nnk_kmeans_lloyd", "nnk_kmeans_relocate_dist",
                 "nnk_kmeans_average", "nnk_kmeans_inertia"):
        assert _abi_call(name, 1000, KM_MAX_D + 1, 4) == _lib.NNK_ERR_UNSUPPORTED, name
        assert _abi_call(name, 1000, 4, KM_MAX_K + 1) == _lib.NNK_ERR_UNSUPPORTED, name
        assert _abi_call(name, 3, 4, 4) == _lib.NNK_ERR_ARG, name
        assert _abi_call(name, 1000, 4, 4, x_ld=3) == _lib.NNK_ERR_ARG, name
        assert _abi_call(name, 1000, 4, 4) == _lib.NNK_ERR_WORKSPACE, name
    for fn in (lambda X, K: _device_kmeans(X, K, random_state=0), lambda X, K: _device_kmeans_plusplus(X, K, 0)):
        with pytest.raises(ValueError, match="features"):
            fn(torch.zeros((300, KM_MAX_D + 1), dtype=torch.float64), 2)
        with pytest.raises(ValueError, match="clusters"):
            fn(torch.zeros((300, 3), dtype=torch.float64), KM_MAX_K + 1)
        with pytest.raises(ValueError, match="n_samples=4 should be >= n_clusters=5"):
            fn(torch.zeros((4, 3), dtype=torch.float64), 5)
    assert _lib.launch_count() == n0
