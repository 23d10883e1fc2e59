"""GPU: nnmnkwii_b200.util on the H100 -- cholesky_inv_banded bit for bit against the reference's golden
output and the C restatement of its recurrence, cholesky_inv within the CPU-measured bar of LAPACK's
dpotri (tests/linalg_mirror.py), the reference's own test cases, the diagonal check, apply_each2d_* on
CUDA tensors against the NumPy path, and every kernel instance the launchers can select."""
import numpy as np
import pytest

import linalg_mirror as M
import oracle
from nnmnkwii_b200 import _lib
from nnmnkwii_b200 import util
from nnmnkwii_b200.util import linalg

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def banded_factor(rng, T, w, B):
    """B lower factors with band width w: diagonally dominant, exact zeros inside the band, NaN, inf and
    huge values outside it (which must never be read)."""
    R = rng.standard_normal((B, T, T)) * 1e300
    R[rng.random((B, T, T)) < 0.05] = np.nan
    R[rng.random((B, T, T)) < 0.05] = np.inf
    for j in range(1, min(w, T)):
        i = np.arange(j, T)
        band = rng.uniform(-0.5, 0.5, (B, T - j))
        band[rng.random((B, T - j)) < 0.2] = 0.0
        R[:, i, i - j] = band
    R[:, np.arange(T), np.arange(T)] = 1.0 + 0.5 * w + rng.random((B, T))
    return R


def test_banded_golden_bit_for_bit(golden):
    P = linalg.cholesky_inv_banded(golden["cib_L"], 3)
    assert P.dtype == np.float64 and np.array_equal(P, golden["cib_Pinv"])


@pytest.mark.parametrize("T", [1, 2, 5, 31, 32, 33, 257, 1000])
@pytest.mark.parametrize("B", [1, 7])
def test_banded_matches_oracle_bit_for_bit(T, B):
    rng = np.random.default_rng(T * 10 + B)
    for w in range(1, 10):
        R = banded_factor(rng, T, w, B)
        got = linalg.cholesky_inv_banded(R if B > 1 else R[0], w)
        ref = np.stack([oracle.cholesky_inv_banded(np.ascontiguousarray(R[b]), w) for b in range(B)])
        assert np.all(np.isfinite(ref))
        assert np.array_equal(got, ref if B > 1 else ref[0]), (T, w, B)


def test_banded_tensor_forms():
    rng = np.random.default_rng(3)
    R = banded_factor(rng, 40, 5, 3)
    ref = np.stack([oracle.cholesky_inv_banded(np.ascontiguousarray(r), 5) for r in R])
    Rc = torch.from_numpy(R).cuda()
    got = linalg.cholesky_inv_banded(Rc, 5)
    assert got.is_cuda and got.dtype == torch.float64 and np.array_equal(got.cpu().numpy(), ref)
    got = linalg.cholesky_inv_banded(torch.from_numpy(R[0]), 5)
    assert not got.is_cuda and np.array_equal(got.numpy(), ref[0])
    R32 = np.where(np.abs(R) < 1e30, R, 0.0).astype(np.float32)
    ref32 = oracle.cholesky_inv_banded(R32[1].astype(np.float64), 5)
    got = linalg.cholesky_inv_banded(torch.from_numpy(R32[1]).cuda(), 5)
    assert got.dtype == torch.float32 and np.array_equal(got.cpu().numpy(), ref32.astype(np.float32))
    # float32 NumPy in: computed in float64 and returned in float64, as the reference does
    assert np.array_equal(linalg.cholesky_inv_banded(R32[1], 5), ref32)


def test_reference_test_linalg_choleskey_inv():
    """The reference's tests/test_util.py:62-81 (its window sets restated in tests/linalg_mirror.py)."""
    import scipy.linalg
    for windows in M.WINDOWS:
        for T in (5, 10):
            P = M.window_precision(windows, T)
            L = scipy.linalg.cholesky(P, lower=True)
            U = scipy.linalg.cholesky(P, lower=False)
            Pinv = np.linalg.inv(P)
            assert np.allclose(Pinv, linalg.cholesky_inv(L, lower=True))
            assert np.allclose(Pinv, linalg.cholesky_inv(U, lower=False))
            assert np.allclose(Pinv, linalg.cholesky_inv_banded(L, width=3))


def _bar(N):
    return M.DENSE_BAR * np.sqrt(N) * M.EPS


@pytest.mark.parametrize("N", [1, 2, 31, 32, 33, 256, 1024])
@pytest.mark.parametrize("lower", [True, False])
def test_dense_within_cpu_bar(N, lower):
    rng = np.random.default_rng(N)
    F, ref = M.spd_factor(rng, N, lower)
    got = linalg.cholesky_inv(F, lower=lower)
    assert got.dtype == np.float64 and got.shape == (N, N)
    assert np.array_equal(got, got.T)
    assert M.rel_to_scale(got, ref) <= _bar(N)
    t = linalg.cholesky_inv(torch.from_numpy(F).cuda(), lower=lower)
    assert t.is_cuda and t.dtype == torch.float64 and np.array_equal(t.cpu().numpy(), got)
    if N <= 256:
        pairs = [M.spd_factor(rng, N, lower) for _ in range(3)]
        Fb = np.stack([F] + [p[0] for p in pairs])
        gb = linalg.cholesky_inv(Fb, lower=lower)
        assert gb.shape == (4, N, N) and np.array_equal(gb[0], got)
        for b, (_, r) in enumerate(pairs, 1):
            assert M.rel_to_scale(gb[b], r) <= _bar(N)


def test_dense_float32_tensor():
    rng = np.random.default_rng(5)
    F, _ = M.spd_factor(rng, 100, True)
    F32 = F.astype(np.float32)
    ref = M.dpotri_full(np.tril(F32.astype(np.float64)), True)
    got = linalg.cholesky_inv(torch.from_numpy(F32).cuda(), lower=True)
    assert got.dtype == torch.float32
    assert np.abs(got.cpu().numpy() - ref).max() <= 4 * np.finfo(np.float32).eps * np.abs(ref).max()


@pytest.mark.parametrize("fn", ["dense", "banded"])
def test_zero_diagonal_names_the_item(fn):
    rng = np.random.default_rng(7)
    F = np.stack([M.spd_factor(rng, 20, True, garbage=False)[0] for _ in range(3)])
    F[1, 4, 4] = 0.0
    F[2, 2, 2] = np.nan
    call = (lambda x: linalg.cholesky_inv(x, lower=True)) if fn == "dense" else (lambda x: linalg.cholesky_inv_banded(x, 3))
    with pytest.raises(np.linalg.LinAlgError, match=r"batch item 1 .*row 4"):
        call(F)
    with pytest.raises(np.linalg.LinAlgError, match=r"batch item 0 .*row 2"):
        call(F[2])
    good = M.spd_factor(rng, 20, True, garbage=False)[0]  # the library stays usable
    assert np.allclose(call(good) @ (good @ good.T), np.eye(20), atol=1e-10) if fn == "dense" else \
        np.array_equal(call(good), oracle.cholesky_inv_banded(good, 3))


def test_non_finite_off_diagonal_does_not_fault():
    R = np.eye(6) * 2.0
    R[3, 2] = np.nan
    R[4, 3] = np.inf
    out = linalg.cholesky_inv_banded(R, 3)
    assert out.shape == (6, 6) and not np.all(np.isfinite(out))
    out = linalg.cholesky_inv(R, lower=True)
    assert out.shape == (6, 6)
    assert np.array_equal(linalg.cholesky_inv_banded(np.eye(4) * 2.0, 3), np.eye(4) * 0.25)


def test_wide_band_is_unsupported():
    with pytest.raises(NotImplementedError):
        linalg.cholesky_inv_banded(np.eye(12), 10)
    assert np.array_equal(linalg.cholesky_inv_banded(np.eye(8) * 2.0, 40), np.eye(8) * 0.25)  # min(width, T)


def test_empty_inputs():
    assert linalg.cholesky_inv(np.zeros((0, 0))).shape == (0, 0)
    assert linalg.cholesky_inv_banded(np.zeros((2, 0, 0))).shape == (2, 0, 0)


# ---- apply_each2d_* on CUDA tensors -------------------------------------------------------------------------
def _edge_batch(dtype):
    rng = np.random.default_rng(11)
    X = rng.standard_normal((5, 24, 4)).astype(dtype)
    X[0, 18:] = 0.0                       # zero tail
    X[1] = 0.0                            # all-zero slice
    X[2, 10:] = 0.0
    X[2, 9] = [1e-7, 0.0, 0.0, 0.0]       # abs sum exactly eps: kept
    X[3, 7:] = 0.0
    X[3, 6] = [np.nextafter(dtype(1e-7), dtype(0)), 0.0, 0.0, 0.0]  # just below eps: trimmed
    X[4, 20:] = 0.0
    X[4, 19] = [-5e-8, 5e-8, 0.0, 0.0]    # pairwise sum of |x| reaches eps
    return X


def _f(x):
    return x[:, [0, 1, 2, 3, 0, 1]] * 2


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_apply_each2d_trim_cuda_matches_numpy(dtype):
    X = _edge_batch(dtype)
    ref = util.apply_each2d_trim(_f, X)
    lens = [len(util.trim_zeros_frames(x)) for x in X]
    assert lens[1] == 0 and lens[2] == 10 and lens[3] == 6
    n0 = _lib.launch_count()
    got = util.apply_each2d_trim(_f, torch.from_numpy(X).cuda())
    assert _lib.launch_count() == n0 + 1  # one trim_len launch for all slices
    assert got.is_cuda and got.dtype == torch.from_numpy(X).dtype and got.shape == (5, 24, 6)
    assert np.array_equal(got.cpu().numpy().astype(np.float64), ref)


def test_apply_each2d_cuda_with_delta_features():
    from conftest import windows_set
    windows = windows_set()[2]
    X = _edge_batch(np.float32)[[0, 2, 4]]
    ref = util.apply_each2d_trim(util.delta_features, X, windows)
    got = util.apply_each2d_trim(util.delta_features, torch.from_numpy(X).cuda(), windows)
    assert got.is_cuda and got.dtype == torch.float32
    assert np.array_equal(got.cpu().numpy().astype(np.float64), ref)
    lengths = torch.tensor([18, 3, 24]).cuda()
    ref = util.apply_each2d_padded(util.delta_features, X, [18, 3, 24], windows)
    got = util.apply_each2d_padded(util.delta_features, torch.from_numpy(X).cuda(), lengths, windows)
    assert got.is_cuda and np.array_equal(got.cpu().numpy().astype(np.float64), ref)


# ---- every kernel instance ---------------------------------------------------------------------------------
def launch_group(group):
    """The calls of one group of kernel instances (run in a child process by `profiled_in_child`)."""
    rng = np.random.default_rng(0)
    if group == "banded":
        for w in range(1, 10):
            linalg.cholesky_inv_banded(banded_factor(rng, 20, w, 1)[0], w)
    else:
        for lower in (True, False):
            linalg.cholesky_inv(M.spd_factor(rng, 70, lower)[0], lower=lower)
    torch.cuda.synchronize()


def test_every_kernel_instance_runs():
    from variant_mirror import launched, profiled_in_child
    res = profiled_in_child("test_util_gpu", "launch_group", [(["banded"], r"cholinv_banded_kernel"),
                                                               (["dense"], r"cholinv_dense_kernel")])
    for r in res:
        assert r[1] == "None", r[1]
    for w in range(1, 10):
        assert launched(res[0][0], r"cholinv_banded_kernel<%d>" % w), w
    for lower in ("true", "false"):
        assert launched(res[1][0], r"cholinv_dense_kernel<%s>" % lower), lower
