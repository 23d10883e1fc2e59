"""Host mirrors for util.linalg tests: the SPD test factors, the reference's ``dpotri`` + mirror on
scipy, a float64 NumPy restatement of the substitution order of ``cholinv_dense_kernel``
(csrc/nnk_linalg.cu), and the tolerance the GPU result is held to.

The restatement sets the bar: it runs the kernel's own order (tiles of ``ROWS`` rows per group of
``BLOCK`` columns, sequential sums) and tests/test_util_cpu.py measures how far it lands from
``dpotri``.  The only difference from the kernel is that it rounds products and sums separately where
the kernel fuses them (FMA), which does not change the size of the error."""
import numpy as np
import scipy.linalg

BLOCK, ROWS = 64, 8  # kDenseBlock, kDenseRows of csrc/nnk_linalg.cu (kDenseK chunks keep the order)
EPS = np.finfo(np.float64).eps

# max |P_gpu - P_dpotri| / max |P_dpotri| <= DENSE_BAR * sqrt(N) * EPS on the factors of `spd_factor`.
# The restatement measured at most 0.52 of sqrt(N) * EPS (N = 1; 0.34 at N = 2, below 0.05 from N = 31 up
# to 512); tests/test_util_cpu.py holds it to half of DENSE_BAR, so the GPU keeps a margin of 2 over that.
DENSE_BAR = 2.0

WINDOWS = [  # the reference's tests/test_util.py:7-25
    [(0, 0, np.array([1.0]))],
    [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5]))],
    [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))],
]


def window_precision(windows, T):
    """sum_w W_w^T W_w (the reference's _get_banded_test_mat) with W_w[t, t + k] = coeff[l + k], dense."""
    P = np.zeros((T, T))
    for l, u, c in windows:
        W = np.zeros((T, T))
        for t in range(T):
            for k in range(-l, u + 1):
                if 0 <= t + k < T:
                    W[t, t + k] = c[l + k]
        P += W.T @ W
    return P


def spd_factor(rng, N, lower, garbage=True):
    """(factor, P^-1 by dpotri + mirror): the Cholesky factor of M M^T / N + I / 2 (condition number below
    about 9), with the unused triangle filled with garbage when ``garbage``."""
    M = rng.standard_normal((N, N))
    A = M @ M.T / max(N, 1) + 0.5 * np.eye(N)
    F = scipy.linalg.cholesky(A, lower=lower)
    ref = dpotri_full(F, lower)
    if garbage and N > 1:
        junk = rng.standard_normal((N, N)) * 1e3
        mask = np.triu(np.ones((N, N), bool), 1) if lower else np.tril(np.ones((N, N), bool), -1)
        F = np.where(mask, junk, F)
    return F, ref


def dpotri_full(F, lower):
    """The reference's cholesky_inv (util/linalg.py:7-36): LAPACK dpotri on the named triangle, mirrored."""
    inv, info = scipy.linalg.lapack.dpotri(F, lower=lower)
    assert info == 0
    return np.tril(inv) + np.tril(inv, -1).T if lower else np.triu(inv) + np.triu(inv, 1).T


def dense_restatement(F, lower):
    """cholinv_dense_kernel's order in float64 NumPy: per group of BLOCK columns, forward tiles of ROWS rows
    (sum over earlier rows in ascending order, then the tile's own rows), then backward tiles (sum over
    later tiles in ascending order, then the tile's own later rows), lower triangle mirrored."""
    N = F.shape[0]
    L = np.tril(F) if lower else np.triu(F).T  # the lower factor the kernel reads
    P = np.zeros((N, N))
    for c0 in range(0, N, BLOCK):
        cols = np.arange(c0, min(c0 + BLOCK, N))
        Y = np.zeros((N, len(cols)))  # Y[t, j]: y (then x) of column cols[j]; zero above the column
        n_tiles = (N - c0 + ROWS - 1) // ROWS
        for m in range(n_tiles):
            t0 = c0 + m * ROWS
            rows = range(t0, min(t0 + ROWS, N))
            acc = {t: _seqsum(L[t, c0:t0, None] * Y[c0:t0]) for t in rows}
            for t in rows:
                s = acc[t]
                for q in range(t0, t):
                    s = s + L[t, q] * Y[q]
                y = ((cols == t).astype(np.float64) - s) / L[t, t]
                Y[t] = np.where(t >= cols, y, 0.0)
        for m in range(n_tiles - 1, -1, -1):
            t0 = c0 + m * ROWS
            hi = min(t0 + ROWS, N)
            acc = {t: _seqsum(L[hi:, t, None] * Y[hi:]) for t in range(t0, hi)}
            for t in range(hi - 1, t0 - 1, -1):
                s = acc[t]
                for q in range(t + 1, hi):
                    s = s + L[q, t] * Y[q]
                Y[t] = np.where(t >= cols, (Y[t] - s) / L[t, t], 0.0)
        P[:, cols] = Y
    return np.tril(P) + np.tril(P, -1).T


def _seqsum(a):
    """Sum over axis 0 in ascending order (np.cumsum is sequential; np.sum would be pairwise)."""
    return np.cumsum(a, axis=0)[-1] if len(a) else np.zeros(a.shape[1:])


def rel_to_scale(a, ref):
    return float(np.abs(np.asarray(a) - ref).max() / max(np.abs(ref).max(), 1e-300))
