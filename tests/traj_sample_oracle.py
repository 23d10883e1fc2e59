"""Float64 NumPy / SciPy restatement of sampling from the trajectory model (paramgen.trajectory_sample_batch,
DESIGN.md 3.21; the comment of nnk_mlpg_traj_sample in include/nnk_b200.h).  TEST INFRASTRUCTURE, NOT PRODUCT.

Three parts:

    philox / normals  Philox4x32-10 (Salmon et al. 2011) and the Box-Muller mapping of the header, vectorised in
                      uint32 / uint64 NumPy, bit for bit
    chain(banded)     the sample recurrence on the top-down L D L^T factors of the banded P:
                      y_t = zs_t + scale z_t / sqrt(d_t) - sum_j l_j[t] y_{t+j}
    chain(dense)      x = cbar + scale C^-T z with C = cholesky(P, lower=True) = L D^1/2

P, b and tau (edge rule, float32 division for float32 variances) come from tests/traj_ll_oracle.py.  Copied columns
repeat the means column in every sample.
"""
import numpy as np
from scipy import linalg

import traj_ll_oracle as TL

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_MASK = np.uint64(0xFFFFFFFF)


def philox(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 of broadcastable uint32 counter words and key words: (r0, r1, r2, r3) as uint32 arrays."""
    c0, c1, c2, c3, k0, k1 = np.broadcast_arrays(*(np.asarray(a, dtype=np.uint64) for a in (c0, c1, c2, c3, k0, k1)))
    for r in range(10):
        p0 = M0 * c0  # exact: both factors < 2^32
        p1 = M1 * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _MASK)
        if r < 9:
            k0, k1 = (k0 + W0) & _MASK, (k1 + W1) & _MASK
    return tuple(a.astype(np.uint32) for a in (c0, c1, c2, c3))


def pair_normals(seed, key, s, pair, out_col):
    """The two normals (z of frame 2 pair, z of frame 2 pair + 1) of counter (pair, out_col, s, key) under ``seed``."""
    seed = int(seed)
    r0, r1, r2, r3 = (a.astype(np.uint64) for a in
                      philox(pair, out_col, s, key, np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)))
    six, sh = np.uint64(6), np.uint64(26)
    nu = ((r0 >> six) << sh) | (r1 >> six)
    nv = ((r2 >> six) << sh) | (r3 >> six)
    U = (nu.astype(np.float64) + 0.5) * 2.0 ** -52
    V = nv.astype(np.float64) * 2.0 ** -52
    R = np.sqrt(-2.0 * np.log(U))
    return R * np.cos(2.0 * np.pi * V), R * np.sin(2.0 * np.pi * V)


def normals(seed, key, n_samples, T, out_col):
    """z (n_samples, T) of one chain: frame t takes the cosine (even t) or sine (odd t) normal of pair t >> 1."""
    s = np.arange(n_samples, dtype=np.uint64)[:, None]
    pair = (np.arange(T, dtype=np.uint64) >> np.uint64(1))[None, :]
    zc, zs = pair_normals(seed, key, s, pair, out_col)
    return np.where((np.arange(T) & 1)[None, :] == 1, zs, zc)


def factors(mean, var, windows):
    """(P sparse, b, d, l (T, S + 1) with l[t, j] = L[t + j, t], zs) of one chain, float64."""
    mean = np.asarray(mean, np.float64)
    T, _ = mean.shape
    st = TL._Stream(windows, True)
    mats = st.window_matrices(T)
    tau = TL.precisions(var, st.kept(T))
    S = max(l for l, _, _ in windows) + max(u for _, u, _ in windows)
    P = sum(W.T @ W.multiply(tau[:, w][:, None]) for w, W in enumerate(mats)).tocsr()
    b = np.asarray(sum(W.T @ (tau[:, w] * mean[:, w]) for w, W in enumerate(mats))).ravel()
    U = linalg.cholesky_banded(TL._band(P, S), lower=False)  # P = U^T U, U[t, t + k] = U_[S - k, t + k]
    diag = U[S]
    d = diag * diag
    lk = np.zeros((T, S + 1))
    for k in range(1, min(S, T - 1) + 1):
        lk[:T - k, k] = U[S - k, k:] / diag[:T - k]
    w = np.zeros(T)
    for t in range(T):
        w[t] = b[t] - sum(lk[t - k, k] * w[t - k] for k in range(1, S + 1) if t - k >= 0)
    return P, b, d, lk, w / d


def chain(mean, var, windows, z, scale=1.0, banded=True):
    """Samples (n_samples, T) of one chain: mean / var (T, nw) (var of its own dtype), z (n_samples, T)."""
    z = np.atleast_2d(np.asarray(z, np.float64))
    P, b, d, lk, zs = factors(mean, var, windows)
    T, S = lk.shape[0], lk.shape[1] - 1
    if not banded:
        P = P.toarray()
        C = np.linalg.cholesky(P)
        cbar = np.linalg.solve(P, b)
        return cbar[None, :] + scale * linalg.solve_triangular(C, z.T, lower=True, trans="T").T
    y = np.zeros((z.shape[0], T + S))
    isd = 1.0 / np.sqrt(d)
    for t in range(T - 1, -1, -1):
        acc = zs[t] + scale * z[:, t] * isd[t]
        for j in range(1, S + 1):
            acc = acc - lk[t, j] * y[:, t + j]
        y[:, t] = acc
    return y[:, :T]


def sample(means, variances, windows, n_samples, seed, key, scale=1.0, streams=None, banded=True):
    """Samples (n_samples, T, D_out) of one utterance (means (T, D), variances (T, D) or (D,)) under key ``key``."""
    means = np.asarray(means)
    variances = np.asarray(variances)
    T, D = means.shape
    nw = len(windows)
    parts, D_out = TL._parts(windows, streams, D)
    out = np.zeros((n_samples, T, D_out))
    var_t = np.broadcast_to(variances[:D], (T, D)) if variances.ndim == 1 else variances
    for in_col, sd, copy, oc in parts:
        for k in range(sd):
            if copy:
                out[:, :, oc + k] = means[:, in_col + k].astype(np.float64)[None, :]
                continue
            cols = [in_col + w * sd + k for w in range(nw)]
            z = normals(seed, key, n_samples, T, oc + k)
            out[:, :, oc + k] = chain(means[:, cols], var_t[:, cols], windows, z, scale, banded)
    return out


def cbar_and_cov(mean, var, windows):
    """(cbar, inv(P)) of one chain, dense."""
    P, b, _, _, _ = factors(mean, var, windows)
    P = P.toarray()
    return np.linalg.solve(P, b), np.linalg.inv(P)
