"""Float64 NumPy / SciPy restatement of the trajectory-model log-likelihood (paramgen.trajectory_log_likelihood_batch,
DESIGN.md 3.20; Zen, Tokuda & Kitamura 2007).  TEST INFRASTRUCTURE, NOT PRODUCT.

Per static column of a smoothed stream (a "chain") of one utterance of T frames:

    tau_{t,w}   1 / var_{t,w} evaluated in the variance's own dtype, then widened; zero where the edge rule of
                oracle.gmm_traj_em.Model.kept drops window w > 0 at frame t
    P, b        sum_w W_w^T diag(tau_w) W_w,  sum_w W_w^T (tau_w mu_w)   (the window matrices of
                oracle.gmm_traj_em.Model, zero outside the utterance)
    l           1/2 log det P - 1/2 (x - cbar)^T P (x - cbar) - (T/2) log 2 pi,  cbar = P^-1 b
    dl/dmu      tau (W x - W cbar)
    dl/dvar     -tau^2 / 2 [diag(W Sigma W^T) - (W x - mu)^2 + (W cbar - mu)^2],  Sigma = P^-1
    dl/dx       -P (x - cbar)

``banded=False`` forms P densely (slogdet, inv; short T only).  ``banded=True`` factors the band with
scipy.linalg.cholesky_banded and computes the band of Sigma by the backward recurrence of Takahashi et al. (1973)
from the L D L^T factors; ``sigma_band`` exposes that band so the tests can compare it with a dense inverse.
Copied columns have l = 0 and zero gradients.
"""
import numpy as np
from scipy import linalg

from oracle.gmm_traj_em import Model

LOG_2PI = np.log(2.0 * np.pi)


class _Stream(Model):
    """The window matrices and edge rule of oracle.gmm_traj_em.Model for one static column; no GMM."""

    def __init__(self, windows, banded):
        self.windows, self.static_dim, self.banded = windows, 1, banded


def precisions(var, keep):
    """tau: 1 / var in var's dtype (float32 division for float32 input), widened, zero where ``keep`` is False."""
    var = np.asarray(var)
    inv = (var.dtype.type(1) / var) if var.dtype in (np.float32, np.float64) else 1.0 / var.astype(np.float64)
    return np.where(keep, inv.astype(np.float64), 0.0)


def _band(P, S):
    """Upper banded form of the symmetric P: ab[S - k, t + k] = P[t, t + k]."""
    T = P.shape[0]
    ab = np.zeros((S + 1, T))
    for k in range(min(S, T - 1) + 1):
        ab[S - k, k:] = P.diagonal(k)
    return ab


def sigma_band(ab):
    """Band of Sigma = P^-1 from the upper banded P: sig[t, j] = Sigma[t, t + j] for j = 0 .. S (0 past T), by the
    backward recurrence on the L D L^T factors (l_k[t] = L[t + k, t])."""
    S = ab.shape[0] - 1
    T = ab.shape[1]
    U = linalg.cholesky_banded(ab, lower=False)  # P = U^T U, U[t, t + k] = U_[S - k, t + k]
    diag = U[S]
    d = diag * diag
    lk = np.zeros((T, S + 1))
    for k in range(1, min(S, T - 1) + 1):
        lk[:T - k, k] = U[S - k, k:] / diag[:T - k]
    sig = np.zeros((T + S, S + 1))  # rows past T stay zero

    def at(i, j):  # Sigma[i, j], i, j >= 0
        a, b = (i, j) if i <= j else (j, i)
        return sig[a, b - a]

    for t in range(T - 1, -1, -1):
        for j in range(S, 0, -1):
            sig[t, j] = -sum(lk[t, k] * at(t + k, t + j) for k in range(1, S + 1)) if t + j < T else 0.0
        sig[t, 0] = 1.0 / d[t] - sum(lk[t, k] * sig[t, k] for k in range(1, S + 1))
    return sig[:T], U


def chain(x, mean, var, windows, banded=False):
    """One chain: x (T,), mean / var (T, nw) (var of its own dtype).  Returns a dict with ll, cbar, tau, g_mean,
    g_var (T, nw) and g_x (T,)."""
    x = np.asarray(x, np.float64)
    mean = np.asarray(mean, np.float64)
    T, nw = mean.shape
    st = _Stream(windows, banded)
    mats = st.window_matrices(T)
    tau = precisions(var, st.kept(T))
    S = max(l for l, _, _ in windows) + max(u for _, u, _ in windows)
    P = sum(W.T @ (tau[:, w][:, None] * W) if not banded else W.T @ (W.multiply(tau[:, w][:, None]))
            for w, W in enumerate(mats))
    P = np.asarray(P.todense()) if banded else P
    b = sum(W.T @ (tau[:, w] * mean[:, w]) for w, W in enumerate(mats))
    if banded:
        ab = _band(P, S)
        sig, U = sigma_band(ab)
        logdet = 2.0 * np.sum(np.log(U[S]))
        cbar = linalg.cho_solve_banded((U, False), b)
        wsw = np.zeros((T, nw))
        for w, (l, u, coef) in enumerate(windows):
            for a in range(-l, u + 1):
                for c in range(-l, u + 1):
                    t = np.arange(T)
                    i, j = t + a, t + c
                    ok = (i >= 0) & (i < T) & (j >= 0) & (j < T)
                    lo, hi = np.minimum(i, j), np.maximum(i, j)
                    val = np.zeros(T)
                    val[ok] = sig[lo[ok], (hi - lo)[ok]]
                    wsw[:, w] += coef[l + a] * coef[l + c] * val
    else:
        sign, logdet = np.linalg.slogdet(P)
        assert sign > 0
        Sig = np.linalg.inv(P)
        cbar = np.linalg.solve(P, b)
        wsw = np.stack([np.einsum("ti,ij,tj->t", W, Sig, W) for W in mats], axis=1)
    ux = np.stack([W @ x for W in mats], axis=1)
    uc = np.stack([W @ cbar for W in mats], axis=1)
    e = ux - uc
    g_mean = tau * e
    ll = 0.5 * logdet - 0.5 * np.sum(tau * e * e) - 0.5 * T * LOG_2PI
    g_var = -0.5 * tau * tau * (wsw - (ux - mean) ** 2 + (uc - mean) ** 2)
    g_x = -sum(W.T @ g_mean[:, w] for w, W in enumerate(mats))
    return dict(ll=ll, cbar=cbar, tau=tau, g_mean=g_mean, g_var=g_var, g_x=np.asarray(g_x).ravel(), P=P)


def _parts(windows, streams, D):
    if streams is None:
        streams = [(0, D // len(windows))]
    parts, out = [], 0
    for s in streams:
        in_col, sd = int(s[0]), int(s[1])
        copy = len(s) > 2 and s[2] == "copy"
        parts.append((in_col, sd, copy, out))
        out += sd
    return parts, out


def log_likelihood(x, means, variances, windows, streams=None, banded=False):
    """One utterance: targets x (T, D_out), means (T, D), variances (T, D) or (D,).  Returns
    (ll (D_out,), g_means (T, D), g_vars (like variances), g_x (T, D_out)), float64."""
    means = np.asarray(means)
    variances = np.asarray(variances)
    T, D = means.shape
    nw = len(windows)
    parts, D_out = _parts(windows, streams, D)
    ll = np.zeros(D_out)
    g_m = np.zeros((T, D))
    g_v = np.zeros((T, D))
    g_x = np.zeros((T, D_out))
    var_t = np.broadcast_to(variances[:D], (T, D)) if variances.ndim == 1 else variances
    for in_col, sd, copy, out in parts:
        if copy:
            continue
        for d in range(sd):
            cols = [in_col + w * sd + d for w in range(nw)]
            r = chain(np.asarray(x)[:, out + d], means[:, cols], var_t[:, cols], windows, banded)
            ll[out + d] = r["ll"]
            g_m[:, cols] = r["g_mean"]
            g_v[:, cols] = r["g_var"]
            g_x[:, out + d] = r["g_x"]
    if variances.ndim == 1:
        gv = np.zeros(variances.shape[0])
        gv[:D] = g_v.sum(axis=0)
        g_v = gv
    return ll, g_m, g_v, g_x
