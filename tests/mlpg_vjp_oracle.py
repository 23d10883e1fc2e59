"""Float64 NumPy / SciPy restatement of the gradient of MLPG in its means and variances (paramgen.mlpg_vjp_batch,
DESIGN.md 3.22; Wu & Wang 2006).  TEST INFRASTRUCTURE, NOT PRODUCT.

Per static column of a smoothed stream (a "chain") of one utterance of T frames, with tau, P and b of
tests/traj_ll_oracle.py (its window matrices, edge rule and precisions in the variance's own dtype), cbar = P^-1 b
and the gradient o = dL/dcbar:

    g           P^-1 o
    dL/dmu      tau (W g)
    dL/dtau     (W g) (mu - W cbar)
    dL/dvar     -tau^2 dL/dtau

``banded=False`` solves densely (short T only); ``banded=True`` keeps the window matrices sparse and solves with
scipy.linalg.solveh_banded.  Copied columns pass o through to their mean and have a zero variance gradient.
"""
import numpy as np
from scipy import linalg

import traj_ll_oracle as O


def chain(o, mean, var, windows, banded=False):
    """One chain: o (T,), mean / var (T, nw) (var of its own dtype).  Returns a dict with cbar, g, tau, g_mean,
    g_tau and g_var (T, nw)."""
    o = np.asarray(o, np.float64)
    mean = np.asarray(mean, np.float64)
    T, nw = mean.shape
    st = O._Stream(windows, banded)
    mats = st.window_matrices(T)
    tau = O.precisions(var, st.kept(T))
    P = sum(W.T @ (W.multiply(tau[:, w][:, None]) if banded else tau[:, w][:, None] * W) for w, W in enumerate(mats))
    b = sum(W.T @ (tau[:, w] * mean[:, w]) for w, W in enumerate(mats))
    if banded:
        S = max(l for l, _, _ in windows) + max(u for _, u, _ in windows)
        cbar, g = linalg.solveh_banded(O._band(P, S), np.stack([b, o], axis=1)).T
    else:
        cbar, g = np.linalg.solve(P, np.stack([b, o], axis=1)).T
    Wg = np.stack([W @ g for W in mats], axis=1)
    Wc = np.stack([W @ cbar for W in mats], axis=1)
    g_tau = Wg * (mean - Wc)
    return dict(cbar=cbar, g=g, tau=tau, g_mean=tau * Wg, g_tau=g_tau, g_var=-tau * tau * g_tau)


def vjp(means, variances, windows, grad_output, streams=None, banded=False):
    """One utterance: means (T, D), variances (T, D) or (D,), grad_output (T, D_out).  Returns
    (g_means (T, D), g_vars (like variances)), float64."""
    means = np.asarray(means)
    variances = np.asarray(variances)
    go = np.asarray(grad_output, np.float64)
    T, D = means.shape
    nw = len(windows)
    parts, _ = O._parts(windows, streams, D)
    g_m = np.zeros((T, D))
    g_v = np.zeros((T, D))
    var_t = np.broadcast_to(variances[:D], (T, D)) if variances.ndim == 1 else variances
    for in_col, sd, copy, out in parts:
        for d in range(sd):
            if copy:
                g_m[:, in_col + d] = go[:, out + d]
                continue
            cols = [in_col + w * sd + d for w in range(nw)]
            r = chain(go[:, out + d], means[:, cols], var_t[:, cols], windows, banded)
            g_m[:, cols] = r["g_mean"]
            g_v[:, cols] = r["g_var"]
    if variances.ndim == 1:
        g_v = g_v.sum(axis=0)
    return g_m, g_v
