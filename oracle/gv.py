"""Float64 NumPy / SciPy restatement of parameter generation considering global variance.  TEST
INFRASTRUCTURE, NOT PRODUCT.

Written from Toda, Black & Tokuda, "Voice conversion based on maximum-likelihood estimation of spectral
parameter trajectory", IEEE TASLP 15(8), 2007, Sec. IV (diagonal GV covariance), with this project's step
rule (DESIGN.md 3.15).  One chain = one static dimension of one utterance:

    tau, P, b  exactly as paramgen.mlpg builds them (dynamic-window precisions zeroed in the first and last
               max_win_width frames)
    c_m        = P^-1 b
    v(c)       = mean((c - mean(c))^2)
    F(c)       = omega (b^T c - c^T P c / 2) - prec (v(c) - mu)^2 / 2,   prec = 1 / gv_var
    c0         = mean(c_m) + sqrt(mu / v(c_m)) (c_m - mean(c_m))   (c_m when v(c_m) == 0)
    n_iter trials:  g = -(2/T) prec (v(c) - mu) (c - mean(c)),  z = P^-1 g,  delta = (c_m - c) + z / omega,
                    c' = c + alpha delta;  c <- c' if F(c') >= F(c) else alpha <- alpha / 2

The banded solves go through scipy.linalg.solveh_banded.
"""
import numpy as np
from scipy.linalg import solveh_banded


def build_system(mean, var, windows):
    """``(P_upper, b)`` of one chain: ``mean`` / ``var`` are ``(T, nw)`` (column w = window w); P in the upper
    banded form of scipy.linalg.solveh_banded (row S - k holds the k-th superdiagonal)."""
    mean = np.asarray(mean, dtype=np.float64)
    var = np.asarray(var)
    T, nw = mean.shape
    m = max(max(int(l), int(u)) for l, u, _ in windows)
    S = 2 * m
    tau = (1.0 / var).astype(np.float64)  # in the input dtype, like the reference's precisions
    for w in range(1, nw):
        tau[:m, w] = 0.0
        tau[T - m if m else 0:, w] = 0.0  # m == 0: the reference's [-0:] slice covers every frame
    Pd = np.zeros((S + 1, T))  # Pd[k, t] = P[t, t + k]
    b = np.zeros(T)
    for w, (l, u, coef) in enumerate(windows):
        coef = np.asarray(coef, dtype=np.float64)
        # W_w[t, t + k] = coef[l + k]; P += W^T diag(tau) W; b += W^T (tau * mean)
        for k1 in range(-l, u + 1):
            for k2 in range(-l, u + 1):
                if k2 < k1:
                    continue
                # row r of W touches columns r + k1 <= r + k2: P[r + k1, r + k2] += tau[r] c1 c2
                r = np.arange(T)
                ok = (r + k1 >= 0) & (r + k2 < T)
                np.add.at(Pd[k2 - k1], (r + k1)[ok], tau[ok, w] * coef[l + k1] * coef[l + k2])
            r = np.arange(T)
            ok = (r + k1 >= 0) & (r + k1 < T)
            np.add.at(b, (r + k1)[ok], tau[ok, w] * mean[ok, w] * coef[l + k1])
    Pu = np.zeros((S + 1, T))
    for k in range(min(S, T - 1) + 1):  # a diagonal at k >= T lies outside the matrix
        Pu[S - k, k:] = Pd[k, :T - k]
    return Pu, b


def band_matvec(Pu, c):
    """P c for P in upper banded form."""
    S = Pu.shape[0] - 1
    T = len(c)
    y = Pu[S] * c
    for k in range(1, min(S, T - 1) + 1):
        d = Pu[S - k, k:]
        y[:T - k] += d * c[k:]
        y[k:] += d * c[:T - k]
    return y


def variance(c):
    return float(np.mean((c - np.mean(c)) ** 2))


def objective(c, Pu, b, mu, prec, omega):
    """F(c) = omega (b^T c - c^T P c / 2) - prec (v(c) - mu)^2 / 2."""
    c = np.asarray(c, dtype=np.float64)
    v = variance(c)
    return float(omega * (b @ c - 0.5 * c @ band_matvec(Pu, c)) - 0.5 * prec * (v - mu) ** 2)


def solve(Pu, rhs):
    if Pu.shape[0] == 1:
        return rhs / Pu[0]
    return solveh_banded(Pu, rhs)


def mlpg_gv_chain(mean, var, windows, mu, gv_var, n_iter=20, step=1.0, weight=None, trace=None):
    """Generated static trajectory ``(T,)`` of one chain; ``trace`` (a list) receives ``(F, accepted)`` of
    the start point and of every trial."""
    Pu, b = build_system(mean, var, windows)
    T = len(b)
    prec = 1.0 / float(gv_var)
    mu = float(mu)
    omega = float(weight) if weight is not None else 1.0 / (len(windows) * T)
    cm = solve(Pu, b)
    vm = variance(cm)
    c = np.mean(cm) + np.sqrt(mu / vm) * (cm - np.mean(cm)) if vm > 0 else cm.copy()
    f = objective(c, Pu, b, mu, prec, omega)
    if trace is not None:
        trace.append((f, True))
    alpha = float(step)
    for _ in range(int(n_iter)):
        g = -(2.0 / T) * prec * (variance(c) - mu) * (c - np.mean(c))
        z = solve(Pu, g)
        c2 = c + alpha * ((cm - c) + z / omega)
        f2 = objective(c2, Pu, b, mu, prec, omega)
        ok = f2 >= f
        if ok:
            c, f = c2, f2
        else:
            alpha *= 0.5
        if trace is not None:
            trace.append((f2, ok))
    return c


def chain_system(mean_frames, variance_frames, windows, d):
    """``(mean, var)`` ``(T, nw)`` of static dimension ``d`` of a reference-layout ``(T, nw * sd)`` matrix
    (variances ``(T, D)`` or ``(D,)``)."""
    mean_frames = np.asarray(mean_frames, dtype=np.float64)
    T, D = mean_frames.shape
    nw = len(windows)
    sd = D // nw
    v = np.asarray(variance_frames)
    if v.ndim == 1:
        v = np.tile(v[:D], (T, 1))
    cols = [w * sd + d for w in range(nw)]
    return mean_frames[:, cols], v[:, cols]


def mlpg_gv(mean_frames, variance_frames, windows, gv_mean, gv_var, n_iter=20, step=1.0, weight=None):
    """``(T, static_dim)`` float64: :func:`mlpg_gv_chain` for every static dimension of one utterance."""
    T, D = np.shape(mean_frames)
    sd = D // len(windows)
    out = np.zeros((T, sd))
    for d in range(sd):
        m, v = chain_system(mean_frames, variance_frames, windows, d)
        out[:, d] = mlpg_gv_chain(m, v, windows, gv_mean[d], gv_var[d], n_iter, step, weight)
    return out


def mlpg(mean_frames, variance_frames, windows):
    """``c_m`` of every static dimension (the trajectory without GV), ``(T, static_dim)`` float64."""
    T, D = np.shape(mean_frames)
    sd = D // len(windows)
    out = np.zeros((T, sd))
    for d in range(sd):
        m, v = chain_system(mean_frames, variance_frames, windows, d)
        out[:, d] = solve(*build_system(m, v, windows))
    return out


def chain_objective(mean_frames, variance_frames, windows, d, c, mu, gv_var, weight=None):
    """F of trajectory ``c`` of static dimension ``d`` (for comparing two trajectories of one chain)."""
    m, v = chain_system(mean_frames, variance_frames, windows, d)
    Pu, b = build_system(m, v, windows)
    omega = float(weight) if weight is not None else 1.0 / (len(windows) * len(b))
    return objective(c, Pu, b, float(mu), 1.0 / float(gv_var), omega)
