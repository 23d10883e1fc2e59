"""Float64 NumPy / SciPy restatement of parameter generation considering the modulation spectrum.  TEST
INFRASTRUCTURE, NOT PRODUCT.

Written from the definition of DESIGN.md 3.18 (the idea of Takamichi et al., "Parameter generation algorithm
considering modulation spectrum for HMM-based speech synthesis", ICASSP 2015, with this project's step rule).
One chain = one static dimension of one utterance of T <= n frames:

    tau, P, b  exactly as paramgen.mlpg builds them (oracle.gv.build_system), c_m = P^-1 b
    Y          = numpy.fft.rfft(c, n),  s_k = log(max(|Y_k|^2, tiny)),  tiny = the smallest normal float64
    F(c)       = omega (b^T c - c^T P c / 2) - 1/2 sum_{k=1}^{n/2} q_k (s_k - nu_k)^2,  q_k = 1 / ms_var_k (0 for inf)
    c0         = c_m
    n_iter trials:  g = dF_MS/dc,  h = P^-1 g,  delta = (c_m - c) + h / omega,
                    c' = c + alpha delta;  c <- c' if F(c') >= F(c) else alpha <- alpha / 2

The banded solves go through scipy.linalg.solveh_banded (oracle.gv.solve).
"""
import numpy as np

from oracle.gv import band_matvec, build_system, chain_system, solve

TINY = np.finfo(np.float64).tiny


def _precisions(ms_var):
    v = np.asarray(ms_var, dtype=np.float64)
    with np.errstate(divide="ignore"):
        return np.where(np.isinf(v), 0.0, 1.0 / v)


def ms_term(c, nu, q, n):
    """-1/2 sum_{k >= 1} q_k (s_k - nu_k)^2 of trajectory ``c``."""
    p = np.abs(np.fft.rfft(c, n)) ** 2
    s = np.log(np.maximum(p, TINY))
    on = q > 0
    on[0] = False
    return float(-0.5 * np.sum(q[on] * (s[on] - nu[on]) ** 2))


def ms_gradient(c, nu, q, n):
    """Analytic gradient of :func:`ms_term`: sum_k 2 G_k Re(Y_k e^{2 pi i k t / n}), G_k = -q_k (s_k - nu_k) / |Y_k|^2
    (0 for bin 0, exempt bins and bins of power <= tiny)."""
    T = len(c)
    Y = np.fft.rfft(c, n)
    p = np.abs(Y) ** 2
    on = (q > 0) & (p > TINY)
    on[0] = False
    G = np.zeros_like(p)
    G[on] = -q[on] * (np.log(p[on]) - nu[on]) / p[on]
    C = G * Y
    C[-1] *= 2.0  # irfft counts bin n / 2 once, the other bins twice
    return n * np.fft.irfft(C, n)[:T]


def objective(c, Pu, b, nu, q, n, omega):
    c = np.asarray(c, dtype=np.float64)
    return float(omega * (b @ c - 0.5 * c @ band_matvec(Pu, c)) + ms_term(c, nu, q, n))


def _scale(c, Pu, b, nu, q, n, omega, const):
    """Size of the terms whose rounding bounds an F difference: omega (|b^T c| + c^T P c / 2 + const / 2) plus the
    MS term (const = sum tau mu^2, the constant a stencil form of the quadratic term carries)."""
    return omega * (abs(b @ c) + 0.5 * abs(c @ band_matvec(Pu, c)) + 0.5 * const) - ms_term(c, nu, q, n)


def _tau_mu2(mean, var, windows):
    """sum_w sum_t tau_w,t mu_w,t^2 with the edge rule of oracle.gv.build_system."""
    mean = np.asarray(mean, dtype=np.float64)
    tau = 1.0 / np.asarray(var, dtype=np.float64)
    T, nw = mean.shape
    m = max(max(int(l), int(u)) for l, u, _ in windows)
    for w in range(1, nw):
        tau[:m, w] = 0.0
        tau[T - m if m else 0:, w] = 0.0
    return float(np.sum(tau * mean ** 2))


def mlpg_ms_chain(mean, var, windows, nu, ms_var, n, n_iter=20, step=1.0, weight=None, trace=None):
    """Generated static trajectory ``(T,)`` of one chain (``mean`` / ``var`` ``(T, nw)``, ``nu`` / ``ms_var``
    ``(n // 2 + 1,)``).  ``trace`` (a list) receives ``(F, accepted, margin)`` of the start point and of every
    trial; ``margin = |F(c') - F(c)| / scale``, with ``scale`` the size of the terms whose rounding bounds the
    difference, so a margin far above 1e-16 means the accept decision cannot flip under rounding.  The margin is
    ``inf`` for the start point and for a trial that moves c by at most 1e-11 of its size, whose decision does not
    matter."""
    Pu, b = build_system(mean, var, windows)
    T = len(b)
    assert T <= n
    q = _precisions(ms_var)
    nu = np.where(q > 0, np.asarray(nu, dtype=np.float64), 0.0)
    omega = float(weight) if weight is not None else 1.0 / (len(windows) * T)
    const = _tau_mu2(mean, var, windows) if trace is not None else 0.0
    cm = solve(Pu, b)
    c = cm.copy()
    f = objective(c, Pu, b, nu, q, n, omega)
    if trace is not None:
        trace.append((f, True, np.inf))
    alpha = float(step)
    for _ in range(int(n_iter)):
        h = solve(Pu, ms_gradient(c, nu, q, n))
        c2 = c + alpha * ((cm - c) + h / omega)
        f2 = objective(c2, Pu, b, nu, q, n, omega)
        ok = f2 >= f
        if trace is not None:
            sc = max(_scale(c, Pu, b, nu, q, n, omega, const), _scale(c2, Pu, b, nu, q, n, omega, const))
            # either decision is safe when the trial leaves c where it is (every bin exempt and c = c_m) or moves it
            # by less than 1e-11 of its size (at a fixed point): both keep c within rounding of that point
            clear = not np.isfinite(f2) or np.abs(c2 - c).max() <= 1e-11 * max(np.abs(c).max(), TINY)
            trace.append((f2, ok, np.inf if clear else abs(f2 - f) / sc))
        if ok:
            c, f = c2, f2
        else:
            alpha *= 0.5
    return c


def mlpg_ms(mean_frames, variance_frames, windows, ms_mean, ms_var, n_iter=20, step=1.0, weight=None, traces=None):
    """``(T, static_dim)`` float64: :func:`mlpg_ms_chain` for every static dimension of one utterance in the
    reference layout (``ms_mean`` / ``ms_var`` ``(n // 2 + 1, static_dim)``).  ``traces`` (a list) receives one
    trace per static dimension."""
    T, D = np.shape(mean_frames)
    sd = D // len(windows)
    ms_mean, ms_var = np.asarray(ms_mean, dtype=np.float64), np.asarray(ms_var, dtype=np.float64)
    n = 2 * (ms_mean.shape[0] - 1)
    out = np.zeros((T, sd))
    for d in range(sd):
        m, v = chain_system(mean_frames, variance_frames, windows, d)
        tr = [] if traces is not None else None
        out[:, d] = mlpg_ms_chain(m, v, windows, ms_mean[:, d], ms_var[:, d], n, n_iter, step, weight, tr)
        if traces is not None:
            traces.append(tr)
    return out


def chain_objective(mean_frames, variance_frames, windows, d, c, ms_mean, ms_var, weight=None):
    """F of trajectory ``c`` of static dimension ``d`` of one utterance (for comparing trajectories of one chain)."""
    m, v = chain_system(mean_frames, variance_frames, windows, d)
    Pu, b = build_system(m, v, windows)
    q = _precisions(ms_var)
    nu = np.where(q > 0, np.asarray(ms_mean, dtype=np.float64), 0.0)
    omega = float(weight) if weight is not None else 1.0 / (len(windows) * len(b))
    return objective(np.asarray(c, dtype=np.float64), Pu, b, nu, q, 2 * (len(q) - 1), omega)
