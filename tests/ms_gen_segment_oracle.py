"""Float64 NumPy / SciPy restatement of parameter generation considering the segment-level modulation spectrum
(paramgen.mlpg_ms_batch(segment=L), DESIGN.md 3.18).  TEST INFRASTRUCTURE, NOT PRODUCT.

The utterance-level restatement (oracle/ms_gen.py) with its MS term replaced by the mean over the segments of the
segment-level post-filter (oracle/ms_segment.py).  One chain = one static dimension of one utterance of T >= 1
frames, any T:

    tau, P, b  exactly as paramgen.mlpg builds them (oracle.gv.build_system), c_m = P^-1 b
    segments   H = L / 2, J = ceil(T / H) + 1, segment j = c[(j - 1) H : (j - 1) H + L] (zeros outside [0, T)),
               times the periodic Hann window w (oracle.ms_segment.segments)
    Y_j        = numpy.fft.rfft(segment j, n),  s_jk = log(max(|Y_jk|^2, tiny))
    F(c)       = omega (b^T c - c^T P c / 2) - 1/(2 J) sum_j sum_{k=1}^{n/2} q_k (s_jk - nu_k)^2
    gradient   g_t = 1/J sum_{j containing t} w_m [n irfft(C_j, n)]_m,  t = (j - 1) H + m,
               C_jk = -q_k (s_jk - nu_k) / |Y_jk|^2 Y_jk  (C_j0 = 0, C_j,n/2 doubled, 0 for power <= tiny)
    trials     as oracle.ms_gen.mlpg_ms_chain: h = P^-1 g, c' = c + alpha ((c_m - c) + h / omega), kept when
               F(c') >= F(c), otherwise alpha halves

The banded solves go through scipy.linalg.solveh_banded (oracle.gv.solve).
"""
import numpy as np

from oracle.gv import band_matvec, build_system, chain_system, solve
from oracle.ms_gen import TINY, _precisions, _tau_mu2
from oracle.ms_segment import count, segments, window


def _spectra(c, n, L):
    """``(Y, P)`` of every windowed segment of trajectory ``c``, ``(J, n // 2 + 1)`` each."""
    Y = np.fft.rfft(segments(np.asarray(c, dtype=np.float64)[:, None], L)[:, :, 0], n, axis=1)
    return Y, Y.real ** 2 + Y.imag ** 2


def ms_term(c, nu, q, n, L):
    """-1/(2 J) sum_j sum_{k >= 1} q_k (s_jk - nu_k)^2 of trajectory ``c``."""
    _, p = _spectra(c, n, L)
    s = np.log(np.maximum(p, TINY))
    on = q > 0
    on[0] = False
    return float(-0.5 * np.sum(q[on] * (s[:, on] - nu[on]) ** 2) / len(p))


def ms_gradient(c, nu, q, n, L):
    """Analytic gradient of :func:`ms_term` (the closed form above)."""
    T = len(c)
    H = L // 2
    Y, p = _spectra(c, n, L)
    J = len(Y)
    on = (q > 0)[None, :] & (p > TINY)
    on[:, 0] = False
    G = np.zeros_like(p)
    G[on] = -np.broadcast_to(q, p.shape)[on] * (np.log(p[on]) - np.broadcast_to(nu, p.shape)[on]) / p[on]
    C = G * Y
    C[:, -1] *= 2.0  # irfft counts bin n / 2 once, the other bins twice
    R = n * np.fft.irfft(C, n, axis=1)[:, :L] * window(L)
    g = np.zeros((J + 1) * H)  # frames -H .. J H - 1
    for j in range(J):
        g[j * H:j * H + L] += R[j]
    return g[H:H + T] / J


def objective(c, Pu, b, nu, q, n, L, omega):
    c = np.asarray(c, dtype=np.float64)
    return float(omega * (b @ c - 0.5 * c @ band_matvec(Pu, c)) + ms_term(c, nu, q, n, L))


def _scale(c, Pu, b, nu, q, n, L, omega, const):
    """Size of the terms whose rounding bounds an F difference (oracle.ms_gen._scale with this MS term)."""
    return omega * (abs(b @ c) + 0.5 * abs(c @ band_matvec(Pu, c)) + 0.5 * const) - ms_term(c, nu, q, n, L)


def mlpg_ms_chain(mean, var, windows, nu, ms_var, n, L, n_iter=20, step=1.0, weight=None, trace=None, follow=None,
                  floor=1e-9):
    """Generated static trajectory ``(T,)`` of one chain; ``trace`` as oracle.ms_gen.mlpg_ms_chain's.

    ``follow`` (booleans, one per trial) replaces the decision of every trial whose margin is at most ``floor``
    or infinite: such a trial changes F by less than rounding can resolve (or moves c by at most 1e-11 of its
    size), so either decision is a valid path, and a caller that knows which one the device took follows it;
    the two decisions leave different step sizes for the later trials.  The trace keeps the restatement's own
    decision."""
    Pu, b = build_system(mean, var, windows)
    T = len(b)
    q = _precisions(ms_var)
    nu = np.where(q > 0, np.asarray(nu, dtype=np.float64), 0.0)
    omega = float(weight) if weight is not None else 1.0 / (len(windows) * T)
    const = _tau_mu2(mean, var, windows) if trace is not None else 0.0
    cm = solve(Pu, b)
    c = cm.copy()
    f = objective(c, Pu, b, nu, q, n, L, omega)
    if trace is not None:
        trace.append((f, True, np.inf))
    alpha = float(step)
    for _ in range(int(n_iter)):
        h = solve(Pu, ms_gradient(c, nu, q, n, L))
        c2 = c + alpha * ((cm - c) + h / omega)
        f2 = objective(c2, Pu, b, nu, q, n, L, omega)
        ok = f2 >= f
        if trace is not None:
            sc = max(_scale(c, Pu, b, nu, q, n, L, omega, const), _scale(c2, Pu, b, nu, q, n, L, omega, const))
            clear = not np.isfinite(f2) or np.abs(c2 - c).max() <= 1e-11 * max(np.abs(c).max(), TINY)
            margin = np.inf if clear else abs(f2 - f) / sc
            trace.append((f2, ok, margin))
            if follow is not None and (margin <= floor or margin == np.inf):
                ok = bool(follow[len(trace) - 2])
        if ok:
            c, f = c2, f2
        else:
            alpha *= 0.5
    return c


def mlpg_ms(mean_frames, variance_frames, windows, ms_mean, ms_var, L, n_iter=20, step=1.0, weight=None,
            traces=None, follow=None):
    """``(T, static_dim)`` float64: :func:`mlpg_ms_chain` for every static dimension of one utterance in the
    reference layout (``ms_mean`` / ``ms_var`` ``(n // 2 + 1, static_dim)``); ``follow[d]`` is chain d's."""
    T, D = np.shape(mean_frames)
    sd = D // len(windows)
    ms_mean, ms_var = np.asarray(ms_mean, dtype=np.float64), np.asarray(ms_var, dtype=np.float64)
    n = 2 * (ms_mean.shape[0] - 1)
    out = np.zeros((T, sd))
    for d in range(sd):
        m, v = chain_system(mean_frames, variance_frames, windows, d)
        tr = [] if traces is not None or follow is not None else None
        out[:, d] = mlpg_ms_chain(m, v, windows, ms_mean[:, d], ms_var[:, d], n, L, n_iter, step, weight, tr,
                                  None if follow is None else follow[d])
        if traces is not None:
            traces.append(tr)
    return out


def chain_objective(mean_frames, variance_frames, windows, d, c, ms_mean, ms_var, L, weight=None):
    """F of trajectory ``c`` of static dimension ``d`` of one utterance."""
    m, v = chain_system(mean_frames, variance_frames, windows, d)
    Pu, b = build_system(m, v, windows)
    q = _precisions(ms_var)
    nu = np.where(q > 0, np.asarray(ms_mean, dtype=np.float64), 0.0)
    omega = float(weight) if weight is not None else 1.0 / (len(windows) * len(b))
    return objective(np.asarray(c, dtype=np.float64), Pu, b, nu, q, 2 * (len(q) - 1), L, omega)


__all__ = ["count", "ms_term", "ms_gradient", "objective", "mlpg_ms_chain", "mlpg_ms", "chain_objective"]
