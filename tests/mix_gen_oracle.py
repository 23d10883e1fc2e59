"""Float64 NumPy / SciPy restatement of parameter generation from per-frame mixtures by EM
(paramgen.mlpg_mixture_batch, DESIGN.md 3.19; Tokuda et al., ICASSP 2000).  TEST INFRASTRUCTURE, NOT PRODUCT.

One utterance of T frames, M components, D input columns laid out in ``streams`` as ``StreamLayout`` takes them:
``(in_col, static_dim)`` for a smoothed stream (window w of static dimension d in column in_col + w static_dim + d)
or ``(in_col, static_dim, "copy")`` for copied columns; output columns follow in the order given.

    Y = W c           per smoothed stream the sparse window matrices of oracle/gmm_traj_em.py (zero outside the
                      utterance); a copied column is its output column itself
    counted columns   on the first and last H = max_w max(l_w, u_w) frames (every frame when H = 0) the static
                      and copied ones, elsewhere every column a stream reads (oracle.gmm_traj_em.Model.kept)
    L(c)              sum_t logsumexp_m (lw[t, m] - 1/2 sum_{counted d} ((Y - mu)^2 / s2 + log s2 + log 2 pi))
    c_0               the component of the largest log-weight per frame (np.argmax), one solve
    EM step           gamma = softmax_m, P = sum_m gamma / s2, E = (sum_m gamma mu / s2) / P, one solve with
                      (E, 1 / P): per smoothed stream the banded solve of oracle/gmm_traj_em.py (its edge rule
                      included), per copied column E itself
"""
import numpy as np
from scipy.special import logsumexp

from oracle.gmm_traj_em import Model


class _Stream(Model):
    """The window matrices, edge rule and banded solve of oracle.gmm_traj_em.Model for one smoothed stream of
    ``static_dim`` columns; no GMM."""

    def __init__(self, windows, static_dim):
        self.windows, self.static_dim, self.banded = windows, static_dim, True


def _parts(windows, streams):
    """[(stream or None for copied, input columns (T-independent), output columns)] of a layout."""
    parts, out = [], 0
    for s in streams:
        in_col, sd = int(s[0]), int(s[1])
        copy = len(s) > 2 and s[2] == "copy"
        nw = 1 if copy else len(windows)
        cols = np.arange(in_col, in_col + nw * sd)
        parts.append((None if copy else _Stream(windows, sd), cols, np.arange(out, out + sd)))
        out += sd
    return parts, out


class Problem(object):
    """One utterance: log-weights (T, M), means and variances (T, M, D)."""

    def __init__(self, log_weights, means, variances, windows, streams=None):
        self.lw = np.asarray(log_weights, dtype=np.float64)
        self.mu = np.asarray(means, dtype=np.float64)
        self.s2 = np.asarray(variances, dtype=np.float64)
        self.T, self.M, self.D = self.mu.shape
        if streams is None:
            streams = [(0, self.D // len(windows))]
        self.parts, self.D_out = _parts(windows, streams)
        self.mats = [None if st is None else st.window_matrices(self.T) for st, _, _ in self.parts]
        self.counted = np.zeros((self.T, self.D), dtype=bool)
        for st, cols, _ in self.parts:
            self.counted[:, cols] = True if st is None else st.kept(self.T)

    def y(self, c):
        """Y = W c, (T, D); columns no stream reads are 0."""
        Y = np.zeros((self.T, self.D))
        for (st, cols, oc), mats in zip(self.parts, self.mats):
            Y[:, cols] = c[:, oc] if st is None else st.statics_to_y(c[:, oc], mats)
        return Y

    def log_weights(self, c):
        """lw[t, m] + log N(Y_t; mu_{t,m}, diag s2_{t,m}) over the counted columns, (T, M)."""
        r = self.y(c)[:, None, :] - self.mu
        terms = r * r / self.s2 + np.log(self.s2) + np.log(2 * np.pi)
        return self.lw - 0.5 * np.sum(np.where(self.counted[:, None, :], terms, 0.0), axis=2)

    def objective(self, c):
        return float(np.sum(logsumexp(self.log_weights(c), axis=1)))

    def solve(self, mean, var):
        """The MLPG solve of every stream with per-frame (T, D) means and variances, (T, D_out)."""
        c = np.zeros((self.T, self.D_out))
        for (st, cols, oc), mats in zip(self.parts, self.mats):
            c[:, oc] = mean[:, cols] if st is None else st.solve(mean[:, cols], var[:, cols], mats)
        return c

    def start(self):
        mix = np.argmax(self.lw, axis=1)
        t = np.arange(self.T)
        return self.solve(self.mu[t, mix], self.s2[t, mix])

    def step(self, c):
        lw = self.log_weights(c)
        gamma = np.exp(lw - logsumexp(lw, axis=1)[:, None])
        P = np.einsum("tm,tmd->td", gamma, 1.0 / self.s2)
        E = np.einsum("tm,tmd->td", gamma, self.mu / self.s2) / P
        return self.solve(E, 1.0 / P)


def mlpg_mixture(log_weights, means, variances, windows, n_iter, streams=None, trace=None):
    """(c (T, D_out), L at c_0 .. c_n_iter (n_iter + 1,)) of one utterance; ``trace`` (a list) receives every
    c_k."""
    p = Problem(log_weights, means, variances, windows, streams)
    c = p.start()
    L = [p.objective(c)]
    if trace is not None:
        trace.append(c)
    for _ in range(n_iter):
        c = p.step(c)
        L.append(p.objective(c))
        if trace is not None:
            trace.append(c)
    return c, np.array(L)
