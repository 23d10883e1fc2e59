"""Float64 NumPy / SciPy restatement of maximum-likelihood GMM trajectory conversion by EM (Toda, Black &
Tokuda 2007, Sec. III) with the diagonal Eq. 23 variances of the reference's ``MLPG.transform``; the checker of
``baseline.gmm.MLPG.transform_em``.  Independent of the package and of the GPU: dense window matrices, one
``np.linalg.solve`` with ``covarXX[m]`` per mixture over the frames, ``scipy.stats.multivariate_normal``,
``scipy.special.logsumexp`` and a dense solve of ``(W^T P W) c = W^T P E`` per static dimension.  For long
utterances ``banded=True`` keeps the window matrices sparse and solves with ``scipy.linalg.solveh_banded``
instead (the dense solve is O(T^3) per static dimension); tests/test_gmm_traj_em_cpu.py checks the two paths
against each other.

Model: ``Y = W c`` (windows zero outside the utterance), ``E_{m,t} = nu_m + Syx_m Sxx_m^-1 (x_t - mu_m)``,
``lp[t, m] = log w_m + log N(x_t; mu_m, Sxx_m)`` and
``L(c) = sum_t logsumexp_m (lp[t, m] + log N(Y_t; E_{m,t}, diag D_m))``, where on the first and last H frames
(H the widest window half-width; every frame when H = 0) only the static columns count, as the reference's
``mlpg`` gives the dynamic windows zero precision there.  ``c_0`` uses the arg-max mixture
of ``lp`` per frame (Eq. 37); each EM iteration takes the posteriors of the current trajectory and solves
with ``P_t = sum_m gamma / D_m`` and ``E_t = (sum_m gamma E_{m,t} / D_m) / P_t``."""
import numpy as np
from scipy import linalg
from scipy import sparse
from scipy.special import logsumexp
from scipy.stats import multivariate_normal


class Model(object):
    """The joint GMM after ``diff`` / ``swap``, as the reference's ``MLPGBase.__init__`` applies them."""

    def __init__(self, gmm, windows, swap=False, diff=False, banded=False):
        D = gmm.means_.shape[1] // 2
        self.windows = windows
        self.banded = banded
        self.static_dim = D // len(windows)
        self.weights = np.asarray(gmm.weights_, dtype=np.float64)
        mx, my = gmm.means_[:, :D], gmm.means_[:, D:]
        cov = gmm.covariances_
        sxx, sxy, syx, syy = cov[:, :D, :D], cov[:, :D, D:], cov[:, D:, :D], cov[:, D:, D:]
        if diff:
            my = my - mx
            syy = sxx + syy - sxy - syx
            sxy = sxy - sxx
            syx = sxy.transpose(0, 2, 1)
        if swap:
            mx, my, sxx, syy, sxy, syx = my, mx, syy, sxx, syx, sxy
        self.mx, self.my, self.sxx, self.sxy, self.syx, self.syy = mx, my, sxx, sxy, syx, syy
        self.Dm = np.stack([np.diag(syy[m]) - np.diag(syx[m]) / np.diag(sxx[m]) * np.diag(sxy[m])
                            for m in range(len(mx))])

    def frame_terms(self, x):
        """(lp (T, M), E (M, T, D)) of source frames x (T, D)."""
        M = len(self.mx)
        lp = np.stack([np.log(self.weights[m]) + np.atleast_1d(multivariate_normal.logpdf(x, self.mx[m], self.sxx[m]))
                       for m in range(M)], axis=1)
        E = np.stack([self.my[m] + (self.syx[m] @ np.linalg.solve(self.sxx[m], (x - self.mx[m]).T)).T
                      for m in range(M)])
        return lp, E

    def window_matrices(self, T):
        """Dense (T, T) matrix of each window: row t holds coef[l + k] at column t + k inside the utterance.
        Sparse (CSR) matrices of the same entries when the model is banded."""
        if self.banded:
            return [sparse.diags([np.full(T - abs(k), float(coef[l + k])) for k in range(-l, u + 1) if abs(k) < T],
                                 [k for k in range(-l, u + 1) if abs(k) < T], shape=(T, T), format="csr")
                    for l, u, coef in self.windows]
        mats = []
        for l, u, coef in self.windows:
            W = np.zeros((T, T))
            for t in range(T):
                for k in range(-l, u + 1):
                    if 0 <= t + k < T:
                        W[t, t + k] = coef[l + k]
            mats.append(W)
        return mats

    def statics_to_y(self, c, mats):
        return np.concatenate([W @ c for W in mats], axis=1)

    def kept(self, T):
        """(T, D) mask of the columns the model keeps: the reference's mlpg gives the dynamic windows zero
        precision on the first and last H frames (H the widest half-width of the window set).  It zeroes them
        with ``precisions[:H]`` and ``precisions[-H:]``, and ``[-0:]`` is the whole column: with H = 0 every
        frame keeps the static columns only."""
        H = max(max(l, u) for l, u, _ in self.windows)
        keep = np.ones((T, len(self.windows) * self.static_dim), dtype=bool)
        if H == 0:
            keep[:, self.static_dim:] = False
            return keep
        keep[:H, self.static_dim:] = False
        keep[max(T - H, 0):, self.static_dim:] = False
        return keep

    def solve(self, mean, var, mats):
        """argmax_c of sum_t log N(W c; mean_t, diag var_t) over the kept columns: (W^T P W) c = W^T P mean per
        static dimension."""
        S = self.static_dim
        T = mean.shape[0]
        keep = self.kept(T)
        c = np.zeros((T, S))
        for s in range(S):
            A = sparse.csr_matrix((T, T)) if self.banded else np.zeros((T, T))
            b = np.zeros(T)
            for w, W in enumerate(mats):
                p = np.where(keep[:, w * S + s], 1.0 / var[:, w * S + s], 0.0)
                A = A + (W.T @ sparse.diags(p) @ W if self.banded else W.T @ (p[:, None] * W))
                b += W.T @ (p * mean[:, w * S + s])
            if self.banded:  # upper form: ab[bw - k, k:] holds the k-th superdiagonal
                bw = max(l + u for l, u, _ in self.windows)
                ab = np.zeros((bw + 1, T))
                for k in range(min(bw, T - 1) + 1):
                    ab[bw - k, k:] = A.diagonal(k)
                c[:, s] = linalg.solveh_banded(ab, b)
            else:
                c[:, s] = linalg.solve(A, b, assume_a="pos")
        return c

    def log_weights(self, lp, E, Y):
        """lp[t, m] + log N(Y_t; E_{m,t}, diag D_m) over the kept columns of frame t, (T, M)."""
        keep = self.kept(len(Y))
        r = Y[None] - E
        terms = r * r / self.Dm[:, None, :] + np.log(self.Dm)[:, None, :] + np.log(2 * np.pi)
        return lp - 0.5 * np.sum(np.where(keep[None], terms, 0.0), axis=2).T


def transform_em(gmm, windows, src, n_iter, swap=False, diff=False, banded=False):
    """(c (T, static_dim), L at c_0 .. c_{n_iter} (n_iter + 1,)) of one utterance; ``banded`` solves with
    sparse window matrices and ``solveh_banded`` instead of dense ones."""
    model = Model(gmm, windows, swap, diff, banded)
    x = np.asarray(src, dtype=np.float64)
    T = len(x)
    lp, E = model.frame_terms(x)
    mats = model.window_matrices(T)
    mix = np.argmax(lp, axis=1)
    c = model.solve(E[mix, np.arange(T)], model.Dm[mix], mats)
    trace = []
    for k in range(n_iter + 1):
        lw = model.log_weights(lp, E, model.statics_to_y(c, mats))
        lse = logsumexp(lw, axis=1)
        trace.append(np.sum(lse))
        if k == n_iter:
            break
        gamma = np.exp(lw - lse[:, None])
        P = gamma @ (1.0 / model.Dm)
        mean = np.einsum("tm,mtd->td", gamma, E / model.Dm[:, None, :]) / P
        c = model.solve(mean, 1.0 / P, mats)
    return c, np.array(trace)
