"""Write gmm_traj_reference_golden.npz from the reference built under oracle/_ref/ (data only).

    python tests/golden/make_gmm_traj_golden.py

For every case of ``cases()`` (T frames, static_dim, number of windows, mixtures, swap, diff) stores the
synthetic joint GMM ``joint_gmm(...)``, the source frames and the reference's ``MLPG(gmm, windows, swap,
diff).transform(src)``: the arg-max-mixture trajectory that the trajectory EM starts from.  Keys are
``<what>_<case index>``.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
WINDOWS = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))]


def em_window_sets():
    """name -> window set the trajectory-EM tests cover: the reference's test sets with a dynamic window
    (tests/conftest.py ``windows_set()[1:4]``: half-width 1 with two and three windows, half-width 2), an
    asymmetric set whose H = 2 comes from ``l`` alone, half-widths 3 and 4, four windows, and a set whose widest
    half-width is 0 (``mlpg`` then drops the dynamic window on every frame)."""
    from conftest import windows_set
    std = windows_set()
    static = (0, 0, np.array([1.0]))
    return {
        "nw2": std[1], "nw3": std[2], "hw2": std[3],
        "asym": [static, (2, 0, np.array([1.0, -4.0, 3.0]) / 2.0), (0, 1, np.array([-1.0, 1.0]))],
        "hw3": [static, (3, 3, np.array([-1.0, 9.0, -45.0, 0.0, 45.0, -9.0, 1.0]) / 60.0)],
        "hw4": [static, (4, 4, np.array([3.0, -32.0, 168.0, -672.0, 0.0, 672.0, -168.0, 32.0, -3.0]) / 840.0),
                (1, 1, np.array([1.0, -2.0, 1.0]))],
        "nw4": std[2] + [(2, 2, np.array([1.0, -8.0, 0.0, 8.0, -1.0]) / 12.0)],
        "h0": [static, (0, 0, np.array([0.5]))],
    }


def half_width(windows):
    """H = max_w max(l_w, u_w): the number of edge frames at each end of an utterance."""
    return max(max(int(l), int(u)) for l, u, _ in windows)


def cases():
    """(T, static_dim, nw, M, swap, diff) of every stored conversion."""
    return [(60, 2, 2, 4, False, False), (45, 3, 3, 3, True, False), (37, 2, 2, 5, False, True),
            (2, 2, 2, 2, True, True)]


def joint_gmm(rng, M, dim):
    """A full-covariance joint GMM over 2 * dim features with well-conditioned covariances, as the attributes
    of a fitted ``sklearn.mixture.GaussianMixture``."""
    A = rng.standard_normal((M, 2 * dim, 2 * dim)) / np.sqrt(2 * dim)
    cov = A @ A.transpose(0, 2, 1) + 0.5 * np.eye(2 * dim)
    w = rng.random(M) + 0.1
    return types.SimpleNamespace(means_=rng.standard_normal((M, 2 * dim)), covariances_=cov, weights_=w / w.sum(),
                                 covariance_type="full")


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from nnmnkwii.baseline.gmm import MLPG
    out = {}
    for i, (T, S, nw, M, swap, diff) in enumerate(cases()):
        rng = np.random.default_rng(100 + i)
        g = joint_gmm(rng, M, S * nw)
        src = rng.standard_normal((T, S * nw))
        out["weights_%d" % i], out["means_%d" % i], out["covariances_%d" % i] = g.weights_, g.means_, g.covariances_
        out["src_%d" % i] = src
        out["y_%d" % i] = MLPG(g, windows=WINDOWS[:nw], swap=swap, diff=diff).transform(src)
    np.savez_compressed(os.path.join(HERE, "gmm_traj_reference_golden.npz"), **out)


if __name__ == "__main__":
    main()
