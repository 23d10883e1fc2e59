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
