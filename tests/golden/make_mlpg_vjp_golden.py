"""Write mlpg_vjp_reference_golden.npz from the reference built under oracle/_ref/ (data only).

    python tests/golden/make_mlpg_vjp_golden.py

For every case of ``cases()`` (window set, T frames, static_dim, global variances) stores means, variances and a
gradient ``go`` with respect to the generated trajectory, and the central differences of the reference's float64
``paramgen.mlpg`` under ``L = sum(go * mlpg(means, variances, windows))`` with respect to every mean and every
variance.  ``L`` is linear in the means, so their differences are exact up to rounding; the variance steps are
``1e-5`` of each variance, which leaves a truncation error near 1e-10 of the gradient.  Keys are
``<what>_<case index>``.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
WINDOW_SETS = {
    "nw3": [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))],
    "hw2": [(0, 0, np.array([1.0])), (2, 2, np.array([1.0, -8.0, 0.0, 8.0, -1.0]) / 12.0),
            (2, 2, np.array([-1.0, 16.0, -30.0, 16.0, -1.0]) / 12.0)],
}


def cases():
    """(window set, T, static_dim, global variances) of every stored case; T = 2 and T = 4 are at most 2 H."""
    return [("nw3", 12, 2, False), ("nw3", 30, 2, False), ("nw3", 30, 2, True), ("hw2", 20, 2, False),
            ("hw2", 4, 2, False), ("nw3", 2, 2, True)]


def inputs(i):
    """Means, variances and go of case i (seeded, so the test can rebuild them as a check)."""
    name, T, sd, var_global = cases()[i]
    D = len(WINDOW_SETS[name]) * sd
    rng = np.random.default_rng(200 + i)
    m = np.cumsum(rng.standard_normal((T, D)), axis=0) * 0.1 + rng.standard_normal((T, D)) * 0.3
    v = (rng.random(D) + 0.5) if var_global else (rng.random((T, D)) + 0.5)
    go = rng.standard_normal((T, sd))
    return m, v, go


def central_differences(mlpg, m, v, windows, go):
    def loss(mm, vv):
        return float(np.sum(go * mlpg(mm, vv, windows)))
    g_m, g_v = np.zeros_like(m), np.zeros_like(v)
    for idx in np.ndindex(m.shape):
        h = 1e-3
        a, b = m.copy(), m.copy()
        a[idx] += h
        b[idx] -= h
        g_m[idx] = (loss(a, v) - loss(b, v)) / (2 * h)
    for idx in np.ndindex(v.shape):
        h = 1e-5 * v[idx]
        a, b = v.copy(), v.copy()
        a[idx] += h
        b[idx] -= h
        g_v[idx] = (loss(m, a) - loss(m, b)) / (2 * h)
    return g_m, g_v


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from nnmnkwii.paramgen import mlpg
    out = {}
    for i, (name, T, sd, var_global) in enumerate(cases()):
        m, v, go = inputs(i)
        out["means_%d" % i], out["variances_%d" % i], out["go_%d" % i] = m, v, go
        out["g_means_%d" % i], out["g_variances_%d" % i] = central_differences(mlpg, m, v, WINDOW_SETS[name], go)
    np.savez_compressed(os.path.join(HERE, "mlpg_vjp_reference_golden.npz"), **out)


if __name__ == "__main__":
    main()
