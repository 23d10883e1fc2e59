"""Write modspec_reference_golden.npz from the reference built under oracle/_ref/ (data only).

    python tests/golden/make_modspec_golden.py

For every DFT length n in NS, T in (1, n // 4 + 1, n - 1, n) frames and norm in (None, "ortho"), on the
trajectory ``trajectory(T, D, seed)`` (D = 1 for T = 1 and T = n, else 3), stores the reference's
  * ``modspec(x, n, norm, return_phase=True)``: power and phase at the bins ``pick(n // 2 + 1)``;
  * ``inv_modspec`` of that power and phase: the n frames at ``pick(n)``;
  * ``modspec_smoothing(x, MODFS, n, norm, CUTOFF, log_domain)``: the T frames at ``pick(T)``, with
    log_domain True, and also False for norm None.
Keys are ``<what>_<n>_<T>_<norm>``.  The inputs are exact integer hashes and running sums (no library
random generator, no libm), so the tests rebuild them bit for bit.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
NS = (256, 512, 1024, 2048, 4096)
MODFS, CUTOFF = 200, 50
NORMS = (None, "ortho")
PICKS = 48


def cases():
    """(n, T, D, seed) of every stored trajectory."""
    out = []
    for n in NS:
        for T in (1, n // 4 + 1, n - 1, n):
            out.append((n, T, 1 if T in (1, n) else 3, len(out)))
    return out


def trajectory(T, D, seed):
    """(T, D) float64: a hashed white sequence in [-1, 1) plus 0.1 times its running sum along time."""
    i = np.arange(T * D, dtype=np.uint64) + np.uint64(seed * 1000003)
    v = ((i * np.uint64(2654435761)) % np.uint64(1 << 32)).astype(np.float64) / 2.0 ** 31 - 1.0
    v = v.reshape(T, D)
    return v + 0.1 * np.cumsum(v, axis=0)


def pick(size):
    """Up to PICKS indices spread over range(size), the first and the last included."""
    return np.unique(np.linspace(0, size - 1, min(size, PICKS)).round().astype(np.int64))


def key(what, n, T, norm):
    return "%s_%d_%d_%s" % (what, n, T, norm or "none")


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from nnmnkwii import preprocessing as P
    out = {}
    for n, T, D, seed in cases():
        x = trajectory(T, D, seed)
        for norm in NORMS:
            ms, phase = P.modspec(x, n=n, norm=norm, return_phase=True)
            kb = pick(n // 2 + 1)
            out[key("ms", n, T, norm)] = ms[kb]
            out[key("phase", n, T, norm)] = phase[kb]
            out[key("inv", n, T, norm)] = P.inv_modspec(ms, phase, norm=norm)[pick(n)]
            out[key("smooth", n, T, norm)] = P.modspec_smoothing(x, MODFS, n=n, norm=norm, cutoff=CUTOFF)[pick(T)]
            if norm is None:
                out[key("smoothlin", n, T, norm)] = P.modspec_smoothing(x, MODFS, n=n, norm=norm, cutoff=CUTOFF,
                                                                        log_domain=False)[pick(T)]
    np.savez_compressed(os.path.join(HERE, "modspec_reference_golden.npz"), **out)


if __name__ == "__main__":
    main()
