"""Without a GPU: postfilters.modspec_post_filter / modspec_statistics refuse bad arguments before any device work,
and the float64 restatement (oracle/ms_postfilter.py) the GPU tests compare against has the MS of the reference
and the filter's identities."""
import importlib.util
import os

import numpy as np
import pytest

from conftest import ROOT, rel_err

_spec = importlib.util.spec_from_file_location("make_modspec_golden",
                                               os.path.join(ROOT, "tests", "golden", "make_modspec_golden.py"))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)


def _stats(n, D, shift=0.0):
    K = n // 2 + 1
    return np.zeros((K, D)) + shift, np.ones((K, D))


def test_argument_errors():
    import torch

    from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
    x = np.zeros((10, 2))
    good = _stats(256, 2)
    pf = (lambda **kw: modspec_post_filter(kw.pop("x", x), kw.pop("natural", good), kw.pop("generated", good),
                                           n=kw.pop("n", 256), **kw))
    for n in (100, 128, 8192, 300):
        with pytest.raises(ValueError, match="n must be one of"):
            modspec_statistics(x, n=n)
        with pytest.raises(ValueError, match="n must be one of"):
            pf(n=n)
    with pytest.raises(ValueError, match="shorter than the 300 frames"):
        modspec_statistics(np.zeros((300, 2)), n=256)
    with pytest.raises(ValueError, match="shorter than the 300 frames"):
        pf(x=np.zeros((300, 2)))
    with pytest.raises(ValueError, match="shorter than the 300 frames"):
        pf(x=np.zeros((2, 400, 2)), lengths=[300, 10])
    for k in (-0.1, 1.5, float("nan"), float("inf")):
        with pytest.raises(ValueError, match=r"k must be in \[0, 1\]"):
            pf(k=k)
    # statistics of another n or another D
    for bad in (_stats(512, 2), _stats(256, 3), (np.zeros((129, 2)), np.ones((129, 3))), (np.zeros(129), np.ones(129))):
        with pytest.raises(ValueError, match=r"expected \(n // 2 \+ 1, D\)"):
            pf(natural=bad)
        with pytest.raises(ValueError, match=r"expected \(n // 2 \+ 1, D\)"):
            pf(generated=bad)
    for which in ("natural", "generated"):
        for v in (np.nan, np.inf, -np.inf):
            m = np.zeros((129, 2))
            m[3, 1] = v
            with pytest.raises(ValueError, match="%s mean is not finite" % which):
                pf(**{which: (m, np.ones((129, 2)))})
        for v in (-1e-300, -1.0, np.nan, np.inf):
            var = np.ones((129, 2))
            var[128, 0] = v
            with pytest.raises(ValueError, match="%s var must be finite and >= 0" % which):
                pf(**{which: (np.zeros((129, 2)), var)})
        with pytest.raises(TypeError, match="pair"):
            pf(**{which: np.zeros((129, 2))})
        with pytest.raises(ValueError, match="CPU tensor"):
            pf(**{which: (torch.zeros(129, 2, dtype=torch.float64), torch.ones(129, 2, dtype=torch.float64))})
        with pytest.raises(TypeError, match="float32 or float64"):
            pf(**{which: (np.zeros((129, 2), np.int64), np.ones((129, 2)))})
    # zero-length utterances: refused by the statistics (no MS), allowed by the filter (checked on the GPU)
    with pytest.raises(ValueError, match="at least one frame"):
        modspec_statistics(np.zeros((3, 10, 2)), n=256, lengths=[10, 0, 4])
    with pytest.raises(ValueError, match="at least one frame"):
        modspec_statistics(np.zeros((0, 2)), n=256)
    with pytest.raises(ValueError, match="at least one utterance"):
        modspec_statistics(np.zeros((0, 10, 2)), n=256)
    # the input, as for preprocessing.modspec
    for f in (lambda a, **kw: modspec_statistics(a, n=256, **kw), lambda a, **kw: pf(x=a, **kw)):
        with pytest.raises(ValueError, match="CPU tensor"):
            f(torch.zeros(10, 2))
        with pytest.raises(TypeError, match="float32 or float64"):
            f(np.zeros((10, 2), np.int64))
        with pytest.raises(TypeError, match="CUDA tensor or a NumPy array"):
            f([[0.0, 1.0]])
        with pytest.raises(ValueError, match="lengths exceed"):
            f(np.zeros((2, 10, 2)), lengths=[11, 3])
        with pytest.raises(ValueError, match="padded"):
            f(x, lengths=[10])
        with pytest.raises(ValueError, match=r"\(T, D\) or \(B, T, D\)"):
            f(np.zeros(10))


def test_restated_log_ms_is_the_log_of_the_reference_modspec():
    import oracle.ms_postfilter as O
    golden = np.load(os.path.join(ROOT, "tests", "golden", "modspec_reference_golden.npz"))
    for n, T, D, seed in MG.cases():
        s, _, _ = O.log_ms(MG.trajectory(T, D, seed), n)
        kb = MG.pick(n // 2 + 1)
        assert rel_err(s[kb], np.log(golden[MG.key("ms", n, T, None)])) <= 1e-12, (n, T)


def _corpus(rng, B, T, D, smooth):
    """B utterances of T frames: white noise plus a random walk, low-passed by a moving average of ``smooth``."""
    out = []
    for _ in range(B):
        x = rng.standard_normal((T + smooth - 1, D)) + 0.05 * rng.standard_normal((T + smooth - 1, D)).cumsum(0)
        out.append(np.stack([np.convolve(x[:, d], np.ones(smooth) / smooth, "valid") for d in range(D)], axis=1))
    return out


@pytest.mark.parametrize("n", [256, 1024])
def test_restatement_identities(n):
    import oracle.ms_postfilter as O
    rng = np.random.default_rng(n)
    D = 3
    gen = _corpus(rng, 6, n, D, 4)
    G = O.statistics(gen, n)
    N = O.statistics(_corpus(rng, 6, n, D, 1), n)
    for x in (gen[0], gen[1][: n // 3 + 1]):
        assert rel_err(O.post_filter(x, N, G, 0.0, n), x) <= 1e-12  # k = 0: the round trip
        assert rel_err(O.post_filter(x, G, G, 0.6, n), x) <= 1e-12  # natural == generated: the round trip
        assert rel_err(O.post_filter(x, N, G, 0.5, n), x) > 1e-3
    # every T = n, k = 1, the generated statistics those of the input: the output has the natural statistics on
    # bins 1 .. n / 2, and bin 0's statistics are those of the input
    out = [O.post_filter(u, N, G, 1.0, n) for u in gen]
    M, V = O.statistics(out, n)
    assert rel_err(M[1:], N[0][1:]) <= 1e-10 and rel_err(V[1:], N[1][1:]) <= 1e-10
    assert rel_err(M[0], G[0][0]) <= 1e-12 and rel_err(V[0], G[1][0]) <= 1e-10
