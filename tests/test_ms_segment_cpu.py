"""Without a GPU: the segment-level MS post-filter and statistics (postfilters.modspec_post_filter / modspec_statistics
with ``segment=L``) refuse bad arguments before any device work, ``segment=None`` keeps the utterance level's
checks, and the float64 restatement (oracle/ms_segment.py) the GPU tests compare against has the definition's
identities."""
import numpy as np
import pytest

from conftest import rel_err


def _stats(n, D):
    K = n // 2 + 1
    return np.zeros((K, D)), np.ones((K, D))


def test_argument_errors():
    import torch

    from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
    x = np.zeros((10, 2))
    good = _stats(64, 2)

    def pf(**kw):
        return modspec_post_filter(kw.pop("x", x), kw.pop("natural", good), kw.pop("generated", good),
                                   n=kw.pop("n", 64), segment=kw.pop("segment", 50), **kw)

    def st(**kw):
        return modspec_statistics(kw.pop("x", x), n=kw.pop("n", 64), segment=kw.pop("segment", 50), **kw)

    for f in (pf, st):
        # n outside the segment-level set, the utterance level's default 4096 included
        for n in (16, 48, 1024, 4096, 100):
            with pytest.raises(ValueError, match="with segment, n must be one of 32, 64, 128, 256, 512"):
                f(n=n, segment=4)
        for L in (51, 3, 2, 0, -4, 66, 128):
            with pytest.raises(ValueError, match="segment length must be even with 4 <= L <= n"):
                f(segment=L)
        for L in (50.0, "50", True, np.float64(50), [50]):
            with pytest.raises(TypeError, match="segment must be an int"):
                f(segment=L)
        # the input, as at the utterance level
        with pytest.raises(ValueError, match="CPU tensor"):
            f(x=torch.zeros(10, 2))
        with pytest.raises(TypeError, match="float32 or float64"):
            f(x=np.zeros((10, 2), np.int64))
        with pytest.raises(TypeError, match="CUDA tensor or a NumPy array"):
            f(x=[[0.0, 1.0]])
        with pytest.raises(ValueError, match="lengths exceed"):
            f(x=np.zeros((2, 10, 2)), lengths=[11, 3])
        with pytest.raises(ValueError, match="padded"):
            f(lengths=[10])
        with pytest.raises(ValueError, match=r"\(T, D\) or \(B, T, D\)"):
            f(x=np.zeros(10))
    # the filter's range and statistics checks are the utterance level's
    for k in (-0.1, 1.5, float("nan"), float("inf")):
        with pytest.raises(ValueError, match=r"k must be in \[0, 1\]"):
            pf(k=k)
    for bad in (_stats(128, 2), _stats(64, 3), _stats(4096, 2)):
        with pytest.raises(ValueError, match=r"expected \(n // 2 \+ 1, D\)"):
            pf(natural=bad)
        with pytest.raises(ValueError, match=r"expected \(n // 2 \+ 1, D\)"):
            pf(generated=bad)
    m = np.zeros((33, 2))
    m[5, 1] = np.nan
    with pytest.raises(ValueError, match="natural mean is not finite"):
        pf(natural=(m, np.ones((33, 2))))
    v = np.ones((33, 2))
    v[32, 0] = -1.0
    with pytest.raises(ValueError, match="generated var must be finite and >= 0"):
        pf(generated=(np.zeros((33, 2)), v))
    # a set without a segment: no utterance, or only zero-length ones
    for bad in (dict(x=np.zeros((0, 10, 2))), dict(x=np.zeros((0, 2))), dict(x=np.zeros((3, 10, 2)), lengths=[0, 0, 0])):
        with pytest.raises(ValueError, match="at least one segment"):
            st(**bad)


def test_utterance_level_unchanged_without_segment():
    """``segment=None`` keeps refusing what the utterance level refuses: n = 128 and T > n."""
    from nnmnkwii_b200.postfilters import modspec_post_filter, modspec_statistics
    x = np.zeros((10, 2))
    for n in (128, 64, 32):
        with pytest.raises(ValueError, match="n must be one of 256, 512"):
            modspec_statistics(x, n=n)
        with pytest.raises(ValueError, match="n must be one of 256, 512"):
            modspec_post_filter(x, _stats(n, 2), _stats(n, 2), n=n, segment=None)
    with pytest.raises(ValueError, match="shorter than the 300 frames"):
        modspec_statistics(np.zeros((300, 2)), n=256, segment=None)
    with pytest.raises(ValueError, match="shorter than the 300 frames"):
        modspec_post_filter(np.zeros((300, 2)), _stats(256, 2), _stats(256, 2), n=256)
    with pytest.raises(ValueError, match="at least one frame"):
        modspec_statistics(np.zeros((3, 10, 2)), n=256, lengths=[10, 0, 4])


# ---- the restatement ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [4, 10, 50, 64])
def test_segment_counts(L):
    import oracle.ms_segment as O
    from nnmnkwii_b200.postfilters import _segment_counts
    H = L // 2
    Ts = [0, 1, H - 1, H, H + 1, 2 * H, 5000]
    want = [0, 2, 2, 2, 3, 3, -(-5000 // H) + 1]
    for T, w in zip(Ts, want):
        assert O.count(T, L) == w, (T, L)
        assert len(O.segments(np.zeros((T, 1)), L)) == w
    assert list(_segment_counts(Ts, L)) == [O.count(T, L) for T in Ts]


@pytest.mark.parametrize("L", [4, 50, 64])
def test_window_sums_to_one(L):
    """Every frame of [0, T) lies in exactly two segments, whose windows there sum to 1."""
    import oracle.ms_segment as O
    H = L // 2
    w = O.window(L)
    assert rel_err(w[:H] + w[H:], np.ones(H)) <= 1e-15
    for T in (1, H - 1, H, H + 1, 3 * L + 7):
        segs = O.segments(np.ones((T, 1)), L)
        cover = np.zeros(T)
        hits = np.zeros(T, int)
        for j, s in enumerate(segs):
            for m in range(L):
                t = (j - 1) * H + m
                if 0 <= t < T:
                    cover[t] += s[m, 0]
                    hits[t] += 1
        assert (hits == 2).all(), (T, L)
        assert rel_err(cover, np.ones(T)) <= 1e-15, (T, L)


def _corpus(rng, B, T, D, tilt):
    w = rng.standard_normal((B, T + 1, D))
    return 10.0 * (w[:, 1:] + tilt * w[:, :-1])


@pytest.mark.parametrize("n,L", [(64, 50), (32, 4), (128, 128)])
def test_restatement_identities(n, L):
    import oracle.ms_segment as O
    rng = np.random.default_rng(n + L)
    gen = list(_corpus(rng, 3, 300, 3, 0.7))
    nat = list(_corpus(rng, 3, 300, 3, 0.2))
    G, N = O.statistics(gen, n, L), O.statistics(nat, n, L)
    assert G[0].shape == G[1].shape == (n // 2 + 1, 3)
    for x in (gen[0], gen[1][:L // 2 + 1], gen[2][:1]):
        assert rel_err(O.post_filter(x, N, G, 0.0, n, L), x) <= 1e-12  # k = 0: the round trip
        assert rel_err(O.post_filter(x, G, G, 0.6, n, L), x) <= 1e-12  # equal statistics: the round trip
    assert rel_err(O.post_filter(gen[0], N, G, 0.8, n, L), gen[0]) > 1e-3
    # the statistics pool every segment: one utterance's log spectra, stacked
    s = O.log_ms(gen[0], n, L)[0]
    assert len(s) == O.count(300, L)
    M, V = O.statistics(gen[:1], n, L)
    assert rel_err(M, s.mean(0)) <= 1e-15 and rel_err(V, s.var(0)) <= 1e-15
    # a zero-length utterance adds no segment
    M2, V2 = O.statistics(gen[:1] + [np.zeros((0, 3))], n, L)
    assert np.array_equal(M, M2) and np.array_equal(V, V2)
