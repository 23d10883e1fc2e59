"""CPU: the restated SPTK post-filter chain against Merlin's own output, and the argument checks of
postfilters.merlin_post_filter, which must fire without a GPU."""
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle import sptk_postfilter as P


@pytest.fixture(scope="module")
def merlin():
    return np.load(os.path.join(ROOT, "tests", "golden", "merlin_post_filter_golden.npz"))


def test_oracle_reproduces_every_merlin_step(merlin):
    # the reference's tests/test_postfilters.py: alpha 0.58, order 511, fftlen 1024, Merlin's weight file
    r0, p_r0, b0, p_b0, out = P.merlin_post_filter_steps(merlin["mgc"], 0.58, 511, 1024, weight=merlin["weight"])
    assert np.allclose(merlin["mgc_r0"], r0)
    assert np.allclose(merlin["mgc_p_r0"], p_r0)
    assert np.allclose(merlin["mgc_b0"], b0)
    assert np.allclose(merlin["mgc_p_b0"], p_b0)
    assert np.allclose(out, merlin["mgc_p_mgc"], atol=1e-6)
    zero = np.abs(merlin["mgc"]).sum(1) == 0
    assert zero.sum() == 30 and np.all(out[zero] == 0) and np.all(r0[zero] == 1) and np.all(p_r0[zero] == 1)


def test_oracle_chain_collapses_to_weighted_cepstrum(merlin):
    """mc2b and b2mc are exact inverses outside coefficient 0: the chain is w * c plus a column-0 shift."""
    c = merlin["mgc"][:40].astype(np.float64)
    w = np.ones(60) * 1.4
    w[:2] = 1
    r0, p_r0, _, _, out = P.merlin_post_filter_steps(c, 0.41)
    direct = w * c
    direct[:, 0] += np.log(r0 / p_r0) / 2
    assert np.abs(out - direct).max() < 1e-13
    assert np.abs(P.b2mc(P.mc2b(c, 0.41), 0.41) - c).max() < 1e-13


def test_oracle_freqt_is_identity_at_zero_alpha():
    rng = np.random.default_rng(0)
    c = rng.standard_normal((3, 9))
    assert np.array_equal(P.freqt(c, 8, 0.0), c)
    assert np.array_equal(P.freqt(c, 4, 0.0), c[:, :5])
    assert np.array_equal(P.freqt(c, 12, 0.0)[:, 9:], np.zeros((3, 4)))


def _bad_calls():
    mgc = np.zeros((4, 8), np.float32)
    return [
        (ValueError, dict(mgc=np.zeros(8, np.float32))),
        (ValueError, dict(mgc=np.zeros((2, 4, 8), np.float32))),
        (ValueError, dict(mgc=mgc, fftlen=1000)),
        (ValueError, dict(mgc=mgc, fftlen=0)),
        (ValueError, dict(mgc=mgc, fftlen=-8)),
        (ValueError, dict(mgc=mgc, minimum_phase_order=-1)),
        (ValueError, dict(mgc=mgc, minimum_phase_order=1024, fftlen=1024)),
        (ValueError, dict(mgc=mgc, minimum_phase_order=16, fftlen=16)),
        (AssertionError, dict(mgc=mgc, weight=np.ones(7))),
        (AssertionError, dict(mgc=mgc, weight=np.ones(9))),
    ]


@pytest.mark.parametrize("case", range(len(_bad_calls())))
def test_invalid_arguments_raise_without_a_gpu(case):
    from nnmnkwii_b200.postfilters import merlin_post_filter
    exc, kw = _bad_calls()[case]
    mgc = kw.pop("mgc")
    with pytest.raises(exc):
        merlin_post_filter(mgc, 0.41, **kw)


def test_c_abi_rejects_bad_geometry_before_any_launch():
    """Argument errors of the C ABI come back as status codes; nothing is launched (no device needed)."""
    import ctypes
    from nnmnkwii_b200 import _lib
    L = _lib.lib
    n0 = _lib.launch_count()
    p = ctypes.c_void_p(16)  # never dereferenced: every call below fails its checks first
    assert L.nnk_postfilter_basis_elems(60, 1024) == 65 * 4 * 128
    assert L.nnk_postfilter_basis_elems(1, 1) == 128
    assert L.nnk_postfilter_basis_elems(129, 1024) == 0 and L.nnk_postfilter_basis_elems(60, 16384) == 0
    assert L.nnk_postfilter_basis_elems(60, 1000) == 0 and L.nnk_postfilter_basis_elems(0, 1024) == 0
    n = L.nnk_postfilter_basis_elems(60, 1024)
    cases = [
        (L.nnk_postfilter_basis(0.41, 60, 511, 1000, p, n, None), _lib.NNK_ERR_ARG),
        (L.nnk_postfilter_basis(0.41, 60, -1, 1024, p, n, None), _lib.NNK_ERR_ARG),
        (L.nnk_postfilter_basis(0.41, 60, 1024, 1024, p, n, None), _lib.NNK_ERR_ARG),
        (L.nnk_postfilter_basis(0.41, 0, 511, 1024, p, n, None), _lib.NNK_ERR_ARG),
        (L.nnk_postfilter_basis(0.41, 60, 511, 1024, p, n - 1, None), _lib.NNK_ERR_ARG),
        (L.nnk_postfilter_basis(0.41, 60, 511, 1024, None, n, None), _lib.NNK_ERR_ARG),
        (L.nnk_postfilter_basis(0.41, 129, 511, 1024, p, n, None), _lib.NNK_ERR_UNSUPPORTED),
        (L.nnk_postfilter_basis(0.41, 60, 511, 16384, p, n, None), _lib.NNK_ERR_UNSUPPORTED),
        (L.nnk_postfilter_apply(p, 2, 10, 60, 60, p, 1024, p, n, p, 60, None), _lib.NNK_ERR_ARG),
        (L.nnk_postfilter_apply(p, 0, 10, 60, 59, p, 1024, p, n, p, 60, None), _lib.NNK_ERR_ARG),
        (L.nnk_postfilter_apply(p, 0, 10, 60, 60, p, 1024, p, n, p, 59, None), _lib.NNK_ERR_ARG),
        (L.nnk_postfilter_apply(p, 0, -1, 60, 60, p, 1024, p, n, p, 60, None), _lib.NNK_ERR_ARG),
        (L.nnk_postfilter_apply(p, 0, 10, 60, 60, p, 1024, p, n + 128, p, 60, None), _lib.NNK_ERR_ARG),
        (L.nnk_postfilter_apply(p, 0, 10, 60, 60, p, 1023, p, n, p, 60, None), _lib.NNK_ERR_ARG),
        (L.nnk_postfilter_apply(p, 0, 10, 60, 60, None, 1024, p, n, p, 60, None), _lib.NNK_ERR_ARG),
        (L.nnk_postfilter_apply(p, 0, 10, 129, 129, p, 1024, p, n, p, 129, None), _lib.NNK_ERR_UNSUPPORTED),
    ]
    for i, (rc, want) in enumerate(cases):
        assert rc == want, (i, rc, _lib.last_error())
    assert L.nnk_postfilter_apply(p, 0, 0, 60, 60, p, 1024, p, n, p, 60, None) == _lib.NNK_OK  # N = 0: nothing to do
    assert _lib.launch_count() == n0
