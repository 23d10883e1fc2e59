"""CPU: the workspace layout of the GMM EM (csrc/nnk_gmm_em.cu) and the size limits of the GMM mapping
(csrc/nnk_gmm.cu) against tests/variant_mirror.py.  The library loads without a GPU and these calls launch
nothing, so a change to `em_layout` or to a limit fails here as well as in the GPU variant tests."""
import ctypes

import pytest

import variant_mirror as M


@pytest.mark.parametrize("K", [1, 33, 128])
@pytest.mark.parametrize("D", [1, 16, 17, 128])
def test_em_layout_mirror_matches_workspace_bytes(D, K):
    from nnmnkwii_b200 import _lib
    for N in (1, 31, 32, 33, 255, 256, 1023, 1024, 1025, 10 ** 5):
        L = M.em_layout(N, D, K)
        assert L["total"] * 8 == _lib.lib.nnk_gmm_em_workspace_bytes(N, D, K), (N, D, K, L)
        # every frame in exactly one tile / chunk, and no empty covariance chunk
        assert (L["n_tiles"] - 1) * M.EM_ES_FT < N <= L["n_tiles"] * M.EM_ES_FT
        assert (L["n_stat"] - 1) * M.EM_ST_CHUNK < N <= L["n_stat"] * M.EM_ST_CHUNK
        assert L["cov_chunk"] % M.EM_CV_SUB == 0
        assert (L["n_cov"] - 1) * L["cov_chunk"] < N <= L["n_cov"] * L["cov_chunk"]


def test_em_workspace_bytes_is_zero_outside_the_limits():
    from nnmnkwii_b200 import _lib
    ws = _lib.lib.nnk_gmm_em_workspace_bytes
    assert ws(1000, M.EM_MAX_D, M.EM_MAX_K) > 0
    for N, D, K in ((0, 4, 2), (-1, 4, 2), (1000, 0, 2), (1000, M.EM_MAX_D + 1, 2), (1000, 4, 0),
                    (1000, 4, M.EM_MAX_K + 1)):
        assert ws(N, D, K) == 0, (N, D, K)


def _gmm_call(fn_name, Mx, D):
    """``nnk_gmm_logprob`` / ``nnk_gmm_map`` with T = 0: the argument checks run, nothing is launched and
    no pointer is dereferenced (the tables point at a host dummy)."""
    from nnmnkwii_b200 import _lib
    dummy = (ctypes.c_double * 4)()
    p = ctypes.cast(dummy, ctypes.c_void_p).value
    g = _lib.NnkGmm()
    for name in ("src_means", "tgt_means", "prec_chol", "log_const", "A_t", "Dm"):
        setattr(g, name, p)
    g.M, g.D = Mx, D
    if fn_name == "nnk_gmm_logprob":
        return _lib.lib.nnk_gmm_logprob(ctypes.byref(g), p, D, 0, p, None)
    return _lib.lib.nnk_gmm_map(ctypes.byref(g), p, D, 0, p, 0, p, p, None, None)


@pytest.mark.parametrize("fn_name", ["nnk_gmm_logprob", "nnk_gmm_map"])
def test_gmm_mapping_size_limits(fn_name):
    from nnmnkwii_b200 import _lib
    n0 = _lib.launch_count()
    assert _gmm_call(fn_name, M.GMM_MAX_M, M.GMM_MAX_D) == _lib.NNK_OK
    assert _gmm_call(fn_name, M.GMM_MAX_M + 1, 4) == _lib.NNK_ERR_UNSUPPORTED
    assert "65535" in _lib.last_error()
    assert _gmm_call(fn_name, 4, M.GMM_MAX_D + 1) == _lib.NNK_ERR_UNSUPPORTED
    assert "96" in _lib.last_error()
    assert _gmm_call(fn_name, 0, 4) == _lib.NNK_ERR_ARG
    assert _lib.launch_count() == n0
