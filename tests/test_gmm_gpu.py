"""GMM-based conversion in front of MLPG (SURVEY.md section 8f row 1): nnmnkwii_b200.baseline.gmm vs
outputs of the reference's nnmnkwii.baseline.gmm on the same fitted GMM (tests/golden/make_golden.py).
float64 throughout, like the reference; tolerance 1e-9 relative (different but equivalent algebra:
A = Sigma_yx Sigma_xx^-1 is formed once instead of one solve per frame)."""
import types

import numpy as np
import pytest

from conftest import rel_err, windows_set

pytestmark = pytest.mark.gpu


def _gmm(golden):
    return types.SimpleNamespace(means_=golden["gmm_means"], covariances_=golden["gmm_covars"],
                                 weights_=golden["gmm_weights"], covariance_type="full")


def test_gmm_mlpg_matches_reference_golden(golden):
    from nnmnkwii_b200.baseline.gmm import MLPG, MLPGBase
    gmm, src = _gmm(golden), golden["gmm_src"]
    w3 = windows_set()[2]
    static = [(0, 0, np.array([1.0]))]
    cases = [("gmm_default", MLPG(gmm)), ("gmm_w3", MLPG(gmm, windows=w3)), ("gmm_w3_diff", MLPG(gmm, windows=w3, diff=True)),
             ("gmm_w3_swap", MLPG(gmm, windows=w3, swap=True)), ("gmm_static", MLPG(gmm, windows=static))]
    for key, conv in cases:
        y = conv.transform(src)
        assert y.shape == golden[key].shape and y.dtype == golden[key].dtype
        assert rel_err(y, golden[key]) < 1e-9, key
    y32 = MLPG(gmm, windows=static).transform(src.astype(np.float32))
    assert y32.dtype == np.float32 and rel_err(y32, golden["gmm_static_f32"]) < 1e-6
    assert rel_err(MLPGBase(gmm, diff=True).transform(src), golden["gmm_base_2d"]) < 1e-9
    y1 = MLPGBase(gmm).transform(src[3])
    assert y1.shape == (12,) and rel_err(y1, golden["gmm_base_1d"]) < 1e-9
    # batched form == per-utterance form
    conv = MLPG(gmm, windows=w3)
    parts = [src[:7], src[7:8], src[8:40], src[40:]]
    for got, part in zip(conv.transform_batch(parts), parts):
        assert rel_err(got, conv.transform(part)) < 1e-12
    assert conv.transform_batch([]) == []


def test_gmm_kernels_at_voice_conversion_size():
    """The fused GMM kernels (log-posteriors, arg-max map, posterior mean) at a realistic size --
    32 mixtures over 72-dim (static + delta) frames, two dims that do not fill the last lane group --
    against the reference's own per-frame algebra written out in NumPy float64 (gmm.py:97-121, 219-244)."""
    from nnmnkwii_b200.baseline.gmm import MLPG, MLPGBase
    from test_kernel_variants_gmm_gpu import gmm_map_reference
    for M, dim, T in ((32, 72, 333), (3, 5, 17), (7, 96, 40)):
        rng = np.random.default_rng(M * 1000 + dim)
        A = rng.standard_normal((M, 2 * dim, 2 * dim)) / np.sqrt(2 * dim)
        cov = A @ A.transpose(0, 2, 1) + 0.5 * np.eye(2 * dim)
        w = rng.random(M) + 0.1
        gmm = types.SimpleNamespace(means_=rng.standard_normal((M, 2 * dim)), covariances_=cov, weights_=w / w.sum(),
                                    covariance_type="full")
        src = rng.standard_normal((T, dim))
        base = MLPGBase(gmm)
        lp, Em, want, Dm = gmm_map_reference(base, src)  # reference algebra, frame by frame
        assert rel_err(base.transform(src), want) < 1e-9
        conv = MLPG(gmm, windows=[(0, 0, np.array([1.0]))] * 1)
        conv.static_dim = dim // 2  # force the E / D path (feature_dim != static_dim)
        import torch
        x, c = conv._to_device(src)
        E, Dv = conv._means_vars(x, c)
        mix = lp.argmax(1)
        assert rel_err(E.cpu().numpy(), Em[np.arange(T), mix]) < 1e-9
        assert np.array_equal(Dv.cpu().numpy(), Dm[mix])
        del torch
