"""Parameter generation considering global variance on the GPU (nnk_mlpg_gv, nnk_segment_moments) against
the float64 restatement in oracle/gv.py: every window-set instance, float32 and float64, per-frame and global
variances, T = 1 / T <= 2 max_win_width / T = 2000, padded and flat batches, the Merlin layout, determinism,
the GV statistics and baseline.gmm.MLPG(gv=...)."""
import numpy as np
import pytest

from conftest import windows_set

import oracle.gv as ogv

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from nnmnkwii_b200 import paramgen as G  # noqa: E402


def _m_edge(w):
    return max(max(l, u) for l, u, _ in w)


def _data(rng, lens, D, dtype, var_global):
    n = int(np.sum(lens))
    m = np.cumsum(rng.standard_normal((n, D)), axis=0) * 0.05 + rng.standard_normal((n, D)) * 0.3
    v = (rng.random(D) + 0.5) if var_global else (rng.random((n, D)) + 0.5)
    return m.astype(dtype), v.astype(dtype)


def _gv_params(rng, m, v, w, lens, sd):
    """gv_mean a few times the c_m variance of the first utterance, so the GV term pulls hard."""
    T0 = lens[0]
    cm = ogv.mlpg(m[:T0], v if v.ndim == 1 else v[:T0], w)
    vm = cm.var(axis=0) + 1e-3
    gm = vm * (1.5 + 2.5 * rng.random(sd))
    gvv = (0.2 * gm) ** 2 * (0.5 + rng.random(sd))
    return gm, gvv


def _check_utt(y, m, v, w, gm, gvv, f32, n_iter=20, step=1.0, weight=None):
    ref = ogv.mlpg_gv(m, v, w, gm, gvv, n_iter, step, weight)
    scale = max(1e-300, np.abs(ref).max())
    err = np.abs(y.astype(np.float64) - ref).max() / scale
    if f32:
        assert err <= 1e-5, err
        return
    assert err <= 1e-8, err
    for d in range(ref.shape[1]):
        fr = ogv.chain_objective(m, v, w, d, ref[:, d], gm[d], gvv[d], weight)
        fy = ogv.chain_objective(m, v, w, d, y[:, d], gm[d], gvv[d], weight)
        assert abs(fy - fr) <= 1e-10 * max(abs(fr), 1e-300), (d, fy, fr)


@pytest.mark.parametrize("wi", range(4))
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("var_global", [False, True])
def test_matches_oracle_every_instance(wi, dtype, var_global):
    w = windows_set()[wi]
    rng = np.random.default_rng(100 * wi + 10 * var_global + (dtype == np.float32))
    sd = 5
    lens = [157, 1, max(2, 2 * _m_edge(w)), 40]
    m, v = _data(rng, lens, len(w) * sd, dtype, var_global)
    gm, gvv = _gv_params(rng, m, v, w, lens, sd)
    y = G.mlpg_gv_batch(m, v, w, gm, gvv, lengths=lens)
    assert y.dtype == dtype and y.shape == (sum(lens), sd)
    off = np.concatenate([[0], np.cumsum(lens)])
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        _check_utt(y[a:b], m[a:b], v if var_global else v[a:b], w, gm, gvv, dtype == np.float32)


def test_long_utterance_and_options():
    w = windows_set()[2]
    rng = np.random.default_rng(7)
    sd = 4
    lens = [2000]
    m, v = _data(rng, lens, 3 * sd, np.float64, False)
    gm, gvv = _gv_params(rng, m, v, w, lens, sd)
    _check_utt(G.mlpg_gv(m, v, w, gm, gvv), m, v, w, gm, gvv, False)
    for kw in (dict(n_iter=0), dict(n_iter=7, step=0.25), dict(n_iter=10, weight=1e-3)):
        _check_utt(G.mlpg_gv(m, v, w, gm, gvv, **kw), m, v, w, gm, gvv, False, **kw)


def test_padded_flat_batch_and_repeat_are_bit_identical():
    w = windows_set()[2]
    rng = np.random.default_rng(8)
    sd = 7
    lens = [60, 3, 1, 121, 33]
    m, v = _data(rng, lens, 3 * sd, np.float64, False)
    gm, gvv = _gv_params(rng, m, v, w, lens, sd)
    flat = G.mlpg_gv_batch(m, v, w, gm, gvv, lengths=lens)
    again = G.mlpg_gv_batch(m, v, w, gm, gvv, offsets=np.concatenate([[0], np.cumsum(lens)]))
    assert np.array_equal(flat, again)
    Tmax = max(lens)
    pm = np.zeros((len(lens), Tmax, 3 * sd))
    pv = np.ones((len(lens), Tmax, 3 * sd))
    off = np.concatenate([[0], np.cumsum(lens)])
    for u, T in enumerate(lens):
        pm[u, :T], pv[u, :T] = m[off[u]:off[u + 1]], v[off[u]:off[u + 1]]
    padded = G.mlpg_gv_batch(pm, pv, w, gm, gvv, lengths=lens)
    dev = G.mlpg_gv_batch(torch.from_numpy(pm).cuda(), torch.from_numpy(pv).cuda(), w, gm, gvv, lengths=lens)
    assert np.array_equal(padded, dev.cpu().numpy())
    for u, T in enumerate(lens):
        one = G.mlpg_gv(m[off[u]:off[u + 1]], v[off[u]:off[u + 1]], w, gm, gvv)
        assert np.array_equal(flat[off[u]:off[u + 1]], one)
        assert np.array_equal(padded[u, :T], one) and not padded[u, T:].any()


def test_merlin_layout_per_column_gv():
    w = windows_set()[2]
    rng = np.random.default_rng(9)
    lay = G.merlin_layout()
    lens = [90, 45]
    for dtype in (np.float64, np.float32):
        m, v = _data(rng, lens, 187, dtype, False)
        gm = np.zeros(63)
        gvv = np.ones(63)
        gm[:60], gvv[:60] = _gv_params(rng, m[:, :180], v[:, :180], w, lens, 60)
        for col, c0 in ((60, 180), (62, 184)):
            gm[col:col + 1], gvv[col:col + 1] = _gv_params(rng, m[:, c0:c0 + 3], v[:, c0:c0 + 3], w, lens, 1)
        gm[61], gvv[61] = np.nan, -1.0  # vuv is copied: its entries are ignored
        y = G.mlpg_gv_batch(m, v, w, gm, gvv, lengths=lens, layout=lay)
        off = np.concatenate([[0], np.cumsum(lens)])
        for u in range(len(lens)):
            a, b = off[u], off[u + 1]
            f32 = dtype == np.float32
            _check_utt(y[a:b, :60], m[a:b, :180], v[a:b, :180], w, gm[:60], gvv[:60], f32)
            _check_utt(y[a:b, 60:61], m[a:b, 180:183], v[a:b, 180:183], w, gm[60:61], gvv[60:61], f32)
            _check_utt(y[a:b, 62:63], m[a:b, 184:187], v[a:b, 184:187], w, gm[62:63], gvv[62:63], f32)
            assert np.array_equal(y[a:b, 61], m[a:b, 183])


def test_not_positive_definite_raises_like_mlpg():
    w = windows_set()[2]
    rng = np.random.default_rng(10)
    m, v = _data(rng, [50, 30], 6, np.float64, False)
    v[60, 1] = -1e-3  # utterance 1, frame 10, static dimension 1: a negative pivot
    with pytest.raises(np.linalg.LinAlgError) as e_ref:
        G.mlpg_batch(m, v, w, lengths=[50, 30])
    with pytest.raises(np.linalg.LinAlgError) as e_gv:
        G.mlpg_gv_batch(m, v, w, np.ones(2), np.ones(2), lengths=[50, 30])
    assert str(e_gv.value) == str(e_ref.value)


def test_global_variance_and_gv_statistics():
    rng = np.random.default_rng(11)
    lens = [33, 1, 200, 7]
    for dtype in (np.float32, np.float64):
        x = (rng.standard_normal((sum(lens), 13)) * 3 + 1).astype(dtype)
        off = np.concatenate([[0], np.cumsum(lens)])
        ref = np.stack([x[off[u]:off[u + 1]].astype(np.float64).var(axis=0) for u in range(len(lens))])
        for got in (G.global_variance(x, offsets=off), G.global_variance(x, lengths=lens)):
            assert got.dtype == np.float64 and got.shape == ref.shape
            assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
        one = G.global_variance(x[:33])
        assert one.shape == (13,) and np.abs(one - ref[0]).max() <= 1e-12 * np.abs(ref).max()
        pad = np.zeros((len(lens), max(lens), 13), dtype)
        for u, T in enumerate(lens):
            pad[u, :T] = x[off[u]:off[u + 1]]
        pg = G.global_variance(torch.from_numpy(pad).cuda(), lengths=lens)
        assert pg.is_cuda and np.abs(pg.cpu().numpy() - ref).max() <= 1e-12 * np.abs(ref).max()
        gm, gvv = G.gv_statistics(x, lengths=lens)
        assert np.abs(gm - ref.mean(axis=0)).max() <= 1e-12 * np.abs(ref).max()
        assert np.abs(gvv - ref.var(axis=0)).max() <= 1e-12 * np.abs(ref.var(axis=0)).max()


def test_gmm_mlpg_with_gv_matches_oracle_on_its_e_and_d():
    from sklearn.mixture import GaussianMixture

    from nnmnkwii_b200.baseline.gmm import MLPG
    w = windows_set()[1]
    rng = np.random.default_rng(12)
    sd = 3
    src = np.cumsum(rng.standard_normal((600, 2 * sd)), axis=0) * 0.1
    tgt = src * 0.8 + rng.standard_normal((600, 2 * sd)) * 0.1
    gmm = GaussianMixture(n_components=4, covariance_type="full", random_state=0).fit(np.hstack([src, tgt]))
    gm, gvv = np.full(sd, 0.5), np.full(sd, 0.01)
    model = MLPG(gmm, windows=w, gv=(gm, gvv))
    plain = MLPG(gmm, windows=w)
    utts = [src[:80], src[80:200], src[200:203]]
    batch = model.transform_batch(utts)
    for u, s in enumerate(utts):
        x, c = model._to_device(s)
        E, Dv = model._means_vars(x, c)
        E, Dv = E.cpu().numpy(), Dv.cpu().numpy()
        y = model.transform(s)
        _check_utt(y, E, Dv, w, gm, gvv, False)
        assert np.array_equal(batch[u], y)
        assert np.abs(plain.transform(s) - ogv.mlpg(E, Dv, w)).max() <= 1e-10 * np.abs(y).max()
