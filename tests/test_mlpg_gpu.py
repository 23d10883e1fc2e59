"""GPU parity tests for the MLPG family: CUDA path (through the C ABI) vs the oracle, vs the golden
vectors generated from the reference, and size-independent properties at BASELINE.json sizes.

Tolerance: BASELINE.json north_star states "within 1e-4 relative of the reference's CPU output on
float32"; the kernels compute in float64 like the reference, so the tests hold them to 1e-6
(float32 outputs: rounding of the result) and 1e-11 (float64 outputs)."""
import numpy as np
import pytest

import oracle
from conftest import rel_err, windows_set

pytestmark = pytest.mark.gpu

TOL32 = 1e-6
TOL64 = 1e-11


def _G():
    from nnmnkwii_b200 import paramgen as G
    return G


def test_mlpg_matches_reference_golden(golden):
    G = _G()
    for wi, ws in enumerate(windows_set()):
        for dt in ("float32", "float64"):
            tol = TOL32 if dt == "float32" else TOL64
            for T in (1, 2, 5, 12):
                key = "w%d_%s_T%d" % (wi, dt, T)
                m, v, go = golden[key + "_means"], golden[key + "_vars"], golden[key + "_go"]
                y = G.mlpg(m, v, ws)
                assert y.dtype == m.dtype and y.shape == golden[key + "_y"].shape
                assert rel_err(y, golden[key + "_y"]) < tol, key
                assert rel_err(G.mlpg(m, v[0].copy(), ws), golden[key + "_y1d"]) < tol, key
                g = G.mlpg_grad(m, v, ws, go)
                assert g.dtype == np.float32 and g.shape == m.shape
                assert rel_err(g, golden[key + "_grad"]) < 2e-6, key


def test_cfg1_matches_reference_golden(golden):
    """BASELINE.json configs[0]: T=100, static_dim=59, 3 windows, diag variance."""
    G = _G()
    r1 = np.random.default_rng(1234)
    m = r1.random((100, 177)).astype(np.float32)
    v = (r1.random((100, 177)) + 0.1).astype(np.float32)
    ws = windows_set()[2]
    assert rel_err(G.mlpg(m, v, ws), golden["cfg1_y"]) < TOL32
    assert rel_err(G.mlpg(m, np.ones(177, dtype=np.float32), ws), golden["cfg1_y_unitvar"]) < TOL32


def test_mlpg_vs_oracle_grid():
    G = _G()
    rng = np.random.default_rng(11)
    for ws in windows_set():
        nw = len(ws)
        for dt, tol in ((np.float32, TOL32), (np.float64, TOL64)):
            for T, sd in ((1, 1), (2, 3), (3, 33), (4, 2), (7, 64), (100, 59), (257, 5)):
                m = rng.random((T, sd * nw)).astype(dt)
                v = (rng.random((T, sd * nw)) + 0.05).astype(dt)
                assert rel_err(G.mlpg(m, v, ws), oracle.mlpg(m, v, ws)) < tol, (nw, dt, T, sd)
                v1 = (rng.random(sd * nw) + 0.05).astype(dt)
                y1 = G.mlpg(m, v1, ws)
                assert rel_err(y1, oracle.mlpg(m, v1, ws)) < tol
                # 1-D variance == tiled 2-D variance (tests/test_paramgen.py:44-59)
                assert np.allclose(y1, G.mlpg(m, np.tile(v1, (T, 1)), ws))


def test_mlpg_quirks_match_reference():
    G = _G()
    ws = windows_set()[2]
    rng = np.random.default_rng(2)
    # D not a multiple of num_windows -> static_dim = D // nw (paramgen/_mlpg.py:172)
    m = rng.random((9, 7)); v = rng.random((9, 7)) + 0.1
    y = G.mlpg(m, v, ws)
    assert y.shape == (9, 2) and rel_err(y, oracle.mlpg(m, v, ws)) < TOL64
    # mixed dtypes: output dtype follows the means
    y = G.mlpg(m.astype(np.float32), v, ws)
    assert y.dtype == np.float32
    # zero-width dynamic windows: precisions[-0:] = 0 zeroes every dynamic frame (_mlpg.py:192-193)
    wz = [(0, 0, np.array([1.0])), (0, 0, np.array([2.0]))]
    m2 = rng.random((5, 4)); v2 = rng.random((5, 4)) + 0.1
    assert rel_err(G.mlpg(m2, v2, wz), oracle.mlpg(m2, v2, wz)) < TOL64
    # asymmetric windows go through the generic kernel instance
    wa = [(0, 0, np.array([1.0])), (1, 0, np.array([-1.0, 1.0])), (0, 2, np.array([1.0, -2.0, 1.0]))]
    m3 = rng.random((20, 6)); v3 = rng.random((20, 6)) + 0.1
    assert rel_err(G.mlpg(m3, v3, wa), oracle.mlpg(m3, v3, wa)) < TOL64
    # shape mismatch -> AssertionError (_mlpg.py:171)
    with pytest.raises(AssertionError):
        G.mlpg(m, v[:5], ws)


def test_not_positive_definite_raises_like_reference():
    G = _G()
    ws = windows_set()[2]
    rng = np.random.default_rng(3)
    m = rng.random((30, 6)); v = rng.random((30, 6)) + 0.1
    v[:, 1] = -1.0  # negative static variance of dim 1 -> some pivot of chain 1 is not positive
    with pytest.raises(np.linalg.LinAlgError) as e_ref:
        oracle.mlpg(m, v, ws)
    ref_msg = str(e_ref.value)  # "<k>-th leading minor not positive definite" (linalg.pyx:79-82)
    assert "leading minor not positive definite" in ref_msg
    with pytest.raises(np.linalg.LinAlgError) as e_gpu:
        G.mlpg(m, v, ws)
    assert str(e_gpu.value).startswith(ref_msg), (str(e_gpu.value), ref_msg)  # same 1-based frame
    # a failure in a later utterance / chain of a batch reports the first one in reference loop order
    lens = [10, 12, 9]
    mb = rng.random((31, 6)); vb = rng.random((31, 6)) + 0.1
    vb[10:22, 0] = -1.0
    vb[22:, 1] = -1.0
    with pytest.raises(np.linalg.LinAlgError, match=r"utterance 1, chain 0"):
        G.mlpg_batch(mb, vb, ws, lengths=lens)


def test_mlpg_grad_vs_oracle():
    G = _G()
    rng = np.random.default_rng(5)
    for ws in windows_set():
        nw = len(ws)
        for dt in (np.float32, np.float64):
            for T, sd in ((1, 2), (3, 3), (50, 33), (300, 4)):
                m = rng.random((T, sd * nw)).astype(dt)
                v = (rng.random((T, sd * nw)) + 0.05).astype(dt)
                go = rng.standard_normal((T, sd)).astype(np.float32)
                g = G.mlpg_grad(m, v, ws, go)
                assert g.dtype == np.float32 and g.shape == (T, sd * nw)
                assert rel_err(g, oracle.mlpg_grad(m, v, ws, go)) < 2e-6
    # more lengths around the tile sizes, global (D,) variances, float64 grad_output (direct-load kernel)
    ws = windows_set()[2]
    for T in (2, 4, 5, 8, 9, 16, 17, 31, 64, 65):
        sd = 40
        m = rng.random((T, sd * 3)).astype(np.float32)
        v = (rng.random((T, sd * 3)) + 0.05).astype(np.float32)
        v1 = (rng.random(sd * 3) + 0.05).astype(np.float32)
        go = rng.standard_normal((T, sd)).astype(np.float32)
        assert rel_err(G.mlpg_grad(m, v, ws, go), oracle.mlpg_grad(m, v, ws, go)) < 2e-6, T
        assert rel_err(G.mlpg_grad(m, v1, ws, go), oracle.mlpg_grad(m, v1, ws, go)) < 2e-6, T
        g64 = G.mlpg_grad(m, v, ws, go.astype(np.float64))
        assert rel_err(g64, oracle.mlpg_grad(m, v, ws, go)) < 2e-6, T


def test_mlpg_grad_batched_device_call():
    """nnk_mlpg_grad on a ragged batch in one launch (what a batched autograd.MLPG would issue):
    every utterance equals the single-utterance oracle result; rows of other utterances untouched."""
    import torch
    from nnmnkwii_b200 import _device as dev
    from nnmnkwii_b200 import _lib
    ws = windows_set()[2]
    rng = np.random.default_rng(8)
    sd = 59
    lens = np.array([7, 300, 1, 64, 129, 33])
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    n = int(off[-1])
    v = (rng.random((n, 3 * sd)) + 0.05).astype(np.float32)
    go = rng.standard_normal((n, sd)).astype(np.float32)
    dv, dgo = torch.from_numpy(v).cuda(), torch.from_numpy(go).cuda()
    out = torch.zeros(n, 3 * sd, device="cuda")
    dev.run_mlpg("grad", means=None, variances=dv, rhs=dgo, out=out, offsets=torch.from_numpy(off).cuda(), lengths=None,
                 order=None, chains=dev.chains_on_device(dev.simple_chains(sd), dv.device), n_chain=sd,
                 max_T=int(lens.max()), windows_c=_lib.make_windows(ws), in_ld=3 * sd, var_ld=3 * sd, go_ld=sd,
                 out_ld=3 * sd, dtype_code=_lib.NNK_F32, go_f64=0, n_utt=len(lens), device=dv.device, check=True)
    got = out.cpu().numpy()
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        want = oracle.mlpg_grad(np.zeros((b - a, 3 * sd), np.float32), v[a:b], ws, go[a:b])
        assert rel_err(got[a:b], want) < 2e-6, u


def test_unit_variance_mlpg_matrix(golden):
    G = _G()
    for wi, ws in enumerate(windows_set()):
        for T in (3, 10):
            R = G.unit_variance_mlpg_matrix(ws, T)
            assert R.dtype == np.float32 and R.shape == (T, len(ws) * T)
            assert np.abs(R - golden["w%d_R_T%d" % (wi, T)]).max() < 2e-7
        # R @ reshape_means(mu) == mlpg(mu, ones)  (tests/test_paramgen.py:82-95)
        T, sd = 25, 4
        mu = np.random.default_rng(wi).random((T, sd * len(ws)))
        R = G.unit_variance_mlpg_matrix(ws, T)
        y = G.mlpg(mu, np.ones(sd * len(ws)), ws)
        assert np.allclose(R @ G.reshape_means(mu, sd), y, rtol=1e-5, atol=1e-6)
    assert np.abs(G.unit_variance_mlpg_matrix(windows_set()[2], 40) - golden["w2_R_T40"]).max() < 2e-7
    R200 = G.unit_variance_mlpg_matrix(windows_set()[2], 200)
    assert np.abs(R200 - oracle.unit_variance_mlpg_matrix(windows_set()[2], 200)).max() < 2e-7


def _merlin_batch(n_utt, lo, hi, seed, global_var=False):
    rng = np.random.default_rng(seed)
    lens = rng.integers(lo, hi + 1, size=n_utt)
    n = int(lens.sum())
    m = rng.random((n, 187), dtype=np.float32)
    v = (rng.random(187, dtype=np.float32) + 0.1) if global_var else (rng.random((n, 187), dtype=np.float32) + 0.1)
    return lens, m, v


def _oracle_merlin(m, v, ws, lens):
    """The gallery-notebook pattern: per utterance, per stream mlpg; vuv copied."""
    out = np.zeros((m.shape[0], 63), dtype=m.dtype)
    off = np.concatenate([[0], np.cumsum(lens)])
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        vv = (lambda c0, c1: v[c0:c1]) if v.ndim == 1 else (lambda c0, c1: v[a:b, c0:c1])
        out[a:b, 0:60] = oracle.mlpg(m[a:b, 0:180], vv(0, 180), ws)
        out[a:b, 60:61] = oracle.mlpg(m[a:b, 180:183], vv(180, 183), ws)
        out[a:b, 61] = m[a:b, 183]
        out[a:b, 62:63] = oracle.mlpg(m[a:b, 184:187], vv(184, 187), ws)
    return out


def test_batched_merlin_layout_vs_oracle():
    G = _G()
    ws = windows_set()[2]
    for global_var in (False, True):
        lens, m, v = _merlin_batch(12, 1, 90, 21, global_var)
        y = G.mlpg_batch(m, v, ws, lengths=lens, layout=G.merlin_layout())
        assert y.shape == (m.shape[0], 63) and y.dtype == np.float32
        assert rel_err(y, _oracle_merlin(m, v, ws, lens)) < TOL32
    # zero-padded (B, Tmax, D) form and the device-tensor form agree with the flat host form
    import torch
    lens, m, v = _merlin_batch(5, 3, 40, 22)
    y = G.mlpg_batch(m, v, ws, lengths=lens, layout=G.merlin_layout())
    yd = G.mlpg_batch(torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda(), ws, lengths=lens, layout=G.merlin_layout())
    assert yd.is_cuda and np.array_equal(yd.cpu().numpy(), y)
    Tmax = int(lens.max())
    mp = np.zeros((5, Tmax, 187), np.float32); vp = np.ones((5, Tmax, 187), np.float32)
    off = np.concatenate([[0], np.cumsum(lens)])
    for u in range(5):
        mp[u, :lens[u]] = m[off[u]:off[u + 1]]; vp[u, :lens[u]] = v[off[u]:off[u + 1]]
    yp = G.mlpg_batch(mp, vp, ws, lengths=lens, layout=G.merlin_layout())
    ypd = G.mlpg_batch(torch.from_numpy(mp).cuda(), torch.from_numpy(vp).cuda(), ws, lengths=lens, layout=G.merlin_layout()).cpu().numpy()
    for u in range(5):
        assert np.array_equal(yp[u, :lens[u]], y[off[u]:off[u + 1]])
        assert np.array_equal(ypd[u, :lens[u]], y[off[u]:off[u + 1]])
        assert not yp[u, lens[u]:].any() and not ypd[u, lens[u]:].any()


def test_cfg2_full_size_properties():
    """BASELINE.json configs[1]: 256 utterances, T~600, D=187.  Oracle on a sample of utterances +
    size-independent properties on everything: P y == b (residual), linearity in the means,
    utterance independence (batch == solo)."""
    G = _G()
    ws = windows_set()[2]
    lens, m, v = _merlin_batch(256, 540, 660, 1234)
    lay = G.merlin_layout()
    y = G.mlpg_batch(m, v, ws, lengths=lens, layout=lay)
    off = np.concatenate([[0], np.cumsum(lens)])
    for u in (0, 17, 255):
        a, b = off[u], off[u + 1]
        assert rel_err(y[a:b], _oracle_merlin(m[a:b], v[a:b], ws, lens[u:u + 1])) < TOL32
        solo = G.mlpg_batch(m[a:b], v[a:b], ws, lengths=[b - a], layout=lay)
        assert np.array_equal(solo, y[a:b])
    # linearity: mlpg(a*m1 + m2) == a*mlpg(m1) + mlpg(m2) for fixed variances
    m2 = np.random.default_rng(9).random(m.shape, dtype=np.float32)
    y2 = G.mlpg_batch(m2, v, ws, lengths=lens, layout=lay)
    y3 = G.mlpg_batch((0.5 * m + m2).astype(np.float32), v, ws, lengths=lens, layout=lay)
    assert rel_err(y3[:, :61], (0.5 * y.astype(np.float64) + y2)[:, :61]) < 5e-6
    # residual of the normal equations for the lf0 stream of every utterance, in float64 on the host
    tau = 1.0 / v[:, 180:183].astype(np.float64)
    mu = m[:, 180:183].astype(np.float64)
    worst = 0.0
    for u in range(0, 256, 8):
        a, b = off[u], off[u + 1]
        T = b - a
        t = tau[a:b].copy(); t[:1, 1:] = 0; t[-1:, 1:] = 0
        yy = y[a:b, 60].astype(np.float64)
        W = [np.eye(T), 0.5 * (np.eye(T, k=1) - np.eye(T, k=-1)), np.eye(T, k=1) - 2 * np.eye(T) + np.eye(T, k=-1)]
        P = sum(Wk.T @ (t[:, k:k + 1] * Wk) for k, Wk in enumerate(W))
        rhs = sum(Wk.T @ (t[:, k] * mu[a:b, k]) for k, Wk in enumerate(W))
        worst = max(worst, np.abs(P @ yy - rhs).max() / np.abs(rhs).max())
    assert worst < 1e-5  # float32 rounding of y, amplified by ||P||


def test_batch_edge_cases():
    """Empty batch, zero-length utterances inside a batch, utterances shorter than the window
    support (T = 1, 2), all handled without touching neighbours' rows."""
    G = _G()
    ws = windows_set()[2]
    lay = G.merlin_layout()
    # empty batch
    y = G.mlpg_batch(np.zeros((0, 187), np.float32), np.ones((0, 187), np.float32), ws, lengths=[], layout=lay)
    assert y.shape == (0, 63)
    # zero-length and very short utterances between normal ones
    lens = np.array([5, 0, 1, 2, 0, 33, 3, 0])
    rng = np.random.default_rng(77)
    n = int(lens.sum())
    m = rng.random((n, 187), dtype=np.float32)
    v = rng.random((n, 187), dtype=np.float32) + 0.1
    y = G.mlpg_batch(m, v, ws, lengths=lens, layout=lay)
    assert rel_err(y, _oracle_merlin(m, v, ws, lens)) < TOL32
    # one utterance only, T = 1: the dynamic windows are edge-masked, y = means (static part)
    y1 = G.mlpg_batch(m[:1], v[:1], ws, lengths=[1], layout=lay)
    assert np.array_equal(y1[0, :60], m[0, :60])


def test_ill_conditioned_variances():
    """Static variances 1e6 times the delta variances (smooth trajectories, cond(P) ~ 1e7): the
    float64 LDL^T stays within the north_star tolerance by a wide margin."""
    G = _G()
    ws = windows_set()[2]
    rng = np.random.default_rng(5)
    T, sd = 700, 40
    m = rng.standard_normal((T, 3 * sd)).astype(np.float32)
    v = np.empty((T, 3 * sd), np.float32)
    v[:, :sd] = 10.0 ** rng.uniform(0, 3, (T, sd))
    v[:, sd:2 * sd] = 10.0 ** rng.uniform(-4, -3, (T, sd))
    v[:, 2 * sd:] = 10.0 ** rng.uniform(-5, -3, (T, sd))
    y = G.mlpg(m, v, ws)
    ref = oracle.mlpg(m, v, ws)
    assert rel_err(y, ref) < 1e-5
    y64 = G.mlpg(m.astype(np.float64), v.astype(np.float64), ws)
    assert rel_err(y64, oracle.mlpg(m.astype(np.float64), v.astype(np.float64), ws)) < 1e-8


def test_ragged_batch_cfg5_shape():
    """BASELINE.json configs[4] shape at a reduced count: mixed T in [200, 2000], LPT order, waves."""
    G = _G()
    ws = windows_set()[2]
    lay = G.merlin_layout()
    lens, m, v = _merlin_batch(96, 200, 2000, 4242)
    y = G.mlpg_batch(m, v, ws, lengths=lens, layout=lay)
    off = np.concatenate([[0], np.cumsum(lens)])
    for u in (0, 1, int(np.argmax(lens)), int(np.argmin(lens)), 95):
        a, b = off[u], off[u + 1]
        assert rel_err(y[a:b], _oracle_merlin(m[a:b], v[a:b], ws, lens[u:u + 1])) < TOL32
    assert np.array_equal(y[:, 61], m[:, 183])


def test_mlpg_grad_batch_merlin_layout():
    """Batched gradient through the 187-column layout (three smoothed streams + the copied vuv column)."""
    import torch
    G = _G()
    ws = windows_set()[2]
    lay = G.merlin_layout()
    for global_var in (False, True):
        lens, m, v = _merlin_batch(7, 1, 150, 31, global_var)
        n = m.shape[0]
        go = np.random.default_rng(4).standard_normal((n, 63)).astype(np.float32)
        got = G.mlpg_grad_batch(torch.from_numpy(v).cuda(), ws, torch.from_numpy(go).cuda(), lens, layout=lay).cpu().numpy()
        assert got.shape == (n, 187) and got.dtype == np.float32
        off = np.concatenate([[0], np.cumsum(lens)])
        want = np.zeros((n, 187), np.float32)
        for u in range(len(lens)):
            a, b = off[u], off[u + 1]
            z = np.zeros((b - a, 180), np.float32)
            vv = (lambda c0, c1: v[c0:c1]) if v.ndim == 1 else (lambda c0, c1: v[a:b, c0:c1])
            want[a:b, 0:180] = oracle.mlpg_grad(z, vv(0, 180), ws, go[a:b, 0:60])
            want[a:b, 180:183] = oracle.mlpg_grad(z[:, :3], vv(180, 183), ws, go[a:b, 60:61])
            want[a:b, 183] = go[a:b, 61]
            want[a:b, 184:187] = oracle.mlpg_grad(z[:, :3], vv(184, 187), ws, go[a:b, 62:63])
        assert rel_err(got, want) < 2e-6, global_var


def test_ring_protocol_stress_many_launches_reused_scratch():
    """VERDICT r1 item 5: the assembler/solver ring protocol under launch pressure -- hundreds of
    back-to-back launches, odd lengths (tiles that end mid-ring, T smaller than one tile), narrow and
    wide chain groups, scratch handed back and forth by the caching allocator, two streams at once.
    Every launch must be bit-identical to the first run of the same inputs and match the oracle."""
    import torch
    G = _G()
    ws = windows_set()[2]
    rng = np.random.default_rng(77)
    cases = []
    for T, sd in ((1, 1), (3, 59), (5, 60), (13, 3), (31, 33), (97, 59), (100, 59), (255, 60), (300, 7), (641, 62)):
        m = rng.random((T, 3 * sd), dtype=np.float32)
        v = rng.random((T, 3 * sd), dtype=np.float32) + 0.1
        mt, vt = torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda()
        first = G.mlpg(mt, vt, ws).clone()
        assert rel_err(first.cpu().numpy(), oracle.mlpg(m, v, ws)) < TOL32
        cases.append((mt, vt, first))
    side = torch.cuda.Stream()
    outs = []
    for it in range(40):
        for k, (mt, vt, first) in enumerate(cases):
            if (it + k) % 3 == 0:
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    outs.append((k, G.mlpg_batch(mt, vt, ws, lengths=[mt.shape[0]], check=False)))
            else:
                outs.append((k, G.mlpg_batch(mt, vt, ws, lengths=[mt.shape[0]], check="deferred")))
        if it % 10 == 9:
            torch.cuda.synchronize()
            for k, y in outs:
                assert torch.equal(y, cases[k][2]), "launch %d differs" % k
            outs = []
    from nnmnkwii_b200 import _device as dev
    dev.poll_errors(block=True)


def test_deferred_check_surfaces_not_positive_definite():
    """check='deferred' never blocks, and the LinAlgError still arrives (at poll_errors / the next call)."""
    import torch
    from nnmnkwii_b200 import _device as dev
    G = _G()
    ws = windows_set()[0]  # static window only: the pivot of frame t is 1 / variance[t]
    m = torch.rand(20, 3, device="cuda")
    v = torch.rand(20, 3, device="cuda") + 0.1
    v[7, 1] = -1.0  # a negative variance makes the 8-th pivot of chain 1 non-positive
    dev.poll_errors(block=True)
    G.mlpg_batch(m, v, ws, lengths=[20], check="deferred")
    with pytest.raises(np.linalg.LinAlgError):
        dev.poll_errors(block=True)
    dev.poll_errors(block=True)  # the record is consumed


def test_batch_tables_are_checked_before_any_launch_on_every_path():
    """Padded lengths of the wrong size or above Tmax, and flat lengths that do not cover the rows, raise
    AssertionError for CUDA inputs of mlpg_batch / mlpg_grad_batch exactly as for NumPy mlpg_batch."""
    import torch

    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200 import paramgen as G
    ws = windows_set()[2]
    rng = np.random.default_rng(11)
    m = rng.standard_normal((3, 20, 3 * 4)).astype(np.float32)
    v = np.ones_like(m)
    go = torch.ones((3, 20, 4), device="cuda")
    bad_padded = ([20, 20], [20, 20, 20, 20], [5, 21, 5])
    bad_flat = ([20, 20, 19], [20, 20, 20, 1])
    n0 = _lib.launch_count()
    for lens in bad_padded:
        for call in (lambda: G.mlpg_batch(m, v, ws, lengths=lens),
                     lambda: G.mlpg_batch(torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda(), ws, lengths=lens),
                     lambda: G.mlpg_grad_batch(torch.from_numpy(v).cuda(), ws, go, lens)):
            with pytest.raises(AssertionError):
                call()
    for lens in bad_flat:
        for call in (lambda: G.mlpg_batch(m.reshape(60, -1), v.reshape(60, -1), ws, lengths=lens),
                     lambda: G.mlpg_batch(torch.from_numpy(m).cuda().reshape(60, -1),
                                          torch.from_numpy(v).cuda().reshape(60, -1), ws, lengths=lens),
                     lambda: G.mlpg_grad_batch(torch.from_numpy(v).cuda().reshape(60, -1), ws, go.reshape(60, -1),
                                               lens)):
            with pytest.raises(AssertionError):
                call()
    assert _lib.launch_count() == n0
