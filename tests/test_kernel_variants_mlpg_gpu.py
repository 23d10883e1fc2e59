"""Every kernel `launch_mlpg` can select through shapes alone, against the float64 oracle.

The suite's other MLPG tests run the kernels the benchmark workloads use.  Here each case names the kernel
it expects (`variant_mirror.mlpg_kernel_for`, a restatement of the launcher's thresholds) and the profiler
confirms that it ran:
  * template instance 3 (NW = 4, L = U = 4): NT = 9 is beyond the staged kernel, so four windows take
    `mlpg_kernel`; three windows with a half-width-3 window, and two windows of half-width 2 in instance 2,
    take `mlpg_kernel` because nw < NW;
  * both sides of the row-width limit of the staged kernel, forward and gradient;
  * a 513-bin spectral envelope with standard windows (D = 1539), which only `mlpg_kernel` takes;
  * a batch split into several launches ("waves") when its factor scratch exceeds the workspace cap;
  * the not-positive-definite report of every kernel."""
import numpy as np
import pytest

import oracle
import variant_mirror as M
from conftest import rel_err, windows_set

pytestmark = pytest.mark.gpu

TOL32 = 1e-6  # as tests/test_mlpg_gpu.py
TOL64 = 1e-11
TOL_GRAD = 2e-6

STD = windows_set()[2]
NINE_TAP = (4, 4, np.array([1.0, -2.0, 3.0, -4.0, 0.0, 4.0, -3.0, 2.0, -1.0]) / 20.0)
SEVEN_TAP = (3, 3, np.array([-3.0, -2.0, -1.0, 0.0, 1.0, 2.0, 3.0]) / 28.0)
WIN_NW4 = STD + [NINE_TAP]                                            # instance 3, nw == NW
WIN_NW3_HW3 = [STD[0], STD[1], SEVEN_TAP]                             # instance 3, nw < NW
WIN_NW2_HW2 = [STD[0], (2, 2, np.array([1.0, -8.0, 0.0, 8.0, -1.0]) / 12.0)]  # instance 2, nw < NW


def _G():
    from nnmnkwii_b200 import paramgen as G
    return G


def _tol(dt):
    return TOL32 if dt == np.float32 else TOL64


def _data(rng, T, D, dt, var_global=False):
    m = rng.random((T, D)).astype(dt)
    v = ((rng.random(D) if var_global else rng.random((T, D))) + 0.05).astype(dt)
    return m, v


def _assert_ran(names, kernel):
    """`kernel` ran, and no other MLPG kernel did."""
    mlpg = M.launched(names, r"\bmlpg_(fwd_as_)?kernel<")
    assert mlpg and all(kernel + "<" in n for n in mlpg), (kernel, mlpg)


def _fwd(ws, m, v, kernel):
    G = _G()
    y, err, names = M.profiled(lambda: G.mlpg(m, v, ws))
    assert err is None, err
    _assert_ran(names, kernel)
    assert rel_err(y, oracle.mlpg(m, v, ws)) < _tol(m.dtype.type), (kernel, m.shape, m.dtype)


def _grad(ws, m, v, kernel, rng):
    G = _G()
    go = rng.standard_normal((m.shape[0], m.shape[1] // len(ws))).astype(np.float32)
    g, err, names = M.profiled(lambda: G.mlpg_grad(m, v, ws, go))
    assert err is None, err
    _assert_ran(names, kernel)
    assert g.dtype == np.float32 and g.shape == m.shape
    assert rel_err(g, oracle.mlpg_grad(m, v, ws, go)) < TOL_GRAD, (kernel, m.shape, m.dtype)


@pytest.mark.parametrize("name,ws,fwd_kernel,grad_kernel", [
    ("nw4", WIN_NW4, M.DIRECT, M.DIRECT),
    ("nw3_halfwidth3", WIN_NW3_HW3, M.DIRECT, M.DIRECT),
    ("nw2_halfwidth2", WIN_NW2_HW2, M.DIRECT, M.DIRECT),
])
def test_window_sets_of_the_wider_instances(name, ws, fwd_kernel, grad_kernel):
    rng = np.random.default_rng(31)
    sd = 5
    D = sd * len(ws)
    for dt in (np.float32, np.float64):
        es = np.dtype(dt).itemsize
        for var_global in (False, True):
            assert M.mlpg_kernel_for("fwd", ws, D, es, var_global) == fwd_kernel
            assert M.mlpg_kernel_for("grad", ws, D, es, var_global) == grad_kernel
            for T in (1, 2, 3, 4, 5, 8, 9, 17, 257):
                m, v = _data(rng, T, D, dt, var_global)
                _fwd(ws, m, v, fwd_kernel)
                _grad(ws, m, v, grad_kernel, rng)


@pytest.mark.parametrize("wi", [0, 2, 3], ids=["NT1", "NT3", "NT5"])
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("mode", ["fwd", "grad"])
def test_row_width_limit_of_the_staged_kernels(wi, dt, mode):
    """D = limit - 1 and D = limit (both parities; D not a multiple of nw where that is how the limit
    falls) run the warp-specialised kernel, D = limit + 1 falls back to `mlpg_kernel`."""
    ws = windows_set()[wi]
    es = np.dtype(dt).itemsize
    lim = M.staged_limit(mode, ws, es)
    rng = np.random.default_rng(lim)
    for D, kernel in ((lim - 1, M.AS), (lim, M.AS), (lim + 1, M.DIRECT)):
        assert M.mlpg_kernel_for(mode, ws, D, es) == kernel, (D, lim)
        m, v = _data(rng, 37, D, dt)
        if mode == "fwd":
            _fwd(ws, m, v, kernel)
        else:
            _grad(ws, m, v, kernel, rng)


def test_wide_spectral_envelope():
    """513-bin WORLD spectral envelope with static / delta / delta-delta windows: D = 1539 is wider than
    the staged kernel's rings, so forward and gradient run `mlpg_kernel`."""
    rng = np.random.default_rng(513)
    sd, T = 513, 600
    D = 3 * sd
    assert M.mlpg_kernel_for("fwd", STD, D, 4) == M.DIRECT and M.mlpg_kernel_for("grad", STD, D, 4) == M.DIRECT
    m, v = _data(rng, T, D, np.float32)
    _fwd(STD, m, v, M.DIRECT)
    _grad(STD, m, v, M.DIRECT, rng)


# ---- waves --------------------------------------------------------------------------------------------------
def _cap_for(lens, layout, ws, n_waves_utt):
    """A workspace cap worth `n_waves_utt` utterances of this batch's factor scratch."""
    import ctypes
    from nnmnkwii_b200 import _lib
    need = _lib.lib.nnk_mlpg_workspace_bytes(len(lens), layout.n_chain, int(max(lens)), ctypes.byref(_lib.make_windows(ws)))
    assert need % len(lens) == 0
    return n_waves_utt * (need // len(lens))


def test_wave_split_is_bit_identical(monkeypatch):
    import torch
    from nnmnkwii_b200 import _device as dev
    from nnmnkwii_b200 import _lib
    G = _G()
    lay = G.merlin_layout()
    rng = np.random.default_rng(71)
    lens = rng.integers(1, 160, size=11)
    n = int(lens.sum())
    m = torch.from_numpy(rng.random((n, 187), dtype=np.float32)).cuda()
    v = torch.from_numpy(rng.random((n, 187), dtype=np.float32) + 0.1).cuda()
    go = torch.from_numpy(rng.standard_normal((n, 63)).astype(np.float32)).cuda()

    def run():
        c0 = _lib.launch_count()
        y = G.mlpg_batch(m, v, STD, lengths=lens, layout=lay)
        c1 = _lib.launch_count()
        g = G.mlpg_grad_batch(v, STD, go, lens, layout=lay)
        c2 = _lib.launch_count()
        return y, g, c1 - c0, c2 - c1

    y1, g1, nf1, ng1 = run()
    assert (nf1, ng1) == (1, 1)
    per_wave = 3
    monkeypatch.setattr(dev, "WORKSPACE_CAP_BYTES", _cap_for(lens, lay, STD, per_wave))
    waves = -(-len(lens) // per_wave)
    (y2, g2, nf2, ng2), _, names = M.profiled(run)
    assert (nf2, ng2) == (waves, waves)
    assert len(M.launched(names, r"mlpg_fwd_as_kernel<")) == 2 * waves
    assert torch.equal(y1, y2) and torch.equal(g1, g2)
    # and the split batch still matches the oracle, utterance by utterance
    off = np.concatenate([[0], np.cumsum(lens)])
    mh, vh, yh = m.cpu().numpy(), v.cpu().numpy(), y2.cpu().numpy()
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        want = np.zeros((b - a, 63), np.float32)
        want[:, 0:60] = oracle.mlpg(mh[a:b, 0:180], vh[a:b, 0:180], STD)
        want[:, 60:61] = oracle.mlpg(mh[a:b, 180:183], vh[a:b, 180:183], STD)
        want[:, 61] = mh[a:b, 183]
        want[:, 62:63] = oracle.mlpg(mh[a:b, 184:187], vh[a:b, 184:187], STD)
        assert rel_err(yh[a:b], want) < TOL32, u


def test_wave_split_reports_the_first_failure_in_reference_order(monkeypatch):
    """Longest-first waves of two: utterance 6 (35 frames) runs in the second wave, utterance 3 (20 frames)
    in the third.  Both fail; the report is utterance 3's, the first in (utterance, chain, frame) order."""
    import torch
    from nnmnkwii_b200 import _device as dev
    G = _G()
    rng = np.random.default_rng(72)
    lens = np.array([50, 40, 30, 20, 10, 45, 35])
    sd = 4
    n = int(lens.sum())
    off = np.concatenate([[0], np.cumsum(lens)])
    m = rng.random((n, 3 * sd))
    v = rng.random((n, 3 * sd)) + 0.1
    v[off[3]:off[4], 2] = -1.0  # utterance 3, chain 2
    v[off[6]:off[7], 0] = -1.0  # utterance 6, chain 0
    with pytest.raises(np.linalg.LinAlgError) as e_ref:
        oracle.mlpg(m[off[3]:off[4]], v[off[3]:off[4]], STD)
    monkeypatch.setattr(dev, "WORKSPACE_CAP_BYTES", _cap_for(lens, G.StreamLayout.single(3 * sd, 3), STD, 2))
    for dt in (torch.float32, torch.float64):
        mt, vt = torch.from_numpy(m).to("cuda", dt), torch.from_numpy(v).to("cuda", dt)
        with pytest.raises(np.linalg.LinAlgError) as e_gpu:
            G.mlpg_batch(mt, vt, STD, lengths=lens)
        msg = str(e_gpu.value)
        assert msg.startswith(str(e_ref.value)) and "(utterance 3, chain 2)" in msg, (msg, str(e_ref.value))


# ---- not positive definite ----------------------------------------------------------------------------------
@pytest.mark.parametrize("mode,ws,sd,kernel", [
    ("fwd", STD, 6, M.AS),
    ("fwd", WIN_NW4, 5, M.DIRECT),
    ("fwd", WIN_NW3_HW3, 5, M.DIRECT),
    ("fwd", STD, 200, M.DIRECT),
    ("grad", STD, 6, M.AS),
    ("grad", WIN_NW4, 5, M.DIRECT),
], ids=["fwd-as", "fwd-direct-instance3", "fwd-direct-narrow-set", "fwd-direct-wide-rows", "grad-as", "grad-direct"])
def test_not_positive_definite_through_every_kernel(mode, ws, sd, kernel):
    G = _G()
    rng = np.random.default_rng(sd)
    T, D = 30, sd * len(ws)
    assert M.mlpg_kernel_for(mode, ws, D, 8) == kernel
    m = rng.random((T, D))
    v = rng.random((T, D)) + 0.1
    v[:, 1] = -1.0  # negative static variance of chain 1
    go = rng.standard_normal((T, sd)).astype(np.float32)
    ref_fn = (lambda: oracle.mlpg(m, v, ws)) if mode == "fwd" else (lambda: oracle.mlpg_grad(m, v, ws, go))
    gpu_fn = (lambda: G.mlpg(m, v, ws)) if mode == "fwd" else (lambda: G.mlpg_grad(m, v, ws, go))
    with pytest.raises(np.linalg.LinAlgError) as e_ref:
        ref_fn()
    ref_msg = str(e_ref.value)
    assert "leading minor not positive definite" in ref_msg
    _, err, names = M.profiled(gpu_fn)
    assert isinstance(err, np.linalg.LinAlgError), err
    _assert_ran(names, kernel)
    assert str(err).startswith(ref_msg) and "chain 1)" in str(err), (str(err), ref_msg)
