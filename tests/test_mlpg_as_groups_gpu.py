"""The two-group instance of `mlpg_fwd_as_kernel` (G = 2: one CTA serves chain groups 2j and 2j+1 of an
utterance and stages each input row once for both).  The launcher takes it for float32 forward solves with
two or more chain groups and band depth S <= 2; float64 rows, single groups and the gradient keep G = 1.

Each case asserts, through the profiler, which instance ran (the last template argument is G), and checks
the result against the float64 oracle at the suite's float32 bar, or bit for bit against the G = 1 instance."""
import ctypes
import re

import numpy as np
import pytest

import oracle
import variant_mirror as M
from conftest import rel_err, windows_set

pytestmark = pytest.mark.gpu

TOL32 = 1e-6  # as tests/test_mlpg_gpu.py
STD = windows_set()[2]
# three windows of half-width 1 that are not the standard static / delta / delta-delta set
ODD3 = [(0, 0, np.array([1.0])), (1, 1, np.array([-1.0, 0.0, 1.0])), (0, 1, np.array([-1.0, 1.0]))]
SKEW3 = [(0, 0, np.array([1.0])), (1, 0, np.array([-1.0, 1.0])), (1, 1, np.array([0.25, -0.5, 0.25]))]
AS_FAMILY = r"\bmlpg_(fwd_as_)?kernel<"


def _G():
    from nnmnkwii_b200 import paramgen as G
    return G


def _groups_per_cta(names):
    """G of every MLPG kernel that ran; non-staged kernels count as None."""
    out = []
    for n in M.launched(names, AS_FAMILY):
        m = re.search(r"mlpg_fwd_as_kernel<([^<>]*)>", n)
        out.append(int(m.group(1).split(",")[-1]) if m else None)
    return out


def _run(fn, want_g):
    out, err, names = M.profiled(fn, family=AS_FAMILY)
    assert err is None, err
    got = _groups_per_cta(names)
    assert got and all(g == want_g for g in got), (want_g, got)
    return out


def _want_g(n_chain, D):
    """G of a float32 standard-window forward solve with per-frame variances, D columns in both arrays."""
    return 2 if n_chain > 32 and M.as_geometry_fits(4 * D, 4 * D, False, 1, 3, G=2, NSA=2) else 1


def _single(rng, T, sd, dt=np.float32, var_global=False, nw=3):
    m = rng.random((T, nw * sd)).astype(dt)
    v = ((rng.random(nw * sd) if var_global else rng.random((T, nw * sd))) + 0.05).astype(dt)
    return m, v


def _oracle_merlin(m, v, ws, lens):
    out = np.zeros((m.shape[0], 63), dtype=m.dtype)
    off = np.concatenate([[0], np.cumsum(lens)])
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        out[a:b, 0:60] = oracle.mlpg(m[a:b, 0:180], v[a:b, 0:180], ws)
        out[a:b, 60:61] = oracle.mlpg(m[a:b, 180:183], v[a:b, 180:183], ws)
        out[a:b, 61] = m[a:b, 183]
        out[a:b, 62:63] = oracle.mlpg(m[a:b, 184:187], v[a:b, 184:187], ws)
    return out


# ---- which instance runs ----------------------------------------------------------------------------------------
def test_instance_selection():
    G = _G()
    rng = np.random.default_rng(1)
    lay = G.merlin_layout()
    lens = np.array([40, 7, 90])
    n = int(lens.sum())
    m = rng.random((n, 187), dtype=np.float32)
    v = rng.random((n, 187), dtype=np.float32) + 0.1
    y = _run(lambda: G.mlpg_batch(m, v, STD, lengths=lens, layout=lay), 2)
    assert rel_err(y, _oracle_merlin(m, v, STD, lens)) < TOL32
    y64 = _run(lambda: G.mlpg_batch(m.astype(np.float64), v.astype(np.float64), STD, lengths=lens, layout=lay), 1)
    assert rel_err(y64.astype(np.float32), y) < TOL32
    # the T = 1000, static_dim 60 forward of the benchmark's extras
    m1, v1 = _single(rng, 1000, 60)
    y1 = _run(lambda: G.mlpg(m1, v1, STD), 2)
    assert rel_err(y1, oracle.mlpg(m1, v1, STD)) < TOL32
    # one chain group: nothing to pair
    m2, v2 = _single(rng, 300, 32)
    y2 = _run(lambda: G.mlpg(m2, v2, STD), 1)
    assert rel_err(y2, oracle.mlpg(m2, v2, STD)) < TOL32


# ---- the grouping does not change the arithmetic ----------------------------------------------------------------
def test_two_groups_per_cta_bit_identical_to_one():
    """63 chains in one call (G = 2) against chains 0-31 and 32-62 in two calls (G = 1 each)."""
    G = _G()
    rng = np.random.default_rng(2)
    lens = np.array([1, 2, 5, 64, 131, 257])
    sd = 63
    m, v = _single(rng, int(lens.sum()), sd)
    lay = G.StreamLayout.single(3 * sd, 3)
    y = _run(lambda: G.mlpg_batch(m, v, STD, lengths=lens, layout=lay), 2)
    parts = []
    for c0, c1 in ((0, 32), (32, 63)):
        cols = np.concatenate([np.arange(c0, c1) + w * sd for w in range(3)])
        ms, vs = np.ascontiguousarray(m[:, cols]), np.ascontiguousarray(v[:, cols])
        k = c1 - c0
        parts.append(_run(lambda: G.mlpg_batch(ms, vs, STD, lengths=lens, layout=G.StreamLayout.single(3 * k, 3)), 1))
    assert np.array_equal(y, np.concatenate(parts, axis=1))


# ---- oracle parity ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [1, 2, 3, 4, 5, 8, 9, 17, 257])
def test_lengths(T):
    G = _G()
    m, v = _single(np.random.default_rng(T), T, 63)
    y = _run(lambda: G.mlpg(m, v, STD), 2)
    assert rel_err(y, oracle.mlpg(m, v, STD)) < TOL32


@pytest.mark.parametrize("global_var", [False, True])
def test_ragged_merlin_batch(global_var):
    G = _G()
    rng = np.random.default_rng(3)
    lens = rng.integers(1, 120, size=13)
    lens[[2, 7]] = [0, 1]
    n = int(lens.sum())
    m = rng.random((n, 187), dtype=np.float32)
    v = (rng.random(187, dtype=np.float32) if global_var else rng.random((n, 187), dtype=np.float32)) + 0.1
    y = _run(lambda: G.mlpg_batch(m, v, STD, lengths=lens, layout=G.merlin_layout()), 2)
    vf = np.broadcast_to(v, m.shape) if global_var else v
    assert rel_err(y, _oracle_merlin(m, np.ascontiguousarray(vf), STD, lens)) < TOL32


@pytest.mark.parametrize("n_chain", [33, 63, 64, 65, 96])
@pytest.mark.parametrize("global_var", [False, True])
def test_chain_counts(n_chain, global_var):
    """Odd group counts (65 chains: 3 groups) run the last pair with an empty second half.  96 chains take
    288 columns, too wide for two G = 2 CTAs per SM: they run G = 1."""
    G = _G()
    m, v = _single(np.random.default_rng(n_chain), 97, n_chain, var_global=global_var)
    assert _want_g(n_chain, 3 * n_chain) == (1 if n_chain == 96 else 2)
    y = _run(lambda: G.mlpg(m, v, STD), _want_g(n_chain, 3 * n_chain))
    assert rel_err(y, oracle.mlpg(m, v, STD)) < TOL32


@pytest.mark.parametrize("ws", [ODD3, SKEW3], ids=["odd3", "skew3"])
@pytest.mark.parametrize("T", [2, 9, 130])
def test_non_standard_window_sets(ws, T):
    G = _G()
    m, v = _single(np.random.default_rng(T), T, 65)
    y = _run(lambda: G.mlpg(m, v, ws), 2)
    assert rel_err(y, oracle.mlpg(m, v, ws)) < TOL32


# ---- waves and failures -------------------------------------------------------------------------------------------
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
    y1 = _run(lambda: G.mlpg_batch(m, v, STD, lengths=lens, layout=lay), 2)
    need = _lib.lib.nnk_mlpg_workspace_bytes(len(lens), lay.n_chain, int(max(lens)), ctypes.byref(_lib.make_windows(STD)))
    monkeypatch.setattr(dev, "WORKSPACE_CAP_BYTES", 3 * (need // len(lens)))
    c0 = _lib.launch_count()
    y2 = _run(lambda: G.mlpg_batch(m, v, STD, lengths=lens, layout=lay), 2)
    assert _lib.launch_count() - c0 >= 4
    assert torch.equal(y1, y2)


@pytest.mark.parametrize("bad", [[(40, 0)], [(5, 10), (40, 0)], [(40, 0), (50, 0)], [(64, 3)]],
                         ids=["second-half", "first-half-later-frame", "two-in-second-half", "odd-group"])
def test_not_positive_definite_in_reference_order(bad):
    """`bad` = (chain, first failing frame) pairs; the report is the reference's first failure: lowest chain."""
    G = _G()
    sd = 65 if any(c >= 63 for c, _ in bad) else 63
    m, v = _single(np.random.default_rng(9), 30, sd)
    for c, f in bad:
        v[f:, c] = -1.0
    with pytest.raises(np.linalg.LinAlgError) as e_ref:
        oracle.mlpg(m, v, STD)
    _, err, names = M.profiled(lambda: G.mlpg(m, v, STD), family=AS_FAMILY)
    assert isinstance(err, np.linalg.LinAlgError), err
    assert _groups_per_cta(names) and all(g == 2 for g in _groups_per_cta(names))
    first = min(c for c, _ in bad)
    assert str(err).startswith(str(e_ref.value)) and "chain %d)" % first in str(err), (str(err), str(e_ref.value))


def test_two_stream_stress_bit_identical():
    """Back-to-back launches on two streams over odd lengths and odd group counts, scratch recycled by the
    allocator: every launch bit-identical to the first run of the same inputs."""
    import torch
    from nnmnkwii_b200 import _device as dev
    G = _G()
    rng = np.random.default_rng(77)
    cases = []
    for T, sd in ((1, 33), (3, 63), (5, 64), (13, 65), (31, 96), (97, 63), (100, 33), (255, 65), (641, 63)):
        m, v = _single(rng, T, sd)
        mt, vt = torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda()
        first = _run(lambda: G.mlpg(mt, vt, STD), _want_g(sd, 3 * sd)).clone()
        assert rel_err(first.cpu().numpy(), oracle.mlpg(m, v, STD)) < TOL32
        cases.append((mt, vt, first))
    side = torch.cuda.Stream()
    outs = []
    for it in range(40):
        for k, (mt, vt, first) in enumerate(cases):
            if (it + k) % 3 == 0:
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    outs.append((k, G.mlpg_batch(mt, vt, STD, lengths=[mt.shape[0]], check=False)))
            else:
                outs.append((k, G.mlpg_batch(mt, vt, STD, lengths=[mt.shape[0]], check="deferred")))
        if it % 10 == 9:
            torch.cuda.synchronize()
            for k, y in outs:
                assert torch.equal(y, cases[k][2]), "launch %d differs" % k
            outs = []
    dev.poll_errors(block=True)
