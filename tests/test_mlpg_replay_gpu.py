"""The forward solve of `mlpg_fwd_as_kernel` keeps no factors in memory: the forward sweep stores one
checkpoint of the elimination state per segment (32 frames for float32 inputs with S <= 2, else 16), and the
backward sweep replays each segment's elimination from it before back-substituting the segment.

Lengths at and around segment and tile boundaries, a ragged batch mixing them, float32 and float64, one and
two chain groups per CTA, and both band depths the staged kernel takes, against the float64 oracle; and a
non-positive pivot planted in the first, a middle and the last segment, reported as the reference reports it."""
import numpy as np
import pytest

import oracle
import variant_mirror as M
from conftest import rel_err, windows_set

pytestmark = pytest.mark.gpu

TOL = {np.float32: 1e-6, np.float64: 1e-11}  # as tests/test_mlpg_gpu.py
STD = windows_set()[2]
WIDE = windows_set()[3]  # half-width 2: S = 4
AS_FAMILY = r"\bmlpg_(fwd_as_)?kernel<"
# around 16 and 32 (segments), 4 (tiles) and their small multiples
LENGTHS = (1, 2, 3, 4, 5, 15, 16, 17, 31, 32, 33, 47, 48, 49, 63, 64, 65, 95, 96, 97, 127, 129)


def _G():
    from nnmnkwii_b200 import paramgen as G
    return G


def _staged_groups(names):
    out = []
    for n in M.launched(names, AS_FAMILY):
        assert "mlpg_fwd_as_kernel<" in n, n
        out.append(int(n.split("mlpg_fwd_as_kernel<")[1].split(">")[0].split(",")[-1]))
    return out


def _data(rng, T, D, dt):
    return rng.random((T, D)).astype(dt), (rng.random((T, D)) + 0.05).astype(dt)


@pytest.mark.parametrize("ws", [STD, WIDE], ids=["S2", "S4"])
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("sd", [5, 40], ids=["one_group", "two_groups"])
def test_lengths_around_segment_boundaries(ws, dt, sd):
    G = _G()
    rng = np.random.default_rng(sd * 7 + len(ws))
    D = sd * len(ws)
    want_g = 2 if (sd > 32 and dt == np.float32 and ws is STD) else 1
    m, v = _data(rng, LENGTHS[-1], D, dt)
    _, err, names = M.profiled(lambda: G.mlpg(m, v, ws), family=AS_FAMILY)  # which instance serves the case
    assert err is None, err
    assert _staged_groups(names) == [want_g], names
    for T in LENGTHS:
        m, v = _data(rng, T, D, dt)
        assert rel_err(G.mlpg(m, v, ws), oracle.mlpg(m, v, ws)) < TOL[dt], (T, dt, sd)


@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
def test_ragged_batch(dt):
    import torch
    G = _G()
    rng = np.random.default_rng(5)
    lens = np.array(LENGTHS + (200, 31, 1, 64, 33))
    rng.shuffle(lens)
    sd = 40
    D = 3 * sd
    n = int(lens.sum())
    m, v = _data(rng, n, D, dt)
    y = G.mlpg_batch(torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda(), STD, lengths=lens).cpu().numpy()
    off = np.concatenate([[0], np.cumsum(lens)])
    for u in range(len(lens)):
        a, b = off[u], off[u + 1]
        assert rel_err(y[a:b], oracle.mlpg(m[a:b], v[a:b], STD)) < TOL[dt], (u, lens[u])


@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("dt,sd", [(np.float64, 6), (np.float32, 6), (np.float32, 40)],
                         ids=["f64", "f32", "f32-two-groups"])
def test_not_positive_definite_in_every_segment(where, dt, sd):
    G = _G()
    rng = np.random.default_rng(11)
    T = 150
    frame = {"first": 3, "middle": 77, "last": 146}[where]
    m, v = _data(rng, T, 3 * sd, np.float64)
    v[frame, 1] = -1e-3  # chain 1: a negative static precision that outweighs its neighbours
    with pytest.raises(np.linalg.LinAlgError) as e_ref:
        oracle.mlpg(m, v, STD)
    ref_msg = str(e_ref.value)
    assert "leading minor not positive definite" in ref_msg
    with pytest.raises(np.linalg.LinAlgError) as e_gpu:
        G.mlpg(m.astype(dt), v.astype(dt), STD)
    err = e_gpu.value
    assert str(err).startswith(ref_msg) and "chain 1)" in str(err), (str(err), ref_msg)
