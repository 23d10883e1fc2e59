"""The host side of tests/test_kernel_variants_gv_gpu.py, checked without a GPU: its table of which
`mlpg_kernel` instance serves each window set, the GV workspace size, and the workspace caps that split its
batches into waves of exactly k utterances."""
import ctypes
import os
import re

import pytest

import variant_mirror as M
from conftest import ROOT
from test_kernel_variants_gv_gpu import INSTANCE, SETS, WAVE_KS, WAVE_SETS, _wave_batch, gv_cap, kernel_name


def _lib():
    from nnmnkwii_b200 import _lib
    return _lib


def _dispatch_source():
    with open(os.path.join(ROOT, "nnmnkwii_b200", "csrc", "nnk_mlpg.cu")) as f:
        src = f.read()
    i = src.index("static int dispatch_inst(")
    return src, src[i:src.index("\n}\n", i)]


@pytest.mark.parametrize("name", list(SETS))
def test_instance_table_follows_the_launcher(name):
    inst, NW, L, U = INSTANCE[name]
    assert M.pick_instance(SETS[name]) == (NW, L, U)
    src, dispatch = _dispatch_source()
    if inst < 3:
        assert "case %d: return launch_mlpg<Tin, %d, %d, %d, MODE>" % (inst, NW, L, U) in dispatch
    else:
        assert (M.NNK_MAX_WIN, M.NNK_MAX_HALF, M.NNK_MAX_HALF) == (NW, L, U)
        assert "default: return launch_mlpg<Tin, NNK_MAX_WIN, NNK_MAX_HALF, NNK_MAX_HALF, MODE>" in dispatch
    assert "constexpr int PF = (L + U <= 2) ? 4 : 2;" in src
    assert "mlpg_kernel<Tin, NW, L, U, MODE, PF><<<" in src
    assert re.search(r"MODE_SOLVE = 2, MODE_GV = 3", open(os.path.join(ROOT, "nnmnkwii_b200", "csrc", "nnk_mlpg.cuh")).read())
    PF = 4 if L + U <= 2 else 2
    assert kernel_name(name, "float32", 3) == "mlpg_kernel<float, %d, %d, %d, 3, %d>" % (NW, L, U, PF)
    assert kernel_name(name, "float64", 2) == "mlpg_kernel<double, %d, %d, %d, 2, %d>" % (NW, L, U, PF)


def test_every_instance_is_in_the_table():
    assert sorted({v[0] for v in INSTANCE.values()}) == [0, 1, 2, 3]


@pytest.mark.parametrize("name", ["w0", "w2", "w3", "nw4"])
def test_gv_workspace_bytes(name):
    """n_utt * ceil(n_chain / 32) * max_T * (S + 1 + 4) * 32 * 8: four more float64 columns per frame than the
    forward solve's (pivot, c_m, current and trial trajectory)."""
    lib = _lib()
    _, _, L, U = INSTANCE[name]
    S = L + U
    win = ctypes.byref(lib.make_windows(SETS[name]))
    for n_utt, n_chain, max_T in ((1, 1, 1), (3, 32, 17), (11, 33, 257), (7, 63, 1000), (65537, 5, 3)):
        groups = -(-n_chain // 32)
        want = n_utt * groups * max_T * (S + 1 + 4) * 32 * 8
        assert lib.lib.nnk_mlpg_gv_workspace_bytes(n_utt, n_chain, max_T, win) == want
        assert lib.lib.nnk_mlpg_workspace_bytes(n_utt, n_chain, max_T, win) == want // (S + 5) * (S + 1)


@pytest.mark.parametrize("name", WAVE_SETS)
def test_wave_cap_puts_k_utterances_in_each_wave(name):
    """`_device.run_mlpg` sizes the scratch as max(per_utt, min(need, max(cap, per_utt))) and `launch_mlpg` runs
    (bytes // per_item) // n_groups utterances per launch, per_item = max_T * (S + 5) * 32 * 8 in GV mode."""
    import numpy as np
    lib = _lib()
    _, _, L, U = INSTANCE[name]
    m, v, lens, gm, gvv = _wave_batch(name, np.float64)
    n_chain = m.shape[1] // len(SETS[name])
    groups = -(-n_chain // 32)
    need = lib.lib.nnk_mlpg_gv_workspace_bytes(len(lens), n_chain, int(max(lens)), ctypes.byref(lib.make_windows(SETS[name])))
    per_utt = need // len(lens)
    per_item = int(max(lens)) * (L + U + 5) * 32 * 8
    for k in WAVE_KS[1:]:
        cap = gv_cap(lens, n_chain, SETS[name], k)
        nbytes = max(per_utt, min(need, max(cap, per_utt)))
        assert (nbytes // per_item) // groups == k
        waves = [lens[i:i + k] for i in range(0, len(lens), k)]
        assert len(waves) == -(-len(lens) // k) and all(len(w) == k for w in waves[:-1])
