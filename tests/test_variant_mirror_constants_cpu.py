"""The constants that tests/variant_mirror.py restates, read out of the CUDA sources (no GPU needed).

The metric, statistics, affine, segment-copy, trajectory-EM and modulation-spectrum variant tests pick their
shapes from the mirror; if one of these constants is retuned in a .cu file without the mirror, this test fails
instead of the GPU tests quietly covering other instances than they say."""
import os
import re

import pytest

import variant_mirror as M

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nnmnkwii_b200", "csrc")


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _constexpr(src, name):
    m = re.findall(r"constexpr\s+(?:int|int64_t)\s+%s\s*=\s*(\d+)\s*;" % name, src)
    assert len(m) == 1, (name, m)
    return int(m[0])


def _function(src, signature):
    """Body of the function whose definition starts with `signature` (up to the next top-level brace)."""
    i = src.index(signature)
    j = src.index("{", i)
    depth = 0
    for k in range(j, len(src)):
        depth += {"{": 1, "}": -1}.get(src[k], 0)
        if depth == 0:
            return src[j:k + 1]
    raise AssertionError("unterminated body of " + signature)


def test_number_of_sms():
    assert _constexpr(_source("nnk_common.cuh"), "kNumSMs") == M.K_NUM_SMS


@pytest.mark.parametrize("name", ["MT_TILE_ELEMS", "MT_TBLOCK", "MT_MIN_TILE_FRAMES", "MT_BLOCK", "MT_UNROLL"])
def test_metric_constants(name):
    assert _constexpr(_source("nnk_metrics.cu"), name) == getattr(M, name)


def test_metric_dispatch_rule():
    src = _function(_source("nnk_metrics.cu"), "static void dispatch_frame(")
    assert "p.D < 128 && p.frame_stride == p.D" in src
    assert "MT_TILE_ELEMS * 4 / (int)sizeof(T) / p.D" in src
    assert "while (G < 32 && G < p.D) G <<= 1;" in src
    # the smallest tile (float64, widest tiled row) is the one the partial workspace is sized for
    assert min(M.metric_kernel_for(D, D, 8)[1] for D in range(1, 128)) == M.MT_MIN_TILE_FRAMES


@pytest.mark.parametrize("name", ["ST_BLOCK", "ST_ROWS_PER_THREAD", "ST_THREADS_PER_SM", "AF_BLOCK", "AF_UNROLL"])
def test_stats_constants(name):
    assert _constexpr(_source("nnk_stats.cu"), name) == getattr(M, name)


def test_stats_and_affine_geometry():
    src = _source("nnk_stats.cu")
    shape = _function(src, "static StatsShape stats_shape(")
    assert "if (bps > 8) bps = 8;" in shape
    assert "s.tile_rows = ST_ROWS_PER_THREAD * s.RS;" in shape
    affine = _function(src, "static void launch_affine(")
    assert re.findall(r"kNumSMs \* (\d+)", affine) == [str(M.AF_BLOCKS_PER_SM)] * 2


def test_segment_copy_constants():
    src = _function(_source("nnk_shard.cu"), 'extern "C" int nnk_segment_copy(')
    assert re.findall(r"p\.rows_per_block = (\d+);", src) == [str(M.SEG_ROWS_PER_BLOCK)]
    assert M.segment_copy_vec(4, 4, 4, 4, 0, 0) and not M.segment_copy_vec(4, 4, 4, 4, 4, 0)


def test_gmm_traj_constants_and_dispatch_rule():
    src = _source("nnk_gmm_traj.cu")
    assert _constexpr(src, "TRAJ_MAX_EPL") == M.TRAJ_MAX_EPL
    with open(os.path.join(os.path.dirname(os.path.dirname(CSRC)), "include", "nnk_b200.h")) as f:
        assert re.findall(r"#define NNK_GMM_TRAJ_TILE (\d+)", f.read()) == [str(M.NNK_GMM_TRAJ_TILE)]
    body = _function(src, "static int traj_dispatch(")
    assert "const int epl = (p.g.D + 31) / 32;" in body
    assert re.findall(r"if \(epl == (\d)\) return traj_launch<(\d), EM>", body) == [("1", "1"), ("2", "2")]
    assert "return traj_launch<3, EM>(p, st);" in body
    assert [M.traj_epl(D) for D in (1, 32, 33, 64, 65, 96)] == [1, 1, 2, 2, 3, 3]


def _declared(src, name):
    """Value of `name = <int>` in a constexpr declaration that may declare several names."""
    m = re.findall(r"constexpr\s+int\s+(?:\w+\s*=\s*\d+\s*,\s*)*%s\s*=\s*(\d+)\s*[,;]" % name, src)
    assert len(m) == 1, (name, m)
    return int(m[0])


def test_modspec_constants_and_dispatch_rule():
    from nnmnkwii_b200.preprocessing.modspec import NS
    src = _source("nnk_modspec.cu")
    assert _constexpr(src, "MS_MAX_THREADS") == M.MS_MAX_THREADS
    assert (_declared(src, "MS_LOGN_MIN"), _declared(src, "MS_LOGN_MAX")) == (M.MS_LOGN_MIN, M.MS_LOGN_MAX)
    assert "(1 << (LOGN - 2)) < MS_MAX_THREADS ? (1 << (LOGN - 2)) : MS_MAX_THREADS" in src
    # every LOGN but the largest has a case of its own; the largest is the default
    body = _function(src, "static int dispatch_modspec(")
    cases = re.findall(r"case (\d+): return launch_modspec<T, (\d+), PF>\(a, st\);", body)
    assert [(int(c), int(l)) for c, l in cases] == [(l, l) for l in range(M.MS_LOGN_MIN, M.MS_LOGN_MAX)]
    assert re.findall(r"default: return launch_modspec<T, (\d+), PF>\(a, st\);", body) == [str(M.MS_LOGN_MAX)]
    assert len(re.findall(r"\breturn\b", body)) == len(cases) + 1
    # the C ABI refuses every other n, and the PF instance takes the modes from NNK_MS_LOGPOWER on
    entry = _function(src, 'extern "C" int nnk_modspec(')
    assert "(1 << logn) == n && logn >= MS_LOGN_MIN && logn <= MS_LOGN_MAX" in entry
    pf = r"if \(mode >= NNK_MS_(\w+)\)\s*return dtype == NNK_F32 \? dispatch_modspec<float, true>"
    assert re.findall(pf, entry) == ["LOGPOWER"]
    assert "mode >= NNK_MS_POWER && mode <= NNK_MS_POSTFILTER" in entry
    with open(os.path.join(os.path.dirname(os.path.dirname(CSRC)), "include", "nnk_b200.h")) as f:
        modes = {k: int(v) for k, v in re.findall(r"#define NNK_MS_(\w+) (\d+)", f.read())}
    assert tuple(v for v in sorted(modes.values()) if v >= modes["LOGPOWER"]) == M.MS_PF_MODES
    assert modes["POSTFILTER"] == max(modes.values())
    # the Python layer offers exactly the lengths of the instances
    assert tuple(NS) == tuple(2 ** l for l in range(M.MS_LOGN_MIN, M.MS_LOGN_MAX + 1))
    assert [M.ms_threads(n) for n in NS] == [64, 128, 256, 256, 256]
