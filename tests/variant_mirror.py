"""Host-side mirrors of the kernel-selection rules of the MLPG, UnitVarianceMLPG, DTW, GMM, metric, statistics,
affine, segment-copy and modulation-spectrum launchers, and a profiler helper that names the CUDA kernels a call
launched.

The mirrors restate, in Python, the size thresholds of the launchers (`pick_instance`, `as_geometry`
in csrc/nnk_mlpg*.cu*, `dtw_fused_smem` / `dtw_smem_bytes` / `dtw_fast_cells_bound` /
`dtw_exact_chunk` in csrc/nnk_dtw.cu, `em_layout` / `estep_d` / `mstep_d` in csrc/nnk_gmm_em.cu, the
launch sizes of csrc/nnk_gmm.cu, `traj_dispatch` in csrc/nnk_gmm_traj.cu, `dispatch_frame` in
csrc/nnk_metrics.cu, `stats_shape` and `launch_affine` in csrc/nnk_stats.cu, the vector test of
`nnk_segment_copy` in csrc/nnk_shard.cu and `dispatch_modspec` / `ms_threads` in csrc/nnk_modspec.cu).
The tests of tests/test_kernel_variants_*_gpu.py and tests/test_variants_*_gpu.py pick their shapes from them and then assert, with the
profiler, that the kernel the mirror predicts is the one that ran: a later change to a geometry function
makes those tests fail instead of silently moving their coverage.  tests/test_variant_mirror_constants_cpu.py
reads the constants restated here out of the CUDA sources, so a retuned constant fails there first."""
import re

import numpy as np

NNK_MAX_WIN = NNK_MAX_HALF = 4


# ---- which kernels ran ---------------------------------------------------------------------------------------
def profiled(fn, family=r"\b(mlpg|uv|dtw|fastdtw|trim_len)_\w*kernel\b", attempts=8):
    """Run ``fn()`` under torch.profiler (CUDA activity) and return ``(result, error, kernel_names)``.

    ``error`` is the exception ``fn`` raised (None if it returned).  CUPTI records the launches of the
    ctypes library as well as torch's own, but now and then a profile comes back without the records of
    a call; ``fn`` (every call here is repeatable) is then run again, at most ``attempts`` times, until the
    profile holds a kernel of ``family``.  Fails (never skips) when no such name was collected.

    The losses come in bursts: on an H100 one call lost its kernel record in 3 of 20 consecutive profiles,
    while 180 profiles of the same call in a fresh process lost none.  At that rate three attempts still
    miss about once in 300 calls, and the suite makes hundreds; eight miss about once in 4 million.
    Pass a ``family`` that names the kernel the caller asserts on, so that a profile that kept only the
    call's other kernels is repeated too.  A caller that asserts on several kernels of one call passes a list
    of patterns: the call is repeated until the profile holds a kernel of each, since a profile can also lose
    the record of one kernel of a call and keep another's."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    for _ in range(attempts):
        torch.cuda.synchronize()
        out = err = None
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            try:
                out = fn()
            except Exception as e:  # noqa: BLE001 -- handed back to the caller
                err = e
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
        if all(launched(names, p) for p in ([family] if isinstance(family, str) else family)):
            return out, err, names
    raise AssertionError("the profiler collected no kernel names of %r in %d attempts: %s" % (family, attempts, names))


def launched(names, pattern):
    """Names matching the regular expression ``pattern`` (a list of them: any of them)."""
    rx = [re.compile(p) for p in ([pattern] if isinstance(pattern, str) else pattern)]
    return [n for n in names if any(r.search(n) for r in rx)]


# ---- MLPG ------------------------------------------------------------------------------------------------------
def pick_instance(windows):
    """(NW, L, U) of the template instance `pick_instance` (csrc/nnk_mlpg.cu) chooses."""
    nw = len(windows)
    L = max(int(w[0]) for w in windows)
    U = max(int(w[1]) for w in windows)
    assert 1 <= nw <= NNK_MAX_WIN and L <= NNK_MAX_HALF and U <= NNK_MAX_HALF
    if nw == 1 and L == 0 and U == 0:
        return 1, 0, 0
    if nw <= 3 and L <= 1 and U <= 1:
        return 3, 1, 1
    if nw <= 3 and L <= 2 and U <= 2:
        return 3, 2, 2
    return NNK_MAX_WIN, NNK_MAX_HALF, NNK_MAX_HALF


def _r16(n):
    return (n + 32 + 15) // 16 * 16


def as_geometry_fits(row_bytes_m, row_bytes_v, grad, half_l, nt, G=1, NSA=1):
    """`as_geometry<TT=4, NA=3, NSA, ND=6, TTB=8, NSB=grad ? 4 : 8, G>` of csrc/nnk_mlpg_as.cuh.  The launcher
    asks for NSA = 1 at G = 1 and NSA = 2 at G = 2."""
    TT, NA, ND, TTB = 4, 3, 6, 8
    NSB = 4 if grad else 8
    ld = max(row_bytes_m, row_bytes_v)
    sb_in = _r16((TT + nt - 1) * ld)
    sb_ws = TTB * nt * 32 * 8
    sb_var = _r16((TTB + half_l) * row_bytes_v) if grad else 0
    ring_a = (NSA * 2 * sb_in + 127) // 128 * 128
    pbb = G * ND * TT * (nt + 1) * 32 * 8
    bwd = G * NSB * (sb_ws + sb_var)
    if NA * ring_a + pbb < bwd:
        ring_a = ((bwd - pbb) // NA + 127) // 128 * 128
    return 512 + NA * ring_a + pbb <= (100 if G == 1 else 113) * 1024


AS, DIRECT = "mlpg_fwd_as_kernel", "mlpg_kernel"


def mlpg_kernel_for(mode, windows, D, es, var_global=False, go_ld=None, go_f64=False):
    """Name of the kernel `launch_mlpg` runs for a single-stream call: mode "fwd" (in_ld = D) or "grad"
    (go_ld = columns of grad_output, static_dim for paramgen.mlpg_grad).

    The staged kernel runs when the window set fills its instance (nw == NW), NT <= 5, the call is a forward
    solve or has a float32 grad_output, and `as_geometry` fits; everything else runs `mlpg_kernel`."""
    NW, L, U = pick_instance(windows)
    nt = L + U + 1
    var_ld = 0 if var_global else D
    if mode == "fwd":
        row_bytes_m = D * es
    else:
        if go_f64:
            return DIRECT
        row_bytes_m = 4 * (D // len(windows) if go_ld is None else go_ld)
    staged = len(windows) == NW and nt <= 5 and as_geometry_fits(row_bytes_m, var_ld * es, mode == "grad", L, nt)
    return AS if staged else DIRECT


def staged_limit(mode, windows, es, var_global=False):
    """Widest row D (columns of the means) that still runs a staged kernel; D + 1 runs `mlpg_kernel`."""
    last = None
    for D in range(len(windows), 4097):
        if mlpg_kernel_for(mode, windows, D, es, var_global) != DIRECT:
            last = D
        elif last is not None:
            return last
    raise AssertionError("no staged-kernel limit below 4096 columns")


# ---- DTW -------------------------------------------------------------------------------------------------------
DTW_FR, DTW_CW = 512, 128
DTW_NBR = DTW_FR // 32 + 1
FD_PD, FD_MAXW = 7, 24


def max_smem_optin(device=0):
    import torch
    return int(torch.cuda.get_device_properties(device).shared_memory_per_block_optin)


def _dtw_dp(D):
    dp = (D + 1) & ~1
    if ((dp >> 1) & 1) == 0:
        dp += 2
    return dp


def dtw_fused_smem(max_tx, max_ty, D):
    groups = (max_tx + 31) // 32
    return 8 * (max_ty * _dtw_dp(D) + DTW_NBR * DTW_CW) + 4 * 2 * (groups + 1) + 16


# static shared memory of every dtw_fused_kernel instance (ptxas -v: 16 bytes, the back-track's `s_n`): a
# block may request the opt-in limit less this much dynamic shared memory
DTW_FUSED_STATIC_SMEM = 16


def dtw_fused_ok(max_tx, max_ty, D, max_smem):
    return 8 <= D < 40 and dtw_fused_smem(max_tx, max_ty, D) <= max_smem - DTW_FUSED_STATIC_SMEM


def dtw_fused_ty_limit(max_tx, D, max_smem):
    """Largest padded Ty the fused exact kernel takes at this D."""
    fixed = dtw_fused_smem(max_tx, 0, D)
    return (max_smem - DTW_FUSED_STATIC_SMEM - fixed) // (8 * _dtw_dp(D))


def dtw_dp_bucket(max_tx):
    """MC of the `dtw_dp_kernel<MC>` the two-pass exact path launches."""
    mc = (max_tx + 255) // 256
    return 4 if mc <= 4 else 8 if mc <= 8 else 16


def dtw_exact_chunk(n_pairs, max_tx, max_ty):
    per = max_tx * max_ty * 9
    return max(1, min(n_pairs, (2 << 30) // per))


def _dtw_smem_bytes(max_tx, bp_cap):
    return 8 * (FD_PD + 1) * 32 + 4 * (max_tx * 2 + (max_tx + 1) + 2 * (max_tx // 2 + 1)) + bp_cap + 16


def fast_cells_bound(max_tx, max_ty, radius):
    r2 = 2 * radius + 1
    return 4 * r2 * ((max_tx + max_ty) // 2 + r2 + 2) + 64


def fastdtw_caps(max_tx, max_ty, radius, max_smem):
    """(smem_bp_cap, cost_cap) of `nnk_dtw_align`'s FastDTW launch."""
    bound = fast_cells_bound(max_tx, max_ty, radius)
    if _dtw_smem_bytes(max_tx, bound) > max_smem // 4:
        base = _dtw_smem_bytes(max_tx, 0)
        assert base + 1024 <= max_smem
        bound = max_smem // 4 - base if max_smem // 4 > base + 1024 else 1024
    return bound, fast_cells_bound(max_tx, max_ty, radius)


def fastdtw_levels(x, y, radius, kind):
    """Per level of FastDTW, finest first: (window cells, most rows active on one anti-diagonal).

    Windows come from `oracle.expand_window` of the oracle's path one level coarser, exactly as
    `fastdtw_kernel` builds them; the sum of the cells is what the kernel reports as `cells`."""
    import oracle
    xs, ys = [np.asarray(x, np.float64)], [np.asarray(y, np.float64)]
    while len(xs[-1]) >= radius + 2 and len(ys[-1]) >= radius + 2:
        a, b = xs[-1], ys[-1]  # __reduce_by_half
        na, nb = len(a) // 2, len(b) // 2
        xs.append((a[0:2 * na:2] + a[1:2 * na:2]) / 2)
        ys.append((b[0:2 * nb:2] + b[1:2 * nb:2]) / 2)
    out = []
    for lev in range(len(xs)):
        Tx, Ty = len(xs[lev]), len(ys[lev])
        if lev == len(xs) - 1:
            lo, hi = np.zeros(Tx, np.int64), np.full(Tx, Ty, np.int64)
        else:
            _, pi, pj, _ = oracle.fastdtw(xs[lev + 1], ys[lev + 1], radius=radius, kind=kind)
            lo, hi = oracle.expand_window(pi, pj, Tx, Ty, radius)
            lo, hi = lo.astype(np.int64), hi.astype(np.int64)
        ncells = int(np.maximum(0, hi - lo).sum())
        # the kernel's count: row i enters on anti-diagonal k = i + lo[i]; the lowest row still active
        # there is the first r with r + hi[r] > k (binary search over [0, i])
        end = np.arange(Tx) + hi
        wmax = 0
        for i in range(Tx):
            k = i + lo[i]
            a, b = 0, i
            while a < b:
                m = (a + b) >> 1
                if end[m] > k:
                    b = m
                else:
                    a = m + 1
            wmax = max(wmax, i - a + 1)
        out.append((ncells, wmax))
    return out


# ---- GMM EM (csrc/nnk_gmm_em.cu) -------------------------------------------------------------------------------
EM_MAX_D = EM_MAX_K = 128
EM_ES_FT = 32          # E-step: frames per block (ES_FPW 8 x ES_WARPS 4)
EM_ST_CHUNK = 1024     # statistics: frames per block
EM_ST_SUB = EM_CV_SUB = 32
K_NUM_SMS = 132
EM_CV_TARGET_BLOCKS = 4 * K_NUM_SMS


def em_estep_epl(D):
    """EPL of the `em_estep_kernel<EPL, T>` that `estep_d` launches."""
    assert 1 <= D <= EM_MAX_D
    return min(4, (D + 31) // 32)


def em_cov_ti(D):
    """TI of the `em_cov_kernel<TI, T>` that `mstep_d` launches."""
    assert 1 <= D <= EM_MAX_D
    return min(8, (D + 15) // 16)


def _round4(v):
    return (v + 3) & ~3


def em_layout(N, D, K):
    """`em_layout`: tile / chunk counts and the workspace size `total` (in doubles)."""
    n_tiles = (N + EM_ES_FT - 1) // EM_ES_FT
    n_stat = (N + EM_ST_CHUNK - 1) // EM_ST_CHUNK
    n_cov = (EM_CV_TARGET_BLOCKS + K - 1) // K
    n_cov = max(1, min(n_cov, (N + 255) // 256))  # at least 256 frames per chunk
    cov_chunk = ((N + n_cov - 1) // n_cov + EM_CV_SUB - 1) // EM_CV_SUB * EM_CV_SUB
    n_cov = (N + cov_chunk - 1) // cov_chunk
    # lse, stat, nk, cov, logw, logdet, muu
    total = (_round4(n_tiles) + _round4(n_stat * K * (D + 1)) + _round4(K) + _round4(n_cov * K * D * D)
             + _round4(K) + _round4(K) + _round4(K * D))
    return dict(n_tiles=n_tiles, n_stat=n_stat, n_cov=n_cov, cov_chunk=cov_chunk, total=total)


def em_estep_smem(D, K):
    return 8 * (EM_ES_FT * D + EM_ES_FT * K + EM_ES_FT)


def em_stats_smem(D, K):
    return 8 * (K * (D + 1) + EM_ST_SUB * K + EM_ST_SUB * D)


def em_cov_smem(D):
    return 8 * (2 * EM_CV_SUB * 16 * em_cov_ti(D) + D)


def em_factor_smem(D):
    return 8 * (D * (D + 1) + D)


# ---- GMM mapping (csrc/nnk_gmm.cu) -----------------------------------------------------------------------------
GMM_FT = 16            # frames per block of gmm_logprob_kernel / gmm_posterior_kernel
GMM_SELECT_FT = 4      # frames (one per warp) per block of gmm_select_kernel
GMM_MAX_D = 96         # 32 lanes x GMM_EPL 3 outputs
GMM_MAX_M = 65535      # grid.y of gmm_logprob_kernel


def gmm_logprob_smem(D):
    return 8 * (D * D + GMM_FT * D)


def gmm_posterior_smem(D):
    return 8 * (D * D + GMM_FT * D + 2 * GMM_FT)


# ---- GMM trajectory EM (csrc/nnk_gmm_traj.cu) ------------------------------------------------------------------
TRAJ_MAX_EPL = 3       # D <= 96
NNK_GMM_TRAJ_TILE = 32  # frames per CTA, one utterance per tile


def traj_epl(D):
    """EPL of the `gmm_traj_em_kernel<EPL, EM>` that `traj_dispatch` launches (output dimensions per lane)."""
    assert 1 <= D <= 32 * TRAJ_MAX_EPL
    return (D + 31) // 32


# ---- kernel names in a child process -----------------------------------------------------------------------------
_CHILD_SCRIPT = r"""
import json, sys
sys.path[:0] = sys.argv[1:3]
import importlib
import variant_mirror as M
mod = importlib.import_module(sys.argv[3])
launch = getattr(mod, sys.argv[4])
repeats = sys.argv[6] == "1"
out = []
for case, family in json.loads(sys.argv[5]):
    _, err, names = M.profiled(lambda: launch(*case), family)
    names = M.launched(names, family)
    out.append([sorted(names if repeats else set(names)), repr(err)])
print(json.dumps(out))
"""


def profiled_in_child(module, launcher, cases, repeats=False):
    """``[(kernel names of family, repr(error))]`` of ``module.launcher(*case)`` for each ``(case, family)`` of
    ``cases``, each call profiled by `profiled` in a child Python process.  Profiling many calls in the pytest
    process has made torch.profiler lose the records of later modules' calls on an H100; a child process
    keeps the profiler state of those modules clean.  The names are distinct, or with ``repeats`` one per
    launch, so that a caller can count launches."""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    res = subprocess.run([sys.executable, "-c", _CHILD_SCRIPT, here, root, module, launcher, json.dumps(cases),
                          "1" if repeats else "0"],
                         capture_output=True, text=True, timeout=900, cwd=root)
    assert res.returncode == 0, res.stderr[-3000:]
    return json.loads(res.stdout.strip().splitlines()[-1])


def _itemsize(dtype):
    """Bytes of a NumPy / torch float dtype (or an int that already is one)."""
    if isinstance(dtype, int):
        return dtype
    size = getattr(dtype, "itemsize", None)  # torch.dtype
    return size if isinstance(size, int) else np.dtype(dtype).itemsize


# ---- metrics (csrc/nnk_metrics.cu) -------------------------------------------------------------------------------
MT_BLOCK = 256          # threads of frame_metric_kernel / f0_metric_kernel
MT_UNROLL = 4           # frames in flight per lane group
MT_TILE_ELEMS = 11776   # float32 elements of one frame_metric_tile_kernel tile
MT_TBLOCK = 128         # threads (and most frames) of a tile
MT_MIN_TILE_FRAMES = 46  # the smallest tile (float64, D = 127): sizes the partial workspace


def metric_kernel_for(D, frame_stride, dtype):
    """`dispatch_frame`: ``("tile", F)`` for `frame_metric_tile_kernel<T>` with F frames per tile, or
    ``("frame", G)`` for `frame_metric_kernel<T, G>` with G lanes per frame."""
    if D < 128 and frame_stride == D:
        return "tile", min(MT_TILE_ELEMS * 4 // _itemsize(dtype) // D, MT_TBLOCK)
    G = 1
    while G < 32 and G < D:
        G <<= 1
    return "frame", G


# ---- corpus statistics and the per-column affine map (csrc/nnk_stats.cu) ----------------------------------------
ST_BLOCK = 256             # threads per block at most (CW * RS)
ST_ROWS_PER_THREAD = 64    # rows a thread reads per tile
ST_THREADS_PER_SM = 816    # resident threads per SM the grid is sized for
AF_BLOCK = 256
AF_UNROLL = 4
AF_BLOCKS_PER_SM = 16      # the grid of column_affine_kernel is capped at K_NUM_SMS * 16 blocks


def stats_shape(n_utt, max_rows, D):
    """`stats_shape`: column strips, strip width CW, row slices RS, rows per tile, tiles and the grid."""
    nstrips = max(1, (D + ST_BLOCK - 1) // ST_BLOCK)
    w = (D + nstrips - 1) // nstrips
    CW = max(32, (w + 31) // 32 * 32)
    RS = ST_BLOCK // CW
    tile_rows = ST_ROWS_PER_THREAD * RS
    tiles_per_utt = (max_rows + tile_rows - 1) // tile_rows
    n_tiles = n_utt * tiles_per_utt
    bps = min(8, ST_THREADS_PER_SM // (CW * RS))
    grid = max(1, min(K_NUM_SMS * bps // nstrips, n_tiles))
    return dict(nstrips=nstrips, CW=CW, RS=RS, tile_rows=tile_rows, tiles_per_utt=tiles_per_utt, n_tiles=n_tiles,
                grid=grid)


def affine_passes(n, D):
    """``(passes, step_c, stride_c)`` of `column_affine_kernel` over n = rows * D elements: the grid-stride
    passes of the first thread (the most any thread makes), the column step between its unrolled elements and
    the column step between its passes."""
    per_block = AF_BLOCK * AF_UNROLL
    grid = min((n + per_block - 1) // per_block, K_NUM_SMS * AF_BLOCKS_PER_SM)
    stride = grid * per_block
    return (n + stride - 1) // stride, AF_BLOCK % D, stride % D


# ---- row-segment copy (csrc/nnk_shard.cu) ------------------------------------------------------------------------
SEG_ROWS_PER_BLOCK = 64


def segment_copy_vec(cols, es, src_ld, dst_ld, src_ptr, dst_ptr):
    """True when `nnk_segment_copy` runs `segment_copy_kernel<uint4>` (16-byte words), False for
    `segment_copy_kernel<uint32_t>`."""
    row, sp, dp = cols * es, src_ld * es, dst_ld * es
    return row % 16 == 0 and sp % 16 == 0 and dp % 16 == 0 and src_ptr % 16 == 0 and dst_ptr % 16 == 0


# ---- modulation spectrum (csrc/nnk_modspec.cu) -------------------------------------------------------------------
MS_MAX_THREADS = 256
MS_LOGN_MIN, MS_LOGN_MAX = 8, 12        # n = 256 .. 4096
MS_PF_MODES = (4, 5)                    # NNK_MS_LOGPOWER, NNK_MS_POSTFILTER: the PF instance


def ms_logn(n):
    """LOGN of the instance `dispatch_modspec` launches for DFT length n (the C ABI refuses every other n)."""
    logn = int(n).bit_length() - 1
    assert n == 1 << logn and MS_LOGN_MIN <= logn <= MS_LOGN_MAX, n
    return logn


def ms_threads(n):
    """Threads per CTA of `modspec_kernel` (`ms_threads<LOGN>`): n / 4, at most MS_MAX_THREADS."""
    return min(1 << (ms_logn(n) - 2), MS_MAX_THREADS)


def modspec_kernel_for(n, dtype, mode):
    """`modspec_kernel<T, LOGN, PF>` that `nnk_modspec` launches: LOGN = log2 n, PF exactly for the log-power
    and post-filter modes."""
    return "modspec_kernel<%s, %d, %s>" % ("float" if _itemsize(dtype) == 4 else "double", ms_logn(n),
                                           "true" if mode in MS_PF_MODES else "false")
