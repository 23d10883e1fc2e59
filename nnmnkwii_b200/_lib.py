"""ctypes binding of libnnk_b200.so (C ABI: include/nnk_b200.h).

The CUDA library IS the implementation: if it is missing or the ABI does not match, importing
this module raises.  There is deliberately no CPU / PyTorch fallback (tests/ verify that).
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NNK_LIB_PATH") or os.path.join(_HERE, "libnnk_b200.so")  # NNK_LIB_PATH: A/B builds

NNK_OK, NNK_ERR_ARG, NNK_ERR_UNSUPPORTED, NNK_ERR_CUDA, NNK_ERR_WORKSPACE, NNK_ERR_NOT_PD = 0, -1, -2, -3, -4, -5
NNK_F32, NNK_F64 = 0, 1
NNK_I32, NNK_I64 = 2, 3
NNK_MAX_WIN, NNK_MAX_HALF = 4, 4
NNK_MAX_TAPS = 2 * NNK_MAX_HALF + 1
ABI_VERSION = 2


class NnkWindows(ctypes.Structure):
    _fields_ = [
        ("nw", ctypes.c_int32),
        ("l", ctypes.c_int32 * NNK_MAX_WIN),
        ("u", ctypes.c_int32 * NNK_MAX_WIN),
        ("coef", (ctypes.c_double * NNK_MAX_TAPS) * NNK_MAX_WIN),
    ]


class NnkStatus(ctypes.Structure):
    _fields_ = [("code", ctypes.c_int32), ("utt", ctypes.c_int32), ("chain", ctypes.c_int32), ("frame", ctypes.c_int32)]


class NnkMlpgArgs(ctypes.Structure):
    _fields_ = [
        ("means", ctypes.c_void_p),
        ("vars", ctypes.c_void_p),
        ("grad_out", ctypes.c_void_p),
        ("out", ctypes.c_void_p),
        ("dtype", ctypes.c_int32),
        ("n_utt", ctypes.c_int32),
        ("in_ld", ctypes.c_int64),
        ("var_ld", ctypes.c_int64),
        ("go_ld", ctypes.c_int64),
        ("out_ld", ctypes.c_int64),
        ("utt_off", ctypes.c_void_p),
        ("utt_len", ctypes.c_void_p),
        ("order", ctypes.c_void_p),
        ("chains", ctypes.c_void_p),
        ("n_chain", ctypes.c_int32),
        ("max_T", ctypes.c_int32),
        ("go_f64", ctypes.c_int32),
        ("win", NnkWindows),
        ("workspace", ctypes.c_void_p),
        ("workspace_bytes", ctypes.c_size_t),
        ("status_word", ctypes.c_void_p),
        ("out_off", ctypes.c_void_p),
    ]


class NnkGmm(ctypes.Structure):
    _fields_ = [
        ("src_means", ctypes.c_void_p), ("tgt_means", ctypes.c_void_p), ("prec_chol", ctypes.c_void_p),
        ("log_const", ctypes.c_void_p), ("A_t", ctypes.c_void_p), ("Dm", ctypes.c_void_p),
        ("M", ctypes.c_int32), ("D", ctypes.c_int32),
    ]


class NnkGmmEmArgs(ctypes.Structure):
    _fields_ = [
        ("X", ctypes.c_void_p),
        ("N", ctypes.c_int64),
        ("x_ld", ctypes.c_int64),
        ("dtype", ctypes.c_int32),
        ("D", ctypes.c_int32),
        ("K", ctypes.c_int32),
        ("weight_norm", ctypes.c_int32),
        ("factor", ctypes.c_int32),
        ("reg_covar", ctypes.c_double),
        ("resp", ctypes.c_void_p),
        ("weights", ctypes.c_void_p),
        ("means", ctypes.c_void_p),
        ("covariances", ctypes.c_void_p),
        ("prec_chol", ctypes.c_void_p),
        ("lower_bound", ctypes.c_void_p),
        ("status", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p),
        ("workspace_bytes", ctypes.c_size_t),
    ]


NNK_KM_CHANGED, NNK_KM_EMPTY, NNK_KM_SHIFT, NNK_KM_INERTIA, NNK_KM_DISTINCT, NNK_KM_VAR_MEAN = 0, 1, 2, 3, 4, 5
NNK_KM_STATUS_LEN = 8


class NnkKmeansArgs(ctypes.Structure):
    _fields_ = [
        ("X", ctypes.c_void_p),
        ("N", ctypes.c_int64),
        ("x_ld", ctypes.c_int64),
        ("dtype", ctypes.c_int32),
        ("D", ctypes.c_int32),
        ("K", ctypes.c_int32),
        ("centre", ctypes.c_int32),
        ("update", ctypes.c_int32),
        ("first", ctypes.c_int64),
        ("rand", ctypes.c_void_p),
        ("centers", ctypes.c_void_p),
        ("sums", ctypes.c_void_p),
        ("weights", ctypes.c_void_p),
        ("labels", ctypes.c_void_p),
        ("indices", ctypes.c_void_p),
        ("mean", ctypes.c_void_p),
        ("dist", ctypes.c_void_p),
        ("out_centers", ctypes.c_void_p),
        ("status", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p),
        ("workspace_bytes", ctypes.c_size_t),
    ]


class NnkDtwArgs(ctypes.Structure):
    _fields_ = [
        ("X", ctypes.c_void_p),
        ("Y", ctypes.c_void_p),
        ("dtype", ctypes.c_int32),
        ("n_pairs", ctypes.c_int32),
        ("x_pair_stride", ctypes.c_int64),
        ("y_pair_stride", ctypes.c_int64),
        ("x_ld", ctypes.c_int32),
        ("y_ld", ctypes.c_int32),
        ("D", ctypes.c_int32),
        ("len_x", ctypes.c_void_p),
        ("len_y", ctypes.c_void_p),
        ("order", ctypes.c_void_p),
        ("cost_kind", ctypes.c_int32),
        ("radius", ctypes.c_int32),
        ("path_i", ctypes.c_void_p),
        ("path_j", ctypes.c_void_p),
        ("path_ld", ctypes.c_int32),
        ("path_len", ctypes.c_void_p),
        ("dist", ctypes.c_void_p),
        ("cells", ctypes.c_void_p),
        ("max_tx", ctypes.c_int32),
        ("max_ty", ctypes.c_int32),
        ("workspace", ctypes.c_void_p),
        ("workspace_bytes", ctypes.c_size_t),
    ]


CHAIN_DTYPE = np.dtype([("in_col", np.int32), ("win_stride", np.int32), ("out_col", np.int32), ("flags", np.int32)])

# every symbol include/nnk_b200.h declares (tests check the library exports all of them)
EXPORTS = [
    "nnk_abi_version", "nnk_last_error", "nnk_launch_count", "nnk_status_decode",
    "nnk_mlpg_fwd", "nnk_mlpg_grad", "nnk_mlpg_solve", "nnk_mlpg_workspace_bytes", "nnk_mlpg_host", "nnk_mlpg_batch_host",
    "nnk_uv_band_profile", "nnk_uv_band_extract", "nnk_uv_apply", "nnk_uv_apply_toeplitz", "nnk_uv_apply_factored",
    "nnk_dtw_align", "nnk_dtw_workspace_bytes", "nnk_gather_rows", "nnk_trim_lengths", "nnk_delta_features",
    "nnk_metric_workspace_bytes", "nnk_frame_metric", "nnk_f0_metric", "nnk_segment_copy", "nnk_gmm_logprob", "nnk_gmm_map",
    "nnk_gmm_em_workspace_bytes", "nnk_gmm_em_estep", "nnk_gmm_em_mstep", "nnk_gmm_em_factor",
    "nnk_kmeans_workspace_bytes", "nnk_kmeans_prepare", "nnk_kmeans_seed", "nnk_kmeans_lloyd", "nnk_kmeans_relocate_dist",
    "nnk_kmeans_average", "nnk_kmeans_inertia",
    "nnk_postfilter_basis_elems", "nnk_postfilter_basis", "nnk_postfilter_apply",
    "nnk_frame_stats_workspace_bytes", "nnk_frame_stats", "nnk_column_affine",
    "nnk_f0_interp_workspace_bytes", "nnk_f0_interp", "nnk_preemphasis_workspace_bytes", "nnk_preemphasis", "nnk_mulaw",
    "nnk_peer_alloc", "nnk_peer_free", "nnk_peer_export", "nnk_peer_open", "nnk_peer_close", "nnk_peer_copy",
]


class NnkError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "nnmnkwii_b200: %s is missing. Build it with `python -m nnmnkwii_b200.build` "
            "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    L.nnk_abi_version.restype = ctypes.c_int
    if L.nnk_abi_version() != ABI_VERSION:
        raise ImportError("libnnk_b200.so ABI %d != binding ABI %d: rebuild" % (L.nnk_abi_version(), ABI_VERSION))
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
    L.nnk_last_error.restype = ctypes.c_char_p
    L.nnk_launch_count.restype = ctypes.c_int64
    L.nnk_status_decode.restype = None
    L.nnk_status_decode.argtypes = [ctypes.c_uint64, ctypes.POINTER(NnkStatus)]
    L.nnk_mlpg_fwd.restype = ctypes.c_int
    L.nnk_mlpg_fwd.argtypes = [ctypes.POINTER(NnkMlpgArgs), vp]
    L.nnk_mlpg_grad.restype = ctypes.c_int
    L.nnk_mlpg_grad.argtypes = [ctypes.POINTER(NnkMlpgArgs), vp]
    L.nnk_mlpg_solve.restype = ctypes.c_int
    L.nnk_mlpg_solve.argtypes = [ctypes.POINTER(NnkMlpgArgs), vp]
    L.nnk_mlpg_workspace_bytes.restype = ctypes.c_size_t
    L.nnk_mlpg_workspace_bytes.argtypes = [i32, i32, i32, ctypes.POINTER(NnkWindows)]
    L.nnk_mlpg_host.restype = ctypes.c_int
    L.nnk_mlpg_host.argtypes = [vp, vp, i32, i32, i64, i64, ctypes.POINTER(NnkWindows), vp, ctypes.POINTER(i32)]
    L.nnk_mlpg_batch_host.restype = ctypes.c_int
    L.nnk_mlpg_batch_host.argtypes = [vp, vp, i32, i32, i64, i64, i64, vp, i32, vp, i32,
                                      ctypes.POINTER(NnkWindows), vp, ctypes.POINTER(NnkStatus)]
    L.nnk_uv_band_profile.restype = ctypes.c_int
    L.nnk_uv_band_profile.argtypes = [vp, i32, i32, i32, vp, vp]
    L.nnk_uv_band_extract.restype = ctypes.c_int
    L.nnk_uv_band_extract.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp]
    L.nnk_uv_apply.restype = ctypes.c_int
    L.nnk_uv_apply.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, vp]
    L.nnk_uv_apply_toeplitz.restype = ctypes.c_int
    L.nnk_uv_apply_toeplitz.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp]
    L.nnk_uv_apply_factored.restype = ctypes.c_int
    L.nnk_uv_apply_factored.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp]
    L.nnk_dtw_align.restype = ctypes.c_int
    L.nnk_dtw_align.argtypes = [ctypes.POINTER(NnkDtwArgs), vp]
    L.nnk_dtw_workspace_bytes.restype = ctypes.c_size_t
    L.nnk_dtw_workspace_bytes.argtypes = [i32, i32, i32, i32, i32]
    L.nnk_gather_rows.restype = ctypes.c_int
    L.nnk_gather_rows.argtypes = [vp, i32, i64, i32, vp, i32, vp, vp, i64, i32, i32, i32, vp]
    L.nnk_trim_lengths.restype = ctypes.c_int
    L.nnk_trim_lengths.argtypes = [vp, i32, i64, i32, i32, i32, ctypes.c_double, i32, vp, vp]
    L.nnk_delta_features.restype = ctypes.c_int
    L.nnk_delta_features.argtypes = [vp, i32, i32, i64, vp, vp, i32, i32, ctypes.POINTER(NnkWindows), vp, i64, vp]
    L.nnk_metric_workspace_bytes.restype = i64
    L.nnk_metric_workspace_bytes.argtypes = [i32, i32]
    L.nnk_frame_metric.restype = ctypes.c_int
    L.nnk_frame_metric.argtypes = [vp, vp, i32, i32, i32, i32, i64, i64, vp, i32, vp, vp, vp, i64, vp]
    L.nnk_f0_metric.restype = ctypes.c_int
    L.nnk_f0_metric.argtypes = [vp, vp, vp, vp, i32, i32, i32, i64, i64, vp, i32, vp, vp, vp, i64, vp]
    for name, args in (("nnk_peer_alloc", [ctypes.c_size_t, ctypes.POINTER(vp)]), ("nnk_peer_free", [vp]),
                       ("nnk_peer_export", [vp, vp]), ("nnk_peer_open", [vp, ctypes.POINTER(vp)]), ("nnk_peer_close", [vp]),
                       ("nnk_peer_copy", [vp, vp, ctypes.c_size_t, vp])):
        getattr(L, name).restype = ctypes.c_int
        getattr(L, name).argtypes = args
    L.nnk_gmm_logprob.restype = ctypes.c_int
    L.nnk_gmm_logprob.argtypes = [ctypes.POINTER(NnkGmm), vp, i64, i32, vp, vp]
    L.nnk_gmm_map.restype = ctypes.c_int
    L.nnk_gmm_map.argtypes = [ctypes.POINTER(NnkGmm), vp, i64, i32, vp, i32, vp, vp, vp, vp]
    L.nnk_gmm_em_workspace_bytes.restype = ctypes.c_size_t
    L.nnk_gmm_em_workspace_bytes.argtypes = [i64, i32, i32]
    for name in ("nnk_gmm_em_estep", "nnk_gmm_em_mstep", "nnk_gmm_em_factor"):
        getattr(L, name).restype = ctypes.c_int
        getattr(L, name).argtypes = [ctypes.POINTER(NnkGmmEmArgs), vp]
    L.nnk_kmeans_workspace_bytes.restype = ctypes.c_size_t
    L.nnk_kmeans_workspace_bytes.argtypes = [i64, i32, i32]
    for name in ("nnk_kmeans_prepare", "nnk_kmeans_seed", "nnk_kmeans_lloyd", "nnk_kmeans_relocate_dist",
                 "nnk_kmeans_average", "nnk_kmeans_inertia"):
        getattr(L, name).restype = ctypes.c_int
        getattr(L, name).argtypes = [ctypes.POINTER(NnkKmeansArgs), vp]
    L.nnk_postfilter_basis_elems.restype = i64
    L.nnk_postfilter_basis_elems.argtypes = [i32, i32]
    L.nnk_postfilter_basis.restype = ctypes.c_int
    L.nnk_postfilter_basis.argtypes = [ctypes.c_double, i32, i32, i32, vp, i64, vp]
    L.nnk_postfilter_apply.restype = ctypes.c_int
    L.nnk_postfilter_apply.argtypes = [vp, i32, i64, i32, i64, vp, i32, vp, i64, vp, i64, vp]
    L.nnk_frame_stats_workspace_bytes.restype = i64
    L.nnk_frame_stats_workspace_bytes.argtypes = [i32, i32, i32]
    L.nnk_frame_stats.restype = ctypes.c_int
    L.nnk_frame_stats.argtypes = [vp, i32, i32, i64, vp, vp, i32, i32, vp, vp, i64, vp]
    L.nnk_column_affine.restype = ctypes.c_int
    L.nnk_column_affine.argtypes = [vp, i32, i32, i64, i32, vp, vp, i32, vp, vp]
    L.nnk_f0_interp_workspace_bytes.restype = i64
    L.nnk_f0_interp_workspace_bytes.argtypes = [i32, i32]
    L.nnk_f0_interp.restype = ctypes.c_int
    L.nnk_f0_interp.argtypes = [vp, vp, i32, i32, i32, vp, i32, vp, i64, vp]
    L.nnk_preemphasis_workspace_bytes.restype = i64
    L.nnk_preemphasis_workspace_bytes.argtypes = [i32, i64, i64, ctypes.c_double, i32]
    L.nnk_preemphasis.restype = ctypes.c_int
    L.nnk_preemphasis.argtypes = [vp, vp, i32, i64, i64, vp, ctypes.c_double, i32, vp, i64, vp, vp]
    L.nnk_mulaw.restype = ctypes.c_int
    L.nnk_mulaw.argtypes = [vp, i32, vp, i32, i32, i64, ctypes.c_double, vp]
    L.nnk_segment_copy.restype = ctypes.c_int
    L.nnk_segment_copy.argtypes = [vp, vp, i32, i64, i64, i64, vp, vp, vp, i32, i32, vp]
    return L


lib = _load()


def last_error():
    return lib.nnk_last_error().decode("utf-8", "replace")


def launch_count():
    return int(lib.nnk_launch_count())


def make_windows(windows):
    """Python list of (l, u, coeff) triples -> NnkWindows; validates like build_win_mats (_mlpg.py:44-45)."""
    if len(windows) > NNK_MAX_WIN:
        raise NotImplementedError("at most %d windows are supported by the CUDA kernels (got %d)" % (NNK_MAX_WIN, len(windows)))
    w = NnkWindows()
    w.nw = len(windows)
    for i, (l, u, c) in enumerate(windows):
        l, u = int(l), int(u)
        c = np.asarray(c, dtype=np.float64).ravel()
        assert l >= 0 and u >= 0
        assert len(c) == l + u + 1
        if l > NNK_MAX_HALF or u > NNK_MAX_HALF:
            raise NotImplementedError("window half-width > %d is not supported by the CUDA kernels" % NNK_MAX_HALF)
        w.l[i], w.u[i] = l, u
        for k in range(l + u + 1):
            w.coef[i][k] = float(c[k])
    return w


def check(rc, what="nnk call"):
    if rc == NNK_OK:
        return
    msg = last_error()
    if rc == NNK_ERR_UNSUPPORTED:
        raise NotImplementedError("%s: %s" % (what, msg))
    if rc == NNK_ERR_NOT_PD:
        raise np.linalg.LinAlgError(msg)
    if rc == NNK_ERR_ARG:
        raise ValueError("%s: %s" % (what, msg))
    raise NnkError("%s failed (%d): %s" % (what, rc, msg))
