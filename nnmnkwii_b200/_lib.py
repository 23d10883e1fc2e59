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


class NnkMlpgGv(ctypes.Structure):
    _fields_ = [
        ("gv_mean", ctypes.c_void_p),
        ("gv_var", ctypes.c_void_p),
        ("n_iter", ctypes.c_int32),
        ("step", ctypes.c_double),
        ("weight", ctypes.c_double),
    ]


class NnkGmm(ctypes.Structure):
    _fields_ = [
        ("src_means", ctypes.c_void_p), ("tgt_means", ctypes.c_void_p), ("prec_chol", ctypes.c_void_p),
        ("log_const", ctypes.c_void_p), ("A_t", ctypes.c_void_p), ("Dm", ctypes.c_void_p),
        ("M", ctypes.c_int32), ("D", ctypes.c_int32),
    ]


NNK_GMM_TRAJ_EM, NNK_GMM_TRAJ_OBJECTIVE, NNK_GMM_TRAJ_TILE = 0, 1, 32


class NnkGmmTrajArgs(ctypes.Structure):
    _fields_ = [
        ("x", ctypes.c_void_p),
        ("x_ld", ctypes.c_int64),
        ("lp", ctypes.c_void_p),
        ("c", ctypes.c_void_p),
        ("c_ld", ctypes.c_int64),
        ("T", ctypes.c_int32),
        ("n_utt", ctypes.c_int32),
        ("utt_off", ctypes.c_void_p),
        ("tile_off", ctypes.c_void_p),
        ("n_tiles", ctypes.c_int32),
        ("static_dim", ctypes.c_int32),
        ("win", NnkWindows),
        ("mode", ctypes.c_int32),
        ("inv_Dm", ctypes.c_void_p),
        ("log_norm", ctypes.c_void_p),
        ("E_bar", ctypes.c_void_p),
        ("V", ctypes.c_void_p),
        ("ll_part", ctypes.c_void_p),
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
NNK_MS_POWER, NNK_MS_SMOOTH, NNK_MS_INVERSE, NNK_MS_GRAD, NNK_MS_LOGPOWER, NNK_MS_POSTFILTER = 0, 1, 2, 3, 4, 5


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


NNK_MSSEG_LOGPOWER, NNK_MSSEG_POSTFILTER = 0, 1


class NnkMlpgMs(ctypes.Structure):
    _fields_ = [
        ("ms_mean", ctypes.c_void_p),
        ("ms_var", ctypes.c_void_p),
        ("n", ctypes.c_int32),
        ("n_iter", ctypes.c_int32),
        ("step", ctypes.c_double),
        ("weight", ctypes.c_double),
        ("n_rows", ctypes.c_int64),
    ]


NNK_MIX_GEN_SELECT, NNK_MIX_GEN_ESTEP, NNK_MIX_GEN_OBJECTIVE = 0, 1, 2
NNK_MIX_GEN_TILE, NNK_MIX_GEN_MAX_D, NNK_MIX_GEN_MAX_M = 32, 256, 64


class NnkMixGenArgs(ctypes.Structure):
    _fields_ = [
        ("log_weights", ctypes.c_void_p),
        ("means", ctypes.c_void_p),
        ("vars", ctypes.c_void_p),
        ("dtype", ctypes.c_int32),
        ("M", ctypes.c_int32),
        ("D", ctypes.c_int32),
        ("n_utt", ctypes.c_int32),
        ("utt_off", ctypes.c_void_p),
        ("utt_len", ctypes.c_void_p),
        ("tile_off", ctypes.c_void_p),
        ("n_tiles", ctypes.c_int32),
        ("col_map", ctypes.c_void_p),
        ("win", NnkWindows),
        ("mode", ctypes.c_int32),
        ("c", ctypes.c_void_p),
        ("c_ld", ctypes.c_int64),
        ("c_cols", ctypes.c_int32),
        ("lnorm", ctypes.c_void_p),
        ("E", ctypes.c_void_p),
        ("V", ctypes.c_void_p),
        ("ll_part", ctypes.c_void_p),
        ("status_word", ctypes.c_void_p),
    ]


class NnkTrajLl(ctypes.Structure):
    _fields_ = [
        ("targets", ctypes.c_void_p),
        ("tgt_ld", ctypes.c_int64),
        ("ll", ctypes.c_void_p),
        ("grad", ctypes.c_int32),
        ("grad_means", ctypes.c_void_p),
        ("gm_ld", ctypes.c_int64),
        ("grad_vars", ctypes.c_void_p),
        ("gv_ld", ctypes.c_int64),
        ("grad_targets", ctypes.c_void_p),
        ("gx_ld", ctypes.c_int64),
    ]


class NnkTrajSample(ctypes.Structure):
    _fields_ = [
        ("sample_stride", ctypes.c_int64),
        ("n_samples", ctypes.c_int32),
        ("seed", ctypes.c_uint64),
        ("keys", ctypes.c_void_p),
        ("scale", ctypes.c_double),
    ]


class NnkMlpgVjp(ctypes.Structure):
    _fields_ = [
        ("grad_out", ctypes.c_void_p),
        ("go_ld", ctypes.c_int64),
        ("grad_means", ctypes.c_void_p),
        ("gm_ld", ctypes.c_int64),
        ("grad_vars", ctypes.c_void_p),
        ("gv_ld", ctypes.c_int64),
    ]


CHAIN_DTYPE = np.dtype([("in_col", np.int32), ("win_stride", np.int32), ("out_col", np.int32), ("flags", np.int32)])

P, vp, i32, i64, f64 = ctypes.POINTER, ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_double
size_t = ctypes.c_size_t
_MLPG, _GMM_EM, _KMEANS = [P(NnkMlpgArgs), vp], [P(NnkGmmEmArgs), vp], [P(NnkKmeansArgs), vp]

# name -> (restype, argtypes) of every function include/nnk_b200.h declares (tests check both against it)
SIGNATURES = {
    "nnk_abi_version": (ctypes.c_int, []),
    "nnk_last_error": (ctypes.c_char_p, []),
    "nnk_launch_count": (i64, []),
    "nnk_status_decode": (None, [ctypes.c_uint64, P(NnkStatus)]),
    "nnk_mlpg_fwd": (ctypes.c_int, _MLPG),
    "nnk_mlpg_grad": (ctypes.c_int, _MLPG),
    "nnk_mlpg_solve": (ctypes.c_int, _MLPG),
    "nnk_mlpg_workspace_bytes": (size_t, [i32, i32, i32, P(NnkWindows)]),
    "nnk_mlpg_gv": (ctypes.c_int, [P(NnkMlpgArgs), P(NnkMlpgGv), vp]),
    "nnk_mlpg_gv_workspace_bytes": (size_t, [i32, i32, i32, P(NnkWindows)]),
    "nnk_segment_moments": (ctypes.c_int, [vp, i32, i32, i64, vp, vp, i32, vp, vp, vp]),
    "nnk_mlpg_host": (ctypes.c_int, [vp, vp, i32, i32, i64, i64, P(NnkWindows), vp, P(i32)]),
    "nnk_mlpg_batch_host": (ctypes.c_int, [vp, vp, i32, i32, i64, i64, i64, vp, i32, vp, i32, P(NnkWindows), vp,
                                           P(NnkStatus)]),
    "nnk_uv_band_profile": (ctypes.c_int, [vp, i32, i32, i32, vp, vp]),
    "nnk_uv_band_extract": (ctypes.c_int, [vp, i32, i32, i32, i32, vp, vp, vp]),
    "nnk_uv_apply": (ctypes.c_int, [vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, vp]),
    "nnk_uv_apply_toeplitz": (ctypes.c_int, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp]),
    "nnk_uv_apply_factored": (ctypes.c_int, [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp]),
    "nnk_dtw_align": (ctypes.c_int, [P(NnkDtwArgs), vp]),
    "nnk_dtw_workspace_bytes": (size_t, [i32, i32, i32, i32, i32]),
    "nnk_gather_rows": (ctypes.c_int, [vp, i32, i64, i32, vp, i32, vp, vp, i64, i32, i32, i32, vp]),
    "nnk_trim_lengths": (ctypes.c_int, [vp, i32, i64, i32, i32, i32, f64, i32, vp, vp]),
    "nnk_cholesky_inv": (ctypes.c_int, [vp, i32, i32, i32, vp, vp, vp]),
    "nnk_cholesky_inv_banded": (ctypes.c_int, [vp, i32, i32, i32, vp, vp, vp]),
    "nnk_delta_features": (ctypes.c_int, [vp, i32, i32, i64, vp, vp, i32, i32, P(NnkWindows), vp, i64, vp]),
    "nnk_metric_workspace_bytes": (i64, [i32, i32]),
    "nnk_frame_metric": (ctypes.c_int, [vp, vp, i32, i32, i32, i32, i64, i64, vp, i32, vp, vp, vp, i64, vp]),
    "nnk_f0_metric": (ctypes.c_int, [vp, vp, vp, vp, i32, i32, i32, i64, i64, vp, i32, vp, vp, vp, i64, vp]),
    "nnk_segment_copy": (ctypes.c_int, [vp, vp, i32, i64, i64, i64, vp, vp, vp, i32, i32, vp]),
    "nnk_gmm_logprob": (ctypes.c_int, [P(NnkGmm), vp, i64, i32, vp, vp]),
    "nnk_gmm_map": (ctypes.c_int, [P(NnkGmm), vp, i64, i32, vp, i32, vp, vp, vp, vp]),
    "nnk_gmm_traj_em": (ctypes.c_int, [P(NnkGmm), P(NnkGmmTrajArgs), vp]),
    "nnk_gmm_em_workspace_bytes": (size_t, [i64, i32, i32]),
    "nnk_gmm_em_estep": (ctypes.c_int, _GMM_EM),
    "nnk_gmm_em_mstep": (ctypes.c_int, _GMM_EM),
    "nnk_gmm_em_factor": (ctypes.c_int, _GMM_EM),
    "nnk_kmeans_workspace_bytes": (size_t, [i64, i32, i32]),
    "nnk_kmeans_prepare": (ctypes.c_int, _KMEANS),
    "nnk_kmeans_seed": (ctypes.c_int, _KMEANS),
    "nnk_kmeans_lloyd": (ctypes.c_int, _KMEANS),
    "nnk_kmeans_relocate_dist": (ctypes.c_int, _KMEANS),
    "nnk_kmeans_average": (ctypes.c_int, _KMEANS),
    "nnk_kmeans_inertia": (ctypes.c_int, _KMEANS),
    "nnk_postfilter_basis_elems": (i64, [i32, i32]),
    "nnk_postfilter_basis": (ctypes.c_int, [f64, i32, i32, i32, vp, i64, vp]),
    "nnk_postfilter_apply": (ctypes.c_int, [vp, i32, i64, i32, i64, vp, i32, vp, i64, vp, i64, vp]),
    "nnk_frame_stats_workspace_bytes": (i64, [i32, i32, i32]),
    "nnk_frame_stats": (ctypes.c_int, [vp, i32, i32, i64, vp, vp, i32, i32, vp, vp, i64, vp]),
    "nnk_column_affine": (ctypes.c_int, [vp, i32, i32, i64, i32, vp, vp, i32, vp, vp]),
    "nnk_f0_interp_workspace_bytes": (i64, [i32, i32]),
    "nnk_f0_interp": (ctypes.c_int, [vp, vp, i32, i32, i32, vp, i32, vp, i64, vp]),
    "nnk_preemphasis_workspace_bytes": (i64, [i32, i64, i64, f64, i32]),
    "nnk_preemphasis": (ctypes.c_int, [vp, vp, i32, i64, i64, vp, f64, i32, vp, i64, vp, vp]),
    "nnk_mulaw": (ctypes.c_int, [vp, i32, vp, i32, i32, i64, f64, vp]),
    "nnk_modspec": (ctypes.c_int, [i32, i32, i32, vp, vp, vp, vp, i32, i32, i32, i32, vp, f64, f64, i32, i32, vp]),
    "nnk_mlpg_ms": (ctypes.c_int, [P(NnkMlpgArgs), P(NnkMlpgMs), vp]),
    "nnk_mlpg_ms_workspace_bytes": (size_t, [i32, i32, i32, i64, i64, P(NnkWindows)]),
    "nnk_ms_segment": (ctypes.c_int, [i32, i32, i32, i32, vp, vp, vp, i32, i32, i32, vp, vp, vp]),
    "nnk_mlpg_ms_segment": (ctypes.c_int, [P(NnkMlpgArgs), P(NnkMlpgMs), i32, vp]),
    "nnk_mix_gen": (ctypes.c_int, [P(NnkMixGenArgs), vp]),
    "nnk_mlpg_traj_ll": (ctypes.c_int, [P(NnkMlpgArgs), P(NnkTrajLl), vp]),
    "nnk_mlpg_traj_ll_workspace_bytes": (size_t, [i32, i32, i32, P(NnkWindows)]),
    "nnk_mlpg_traj_sample": (ctypes.c_int, [P(NnkMlpgArgs), P(NnkTrajSample), vp]),
    "nnk_mlpg_traj_sample_workspace_bytes": (size_t, [i32, i32, i32, P(NnkWindows)]),
    "nnk_mlpg_vjp": (ctypes.c_int, [P(NnkMlpgArgs), P(NnkMlpgVjp), vp]),
    "nnk_mlpg_vjp_workspace_bytes": (size_t, [i32, i32, i32, P(NnkWindows)]),
    "nnk_peer_alloc": (ctypes.c_int, [size_t, P(vp)]),
    "nnk_peer_free": (ctypes.c_int, [vp]),
    "nnk_peer_export": (ctypes.c_int, [vp, vp]),
    "nnk_peer_open": (ctypes.c_int, [vp, P(vp)]),
    "nnk_peer_close": (ctypes.c_int, [vp]),
    "nnk_peer_copy": (ctypes.c_int, [vp, vp, size_t, vp]),
}
EXPORTS = list(SIGNATURES)


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
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
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
