"""DTW alignment -- drop-in for ``nnmnkwii.preprocessing.alignment`` (alignment.py:9-190):
``DTWAligner`` and ``IterativeDTWAligner`` with the reference's constructor arguments, defaults,
return shapes / dtypes and padding behaviour.

The reference loops over utterance pairs in Python and calls the third-party ``fastdtw`` with a
Python callable evaluated per DP cell.  Here the whole batch is aligned by one launch of the
sm_90a wavefront kernel (csrc/nnk_dtw.cu, one thread block per pair), followed by a device gather.
``dist`` is therefore not called: the two costs the reference ships are recognised --

* the default ``lambda x, y: norm(x - y)``  -> Euclidean (``cost_kind`` 0)
* ``melcd`` (this package's or the reference's ``nnmnkwii.metrics.melcd``) -> ``cost_kind`` 1

-- by identity, by name (``"euclidean"`` / ``"melcd"``) or, for any other callable, by what it
computes on a few probe frames (so the reference's own default lambda, or a user's re-spelling of it,
is served natively); a callable that computes something else raises ``NotImplementedError`` (no
per-cell CPU fallback).
``radius`` follows fastdtw (default 1); the additive ``radius=None`` / negative selects exact DTW.
"""
import ctypes

import numpy as np
from numpy.linalg import norm

from .. import _lib
from ..metrics import _logdb_const as _melcd_const
from ..metrics import melcd as _melcd


def _default_dist(x, y):
    return norm(x - y)


_PROBE = np.random.default_rng(20260923).standard_normal((6, 2, 13))


def _probe_cost(dist):
    """Which built-in local cost does a user callable compute?  It is evaluated on a handful of fixed
    probe frames (host, once per aligner call, never per DP cell) and compared with the two costs
    the kernel evaluates: returns 0 (Euclidean ``norm(x - y)``), 1 (``melcd``) or None."""
    try:
        got = np.array([float(dist(x, y)) for x, y in _PROBE])
    except Exception:
        return None
    euclid = np.array([float(norm(x - y)) for x, y in _PROBE])
    for kind, want in ((0, euclid), (1, _melcd_const * euclid)):
        if np.allclose(got, want, rtol=1e-9, atol=0.0):
            return kind
    return None


def _cost_kind(dist):
    if dist is _default_dist or dist is None or dist == "euclidean":
        return 0
    if dist is _melcd or dist == "melcd" or (
            getattr(dist, "__name__", "") == "melcd" and "metrics" in getattr(dist, "__module__", "")):
        return 1
    if dist is norm:
        raise NotImplementedError("dist must take two frames (x, y)")
    # any callable that COMPUTES one of the two costs (e.g. the reference's own default
    # ``lambda x, y: norm(x - y)``, alignment.py:35, or a user's re-spelling of it) is served natively
    kind = _probe_cost(dist) if callable(dist) else None
    if kind is not None:
        return kind
    raise NotImplementedError(
        "nnmnkwii_b200 DTW evaluates the local cost inside the CUDA kernel; supported `dist`: callables that "
        "compute the Euclidean norm(x - y) (the reference default) or metrics.melcd, or the names 'euclidean' / "
        "'melcd'. Other Python callables would need a per-cell CPU callback, which this implementation does not "
        "provide.")


class _Aligned(object):
    """Device-side result of one batched alignment."""
    __slots__ = ("path_i", "path_j", "path_len", "dist", "cells", "len_x", "len_y", "Xd", "Yd")


def _align_batch(X, Y, cost_kind, radius, want_cells=False):
    """Run trim -> DTW for all pairs on the GPU.  X, Y: torch CUDA tensors (N, T, D)."""
    import torch

    from .. import _device as dev

    device = X.device
    N, Tx, D = X.shape
    Ty = Y.shape[1]
    assert Y.shape[0] == N and Y.shape[2] == D
    work = torch.float32 if (X.dtype == torch.float32 and Y.dtype == torch.float32) else torch.float64
    Xd = X.to(work).contiguous()
    Yd = Y.to(work).contiguous()
    code = dev.torch_dtype_code(work)
    st = dev.current_stream_ptr(device)
    res = _Aligned()
    res.Xd, res.Yd = Xd, Yd
    res.len_x = torch.empty(N, dtype=torch.int32, device=device)
    res.len_y = torch.empty(N, dtype=torch.int32, device=device)
    _lib.check(_lib.lib.nnk_trim_lengths(Xd.data_ptr(), code, Tx * D, D, Tx, D, 1e-7, N, res.len_x.data_ptr(), st), "nnk_trim_lengths")
    _lib.check(_lib.lib.nnk_trim_lengths(Yd.data_ptr(), code, Ty * D, D, Ty, D, 1e-7, N, res.len_y.data_ptr(), st), "nnk_trim_lengths")
    path_ld = max(1, Tx + Ty)
    res.path_i = torch.empty((N, path_ld), dtype=torch.int32, device=device)
    res.path_j = torch.empty((N, path_ld), dtype=torch.int32, device=device)
    res.path_len = torch.zeros(N, dtype=torch.int32, device=device)
    res.dist = torch.zeros(N, dtype=torch.float64, device=device)
    res.cells = torch.zeros(N, dtype=torch.int64, device=device)
    r = -1 if (radius is None or radius < 0) else int(radius)
    nbytes = _lib.lib.nnk_dtw_workspace_bytes(N, Tx, Ty, D, r)
    ws = dev.workspace(device, max(256, nbytes))
    # longest pairs first
    order = torch.argsort((res.len_x.to(torch.int64) * res.len_y.to(torch.int64)), descending=True).to(torch.int32)
    a = _lib.NnkDtwArgs()
    a.X, a.Y, a.dtype, a.n_pairs = Xd.data_ptr(), Yd.data_ptr(), code, N
    a.x_pair_stride, a.y_pair_stride, a.x_ld, a.y_ld, a.D = Tx * D, Ty * D, D, D, D
    a.len_x, a.len_y, a.order = res.len_x.data_ptr(), res.len_y.data_ptr(), order.data_ptr()
    a.cost_kind, a.radius = cost_kind, r
    a.path_i, a.path_j, a.path_ld = res.path_i.data_ptr(), res.path_j.data_ptr(), path_ld
    a.path_len, a.dist, a.cells = res.path_len.data_ptr(), res.dist.data_ptr(), res.cells.data_ptr()
    a.max_tx, a.max_ty = Tx, Ty
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    _lib.check(_lib.lib.nnk_dtw_align(ctypes.byref(a), st), "nnk_dtw_align")
    return res


def _gather(src, path, path_len, out_rows):
    """(N, out_rows, D) = src[n, path[n, :L]] zero-padded, on the device."""
    import torch

    from .. import _device as dev

    N, T, D = src.shape
    out = torch.empty((N, out_rows, D), dtype=src.dtype, device=src.device)
    _lib.check(_lib.lib.nnk_gather_rows(src.data_ptr(), dev.torch_dtype_code(src.dtype), T * D, D, path.data_ptr(),
                                        path.shape[1], path_len.data_ptr(), out.data_ptr(), out_rows * D, out_rows, D, N,
                                        dev.current_stream_ptr(src.device)), "nnk_gather_rows")
    return out


def _to_device(A):
    from .. import _device as dev

    dev.require_cuda()
    if dev.is_tensor(A):
        assert A.is_cuda, "torch inputs must be CUDA tensors"
        return A, True
    A = np.asarray(A)
    if A.dtype not in (np.float32, np.float64):
        A = A.astype(np.float64)
    return dev.to_device(A), False


class DTWAligner(object):
    """Align feature matrices with (Fast)DTW on the GPU.

    Attributes:
        dist (function): distance function; default ``lambda x, y: norm(x - y)``; ``melcd`` supported.
        radius (int): radius parameter of FastDTW (default 1); ``None`` or negative = exact DTW.
        verbose (int): verbose flag.

    Examples:
        >>> X_aligned, Y_aligned = DTWAligner().transform((X, Y))     # X, Y: (N, T, D) zero padded
    """

    def __init__(self, dist=_default_dist, radius=1, verbose=0):
        self.verbose = verbose
        self.dist = dist
        self.radius = radius

    def transform(self, XY):
        import torch

        X, Y = XY
        assert X.ndim == 3 and Y.ndim == 3
        kind = _cost_kind(self.dist)
        Xd, x_is_t = _to_device(X)
        Yd, _ = _to_device(Y)
        longer_is_x = X.shape[1] > Y.shape[1]  # alignment.py:44
        out_dtype = (Xd if longer_is_x else Yd).dtype
        res = _align_batch(Xd, Yd, kind, self.radius)
        L = res.path_len.cpu().numpy()
        if (L < 0).any():
            raise RuntimeError("DTW back-track failed (internal error)")
        out_rows = max(max(X.shape[1], Y.shape[1]), int(L.max(initial=0)))  # np.pad growth, alignment.py:55-71
        Xa = _gather(res.Xd, res.path_i, res.path_len, out_rows).to(out_dtype)
        Ya = _gather(res.Yd, res.path_j, res.path_len, out_rows).to(out_dtype)
        if self.verbose > 0:
            d = res.dist.cpu().numpy()
            lx, ly = res.len_x.cpu().numpy(), res.len_y.cpu().numpy()
            for idx in range(len(d)):
                print("{}, distance: {}".format(idx, d[idx] / (lx[idx] + ly[idx])))
        self.last_ = res
        if x_is_t:
            return Xa, Ya
        torch.cuda.current_stream().synchronize()
        np_dtype = (X if longer_is_x else Y).dtype if isinstance(X, np.ndarray) else None
        Xa, Ya = Xa.cpu().numpy(), Ya.cpu().numpy()
        if np_dtype is not None and Xa.dtype != np_dtype:
            Xa, Ya = Xa.astype(np_dtype), Ya.astype(np_dtype)
        return Xa, Ya


class IterativeDTWAligner(object):
    """Align feature matrices iteratively using GMM-based feature conversion (alignment.py:79-190).

    Per iteration: DTW of the converted source against the target (GPU), joint-GMM fit on the
    aligned (zero padded) frames, frame-wise GMM mapping of the source.  Finally the ORIGINAL source
    is gathered along the last paths.

    ``gmm`` (additive) picks who fits the joint GMM: ``"sklearn"`` (default, scikit-learn on the host,
    as in the reference) or ``"device"`` (:class:`nnmnkwii_b200.baseline.gmm.GaussianMixture`, EM on the
    GPU in float64, same ``n_components``, ``max_iter`` and ``random_state``).  The two are not
    bit-identical: scikit-learn fits float32 frames in float32, and even on float64 frames the
    summation order differs in the last bits.  ``gmm_init_device=True`` (with ``gmm="device"`` only) runs
    that fit's k-means initialisation on the GPU too (``GaussianMixture(init_device=True)``).
    """

    def __init__(self, n_iter=3, dist=_default_dist, radius=1, max_iter_gmm=100, n_components_gmm=16, verbose=0,
                 random_state=None, gmm="sklearn", gmm_init_device=False):
        if gmm not in ("sklearn", "device"):
            raise ValueError("gmm must be 'sklearn' or 'device' (got %r)" % (gmm,))
        if gmm_init_device and gmm != "device":
            raise ValueError("gmm_init_device=True needs gmm='device' (got gmm=%r)" % (gmm,))
        self.n_iter = n_iter
        self.dist = dist
        self.radius = radius
        self.max_iter_gmm = max_iter_gmm
        self.n_components_gmm = n_components_gmm
        self.verbose = verbose
        self.random_state = random_state  # additive: the reference leaves the GMM unseeded
        self.gmm = gmm
        self.gmm_init_device = gmm_init_device

    def transform(self, XY):
        import torch

        from . import trim_zeros_frames
        from ..baseline.gmm import MLPG
        if self.gmm == "device":
            from ..baseline.gmm import GaussianMixture
        else:
            from sklearn.mixture import GaussianMixture

        X, Y = XY
        assert X.ndim == 3 and Y.ndim == 3
        kind = _cost_kind(self.dist)
        X = np.asarray(X)
        Y = np.asarray(Y)
        longer_features = X if X.shape[1] > Y.shape[1] else Y
        Xc = X.copy()  # updated iteratively
        X_aligned = np.zeros_like(longer_features)
        Y_aligned = np.zeros_like(longer_features)
        Yd, _ = _to_device(Y)
        Xd0, _ = _to_device(X)
        res = None
        for _ in range(self.n_iter):
            Xcd, _ = _to_device(Xc)
            res = _align_batch(Xcd, Yd, kind, self.radius)
            L = res.path_len.cpu().numpy()
            out_rows = max(X_aligned.shape[1], int(L.max(initial=0)))
            if out_rows > X_aligned.shape[1]:  # np.pad growth (alignment.py:148-164)
                pad = out_rows - X_aligned.shape[1]
                X_aligned = np.pad(X_aligned, [(0, 0), (0, pad), (0, 0)], mode="constant", constant_values=0)
                Y_aligned = np.pad(Y_aligned, [(0, 0), (0, pad), (0, 0)], mode="constant", constant_values=0)
            xa = _gather(res.Xd, res.path_i, res.path_len, out_rows).cpu().numpy()
            ya = _gather(res.Yd, res.path_j, res.path_len, out_rows).cpu().numpy()
            for idx in range(len(L)):  # only the first L rows are overwritten, stale tails stay (alignment.py:166-167)
                X_aligned[idx][: L[idx]] = xa[idx][: L[idx]]
                Y_aligned[idx][: L[idx]] = ya[idx][: L[idx]]
            if self.verbose > 0:
                d = res.dist.cpu().numpy()
                lx, ly = res.len_x.cpu().numpy(), res.len_y.cpu().numpy()
                for idx in range(len(d)):
                    print("{}, distance: {}".format(idx, d[idx] / (lx[idx] + ly[idx])))
            init_kw = {"init_device": True} if self.gmm_init_device else {}
            gmm = GaussianMixture(n_components=self.n_components_gmm, covariance_type="full", max_iter=self.max_iter_gmm,
                                  random_state=self.random_state, **init_kw)
            XYj = np.concatenate((X_aligned, Y_aligned), axis=-1).reshape(-1, X.shape[-1] * 2)
            gmm.fit(XYj)
            paramgen = MLPG(gmm, windows=[(0, 0, np.array([1.0]))])  # no delta (alignment.py:179-180)
            trimmed = [trim_zeros_frames(Xc[idx]) for idx in range(len(Xc))]
            for idx, y in enumerate(paramgen.transform_batch(trimmed)):  # one device pass for all utterances
                Xc[idx][: len(y)] = y
        # finally gather the ORIGINAL X along the last paths (alignment.py:186-188)
        if res is not None:
            out_rows = X_aligned.shape[1]
            L = res.path_len.cpu().numpy()
            xa = _gather(Xd0.to(res.Xd.dtype).contiguous(), res.path_i, res.path_len, out_rows).cpu().numpy()
            for idx in range(len(L)):
                X_aligned[idx][: L[idx]] = xa[idx][: L[idx]]
        self.last_ = res
        del torch
        return X_aligned, Y_aligned


__all__ = ["DTWAligner", "IterativeDTWAligner"]
