"""Inverse of a symmetric positive definite matrix from its Cholesky factor -- drop-in for
``nnmnkwii.util.linalg`` (nnmnkwii/util/linalg.py:7-36, util/_linalg.pyx:45-71).

Both functions run on the GPU in float64 (C ABI ``nnk_cholesky_inv`` / ``nnk_cholesky_inv_banded``,
csrc/nnk_linalg.cu), one thread per column of the result.  They return what they were given: a NumPy
array gives a NumPy array, a CUDA (CPU) tensor a CUDA (CPU) tensor.

Additive: a leading batch dimension ``(B, N, N)`` is one launch, and a float32 tensor is computed in
float64 and returned in float32.

``cholesky_inv_banded`` is bit-identical to the reference on finite input, except that an element to
which no term contributes may be +0.0 where the reference's ``hold *= 0.0`` reset gives -0.0.
``cholesky_inv`` cannot be bit-identical to LAPACK's ``dpotri``; it lands within a few ulps of the
result's scale (tests/test_util_cpu.py measures how far a float64 restatement of its order is).

Deliberate differences from the reference:
  * a zero or non-finite diagonal entry of the factor raises ``numpy.linalg.LinAlgError`` naming the
    batch item (the reference ignores ``dpotri``'s ``info`` and returns a partial result);
  * other NaN / inf entries do not follow the reference's propagation through ``hold *= 0.0`` (which
    turns a whole row of ``hold`` into NaN once one element is non-finite); they never fault;
  * ``cholesky_inv_banded`` requires a square matrix and ``width >= 1``, and supports
    ``min(width, T) <= 9`` (``NotImplementedError`` above that).
"""
import ctypes

import numpy as np

from .. import _device as dev
from .. import _lib


def _check_square(L):
    if L.ndim not in (2, 3):
        raise ValueError("expected an (N, N) matrix or a (B, N, N) batch, got shape %s" % (tuple(L.shape),))
    if L.shape[-1] != L.shape[-2]:
        raise AssertionError("the factor must be square, got shape %s" % (tuple(L.shape),))


def _raise_item(status, what):
    word = int(status.item()) & 0xFFFFFFFFFFFFFFFF
    if word:
        st = _lib.NnkStatus()
        _lib.lib.nnk_status_decode(ctypes.c_uint64(word), ctypes.byref(st))
        raise np.linalg.LinAlgError("%s: batch item %d has a zero or non-finite diagonal entry (row %d)"
                                    % (what, st.utt, st.frame - 1))


def _invert(L, fn, arg, what):
    """Run ``fn`` (an nnk_cholesky_inv* entry point) on the float64 device copy of ``L``; the result in the
    form and floating dtype of ``L``."""
    import torch

    dev.require_cuda()
    x = dev.to_device(L)
    d = x.to(torch.float64).contiguous()
    d3 = d if d.ndim == 3 else d[None]
    B, N = d3.shape[0], d3.shape[1]
    out = torch.empty_like(d3)
    status = torch.zeros(1, dtype=torch.int64, device=d3.device)
    _lib.check(fn(d3.data_ptr(), arg, N, B, out.data_ptr(), status.data_ptr(), dev.current_stream_ptr(d3.device)), what)
    _raise_item(status, what)
    out = out if d.ndim == 3 else out[0]
    if x.dtype == torch.float32:
        out = out.to(torch.float32)
    return dev.like_input(out, L)


def _as_input(L):
    if dev.is_tensor(L):
        import torch
        if L.dtype not in (torch.float32, torch.float64):
            raise TypeError("expected a float32 or float64 tensor, got %s" % L.dtype)
        return L
    return np.asarray(L)


def cholesky_inv(L, lower=False):
    """Inverse of the symmetric positive definite matrix whose Cholesky factor is ``L``, in full storage.

    ``lower=True``: ``L`` is lower triangular and the result is ``(L L^T)^-1``; ``lower=False``: ``L`` is
    upper triangular and the result is ``(L^T L)^-1``.  Only that triangle of ``L`` is read.  A NumPy
    ``L`` must be float64, as in the reference."""
    L = _as_input(L)
    _check_square(L)
    if not dev.is_tensor(L) and L.dtype != np.float64:
        raise AssertionError("cholesky_inv: a NumPy factor must be float64, got %s" % L.dtype)
    return _invert(L, _lib.lib.nnk_cholesky_inv, int(bool(lower)), "cholesky_inv")


def cholesky_inv_banded(L, width=3):
    """``(L L^T)^-1`` in full storage from the band ``L[t, t-j]``, ``0 <= j < width``, of the lower
    Cholesky factor ``L`` (entries outside the band are not read).  A NumPy ``L`` is computed in float64
    and the result is float64, as in the reference."""
    L = _as_input(L)
    _check_square(L)
    if int(width) != width or width < 1:
        raise ValueError("width must be an integer >= 1, got %r" % (width,))
    if not dev.is_tensor(L) and L.dtype != np.float64:
        L = L.astype(np.float64)
    return _invert(L, _lib.lib.nnk_cholesky_inv_banded, int(width), "cholesky_inv_banded")


__all__ = ["cholesky_inv", "cholesky_inv_banded"]
