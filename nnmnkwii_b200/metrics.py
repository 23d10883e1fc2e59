"""Objective metrics -- drop-in for ``nnmnkwii.metrics`` (nnmnkwii/metrics/__init__.py).

``melcd``, ``mean_squared_error``, ``lf0_mean_squared_error`` and ``vuv_error`` keep the reference's
signatures, accepted shapes and scalar finish; the reductions themselves (including the
``lengths``-masked mini-batch forms, which the reference evaluates with a Python loop over the
batch) run as one sm_90a kernel launch each (csrc/nnk_metrics.cu, SURVEY.md section 8f row 4).
NumPy arrays and CPU tensors are copied to the current CUDA device first; there is no CPU path.

As the DTW *local cost* (``DTWAligner(dist=melcd)``) ``melcd`` is never called per cell: the aligner
recognises it and the wavefront kernel evaluates ``10/ln10 * sqrt(2) * ||x - y||_2`` in registers
(csrc/nnk_dtw.cu).
"""
import ctypes
import math

import numpy as np

_logdb_const = 10.0 / np.log(10.0) * np.sqrt(2.0)  # metrics/__init__.py:5
_ws_cache = {}


def _prepare(arrays):
    """Move to one device, promote to a common float dtype, make contiguous."""
    import torch

    from . import _device as dev
    dev.require_cuda()
    device = None
    for a in arrays:
        if isinstance(a, torch.Tensor) and a.is_cuda:
            device = a.device
            break
    ts = [dev.to_device(a, device) for a in arrays]
    dt = torch.float32 if all(t.dtype == torch.float32 for t in ts) else torch.float64
    return [t.to(dt).contiguous() for t in ts], ts[0].device, dt


def _lengths_on(device, lengths, B):
    import torch
    if lengths is None:
        return None
    if isinstance(lengths, torch.Tensor):
        l = lengths.to(device=device, dtype=torch.int32)
    else:
        l = torch.as_tensor(np.asarray(lengths, dtype=np.int64).astype(np.int32), device=device)
    return l.contiguous()  # the reference zips (X, Y, lengths): the shorter of the two bounds the loop


def _reduce(call, device, B, T):
    """Run one of the C-ABI reductions; returns (sum, count) as Python numbers (synchronises)."""
    import torch

    from . import _device as dev
    from ._lib import check, lib
    need = int(lib.nnk_metric_workspace_bytes(max(1, B), max(1, T)))
    # one ticketed partial buffer per (device, stream): reductions on different streams never share it
    key = (str(device), torch.cuda.current_stream(device).cuda_stream)
    ws = _ws_cache.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.zeros(need, dtype=torch.uint8, device=device)  # zeroed once; every call leaves it reusable
        if len(_ws_cache) > 32:
            _ws_cache.clear()
        _ws_cache[key] = ws
    res = torch.zeros(2, dtype=torch.float64, device=device)  # [sum, count (int64 bits)]
    rc = call(ctypes.c_void_p(res.data_ptr()), ctypes.c_void_p(res.data_ptr() + 8),
              ctypes.c_void_p(ws.data_ptr()), ctypes.c_int64(ws.numel()), dev.current_stream_ptr(device))
    check(rc, "nnk metric")
    s = float(res[0].item())
    c = int(res[1:2].view(torch.int64).item())
    return s, c


def _frame_metric(X, Y, B, T, D, lengths, kind):
    from . import _device as dev
    from ._lib import lib
    (x, y), device, dt = _prepare([X, Y])
    assert x.numel() == y.numel() == B * T * D
    l = _lengths_on(device, lengths, B)
    nb = B if l is None else min(B, int(l.numel()))
    code = dev.torch_dtype_code(dt)

    def call(sum_p, cnt_p, ws_p, ws_n, stream):
        return lib.nnk_frame_metric(x.data_ptr(), y.data_ptr(), code, nb, T, D, T * D, D,
                                    l.data_ptr() if l is not None else None, kind, sum_p, cnt_p, ws_p, ws_n, stream)
    return _reduce(call, device, nb, T)


def _f0_metric(arrays, B, T, lengths, kind):
    from . import _device as dev
    from ._lib import lib
    ts, device, dt = _prepare(arrays)
    for t in ts:
        assert t.numel() == B * T
    l = _lengths_on(device, lengths, B)
    nb = B if l is None else min(B, int(l.numel()))
    code = dev.torch_dtype_code(dt)
    if kind == 2:
        xv, yv = ts
        xf = yf = None
    else:
        xf, xv, yf, yv = ts

    def call(sum_p, cnt_p, ws_p, ws_n, stream):
        return lib.nnk_f0_metric(xf.data_ptr() if xf is not None else None, xv.data_ptr(),
                                 yf.data_ptr() if yf is not None else None, yv.data_ptr(), code, nb, T, T, 1,
                                 l.data_ptr() if l is not None else None, kind, sum_p, cnt_p, ws_p, ws_n, stream)
    return _reduce(call, device, nb, T)


def _numel(shape):
    n = 1
    for s in shape:
        n *= int(s)
    return n


def melcd(X, Y, lengths=None):
    """Mel-cepstrum distortion (MCD) in dB (metrics/__init__.py:27-71).

    Args:
        X, Y: shape ``(D,)``, ``(T, D)`` or ``(B, T, D)``; NumPy arrays or torch tensors.
        lengths (list): lengths of padded inputs (mini-batch case).

    Returns:
        float: mean mel-cepstrum distortion in dB.
    """
    shape = tuple(X.shape)
    if lengths is None:
        D = int(shape[-1]) if len(shape) else 1
        frames = _numel(shape[:-1])
        s, c = _frame_metric(X, Y, 1, frames, D, None, 0)
        return _logdb_const * (s / c if c else float("nan"))
    if len(shape) == 2:  # (B, T) -> (B, T, 1)  (:62-63)
        shape = shape + (1,)
    B, T = int(shape[0]), int(shape[1])
    s, _ = _frame_metric(X, Y, B, T, _numel(shape[2:]), lengths, 0)
    return _logdb_const * float(s) / float(_sum_lengths(lengths))


def mean_squared_error(X, Y, lengths=None):
    """Root of the mean squared error, as in the reference (metrics/__init__.py:74-110).

    Args:
        X, Y: ``(D,)``, ``(T, D)`` or ``(B, T, D)``; NumPy arrays or torch tensors.
        lengths (list): lengths of padded inputs (mini-batch case).
    """
    shape = tuple(X.shape)
    if lengths is None:
        n = _numel(shape)
        s, _ = _frame_metric(X, Y, 1, n, 1, None, 1)
        return math.sqrt(s / n) if n else float("nan")
    B, T = int(shape[0]), int(shape[1])
    denom = _sum_lengths(lengths) * int(shape[-1])  # (:103) -- X.shape[-1] even for 2-D inputs
    s, _ = _frame_metric(X, Y, B, T, _numel(shape[2:]), lengths, 1)
    return math.sqrt(float(s) / float(denom))


def lf0_mean_squared_error(src_f0, src_vuv, tgt_f0, tgt_vuv, lengths=None, linear_domain=False):
    """MSE of log-F0 over frames voiced in both sequences (metrics/__init__.py:113-165).

    Shapes ``(T,)``, ``(B, T)`` or ``(B, T, 1)``; ``linear_domain`` exponentiates first.
    """
    shape = tuple(src_f0.shape)
    kind = 1 if linear_domain else 0
    if lengths is None:
        n = _numel(shape)
        s, c = _f0_metric([src_f0, src_vuv, tgt_f0, tgt_vuv], 1, n, None, kind)
        return math.sqrt(s / c) if c else float("nan")
    B, T = int(shape[0]), int(shape[1])
    assert _numel(shape[2:]) == 1
    s, c = _f0_metric([src_f0, src_vuv, tgt_f0, tgt_vuv], B, T, lengths, kind)
    return math.sqrt(float(s) / float(c))


def vuv_error(src_vuv, tgt_vuv, lengths=None):
    """Voiced/unvoiced error rate in [0, 1] (metrics/__init__.py:168-190)."""
    shape = tuple(src_vuv.shape)
    if lengths is None:
        n = _numel(shape)
        s, _ = _f0_metric([src_vuv, tgt_vuv], 1, n, None, 2)
        return float(s) / float(n)
    B, T = int(shape[0]), int(shape[1])
    assert _numel(shape[2:]) == 1
    s, _ = _f0_metric([src_vuv, tgt_vuv], B, T, lengths, 2)
    return float(s) / float(_sum_lengths(lengths))


def _sum_lengths(lengths):
    import torch
    if isinstance(lengths, torch.Tensor):
        return float(lengths.sum())
    return float(np.sum(lengths))


__all__ = ["melcd", "mean_squared_error", "lf0_mean_squared_error", "vuv_error"]
