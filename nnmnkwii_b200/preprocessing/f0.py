"""Continuous F0 interpolation -- drop-in for ``nnmnkwii.preprocessing.interp1d``
(nnmnkwii/preprocessing/f0.py).

One CTA per row (C ABI ``nnk_f0_interp``, csrc/nnk_wave.cu) finds the previous and next voiced frame of
every frame with block scans and evaluates the kind in float64 with the operation order of the scipy
routine the reference reaches, so the result is bit-identical to scipy's.

Deliberate differences from the reference:
  * only the two-point kinds are supported (``linear``, ``slinear`` = 1, ``zero`` = 0, ``nearest``,
    ``nearest-up``, ``previous``, ``next``); ``quadratic``, ``cubic`` and integer orders >= 2 raise
    ``ValueError``;
  * ``f0`` must be float32 or float64 (``TypeError`` otherwise);
  * with ``lengths``, a row of length 1 is returned unchanged whatever the kind.
"""
import numpy as np

KINDS = {"linear": 0, "slinear": 1, "zero": 2, "nearest": 3, "nearest-up": 4, "previous": 5, "next": 6}
_SPLINE = ("zero", "slinear", "quadratic", "cubic")


def _kind_code(kind):
    if isinstance(kind, (int, np.integer)) and not isinstance(kind, bool):
        if int(kind) in (0, 1):
            return KINDS["zero" if int(kind) == 0 else "slinear"], True
        raise ValueError("interp1d: spline order %d is not supported; supported kinds: %s, 0, 1"
                         % (int(kind), ", ".join(KINDS)))
    if kind in ("quadratic", "cubic"):
        raise ValueError("interp1d: kind %r is not supported; supported kinds: %s, 0, 1" % (kind, ", ".join(KINDS)))
    if kind not in KINDS:
        raise NotImplementedError("%s is unsupported: Use fitpack routines for other types." % (kind,))
    return KINDS[kind], kind in _SPLINE


def _launch(xt, B, T, lens, code):
    import torch

    from .. import _device as dev
    from .._lib import check, lib
    out = torch.empty_like(xt)
    ws = dev.workspace(xt.device, int(lib.nnk_f0_interp_workspace_bytes(B, T)))
    lt = dev.lengths_on(lens, xt.device, T)
    check(lib.nnk_f0_interp(xt.data_ptr(), out.data_ptr(), dev.torch_dtype_code(xt.dtype), B, T,
                            lt.data_ptr() if lt is not None else None, code, ws.data_ptr(), ws.numel(),
                            dev.current_stream_ptr(xt.device)), "nnk_f0_interp")
    return out


def interp1d(f0, kind="slinear", lengths=None):
    """Continuous F0 interpolation of a discontinuous F0 trajectory (preprocessing/f0.py).

    Values ``> 0`` are voiced; zero and negative frames are filled (NaN frames, as in the reference, are
    neither voiced nor filled).  Frames 0 and T - 1 first take the first and last voiced values.

    Args:
        f0: ``(T,)`` or ``(T, 1)`` F0 or log-F0 (NumPy array or CUDA tensor, float32 / float64); with
            ``lengths``, a padded ``(B, Tmax)`` or ``(B, Tmax, 1)`` batch.
        kind (str or int): a two-point kind of :class:`scipy.interpolate.interp1d`.
        lengths: frames of each row (additive); frames at or beyond ``lengths[b]`` are copied.

    Returns:
        The interpolated trajectory, of ``f0``'s shape and dtype (NumPy in, NumPy out; a CUDA tensor in,
        a new CUDA tensor out).  For a single NumPy trajectory without a voiced frame, ``f0`` itself.
    """
    from .. import _device as dev
    code, spline = _kind_code(kind)
    shape = tuple(int(s) for s in f0.shape)
    dt = dev.np_dtype(f0)
    if dt not in (np.float32, np.float64):
        raise TypeError("interp1d: f0 must be float32 or float64, got %s" % dt)
    if lengths is None:
        if len(shape) == 0 or shape[0] != int(np.prod(shape)):
            raise RuntimeError("1d array is only supported")
        B, T, lens = 1, shape[0], None
    else:
        if len(shape) not in (2, 3) or (len(shape) == 3 and shape[2] != 1):
            raise ValueError("interp1d: with lengths, f0 must be (B, Tmax) or (B, Tmax, 1), got %s" % (shape,))
        B, T = shape[0], shape[1]
        lens = dev.check_lengths(lengths, B)
    dev.require_cuda()
    xt = dev.to_device(f0).contiguous()
    if lengths is None and spline and T == 1 and code == KINDS["slinear"] and bool((xt > 0).any()):
        raise ValueError("x and y arrays must have at least 2 entries")
    out = _launch(xt, B, T, lens, code) if B and T else xt.clone()
    res = dev.like_input(out, f0)
    if dev.is_tensor(f0):
        return res
    if lengths is None and not (res.reshape(-1) > 0).any():
        return f0  # nothing to do: the reference returns its input object
    if lengths is None:
        return res.reshape(-1)[:, None] if len(shape) == 2 else res.reshape(-1)
    return res


__all__ = ["interp1d"]
