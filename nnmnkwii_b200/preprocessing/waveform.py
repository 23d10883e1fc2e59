"""Pre-emphasis and mu-law companding -- drop-in for ``nnmnkwii.preprocessing.preemphasis``,
``inv_preemphasis``, ``mulaw``, ``inv_mulaw``, ``mulaw_quantize`` and ``inv_mulaw_quantize``
(nnmnkwii/preprocessing/generic.py:56-226).

``preemphasis`` / ``inv_preemphasis`` (C ABI ``nnk_preemphasis``, csrc/nnk_wave.cu) filter along the last
axis in the input dtype, bit-identically to ``scipy.signal.lfilter`` (NaN payloads aside: the GPU
returns its canonical NaN).  The inverse, a first-order IIR filter, runs in parallel chunks that start
from a float64 estimate of the state and are repaired until they equal the sequential filter bitwise
(DESIGN.md 3.13).  The mu-law functions are one elementwise kernel (``nnk_mulaw``) in the reference's
promotion chain: NumPy in gives NumPy out of the reference's dtype, a tensor gives a tensor, a scalar a
NumPy or Python scalar, as the reference's ``_sign`` / ``_log1p`` / ``_asint`` / ``_asfloat`` do.

Deliberate differences from the reference: ``mulaw``, ``inv_mulaw`` and ``mulaw_quantize`` take floating
inputs only (float32 / float64 arrays and tensors, Python and NumPy scalars); ``log1p`` and ``pow`` are
evaluated on the GPU, so their last bit may differ from the host's libm.
"""
import numbers

import numpy as np

_last_counters = None


def _filter(x, coef, lengths, inverse):
    global _last_counters
    from .. import _device as dev
    from .._lib import check, lib
    dt = dev.np_dtype(x)
    if dt not in (np.float32, np.float64):
        # what scipy.signal.lfilter raises for the reference's coefficient arrays of this dtype
        if inverse:
            raise NotImplementedError("input type '%s' not supported\n" % dt)
        raise NotImplementedError("Parameter's dtypes produced result type '%s', which is not supported!" % dt)
    shape = tuple(int(s) for s in x.shape)
    if len(shape) == 0:
        raise ValueError("x must have at least one dimension")
    lens = None
    if lengths is not None:
        if len(shape) != 2:
            raise ValueError("lengths requires a 2-D (B, T) x, got %d-D" % len(shape))
        lens = dev.check_lengths(lengths, shape[0])
    coef = float(coef)
    dev.require_cuda()
    import torch
    xt = dev.to_device(x).contiguous()
    T = shape[-1]
    rows = xt.numel() // T if T else 0
    out = torch.empty_like(xt)
    if rows and T:
        lt = dev.lengths_on(lens, xt.device, T)
        code = dev.torch_dtype_code(xt.dtype)
        ws = dev.workspace(xt.device, int(lib.nnk_preemphasis_workspace_bytes(code, rows, T, coef, int(inverse))))
        counters = torch.empty(2, dtype=torch.int64, device=xt.device)
        check(lib.nnk_preemphasis(xt.data_ptr(), out.data_ptr(), code, rows, T,
                                  lt.data_ptr() if lt is not None else None, coef, int(inverse), ws.data_ptr(),
                                  ws.numel(), counters.data_ptr(), dev.current_stream_ptr(xt.device)),
              "nnk_preemphasis")
        if inverse:
            _last_counters = counters
    return dev.like_input(out, x)


def _repair_counters():
    """(chunks rerun, samples rewritten) by the repair walk of the last ``inv_preemphasis`` call.  Reads
    a two-word device buffer, so it synchronises; the filter itself never does."""
    if _last_counters is None:
        return 0, 0
    c = _last_counters.cpu().numpy()
    return int(c[0]), int(c[1])


def preemphasis(x, coef=0.97, lengths=None):
    """Pre-emphasis ``y[t] = x[t] - coef * x[t - 1]`` along the last axis (preprocessing/generic.py:182).

    Args:
        x: float32 / float64 signal(s), any shape (NumPy array or tensor).
        coef (float): pre-emphasis coefficient, rounded to ``x.dtype``.
        lengths: with a 2-D ``(B, T)`` ``x``, samples of each row (additive); later samples are copied.
    """
    return _filter(x, coef, lengths, False)


def inv_preemphasis(x, coef=0.97, lengths=None):
    """Inverse of pre-emphasis, ``y[t] = x[t] + coef * y[t - 1]`` along the last axis
    (preprocessing/generic.py:205), bit-identical to the sequential filter in ``x.dtype``."""
    return _filter(x, coef, lengths, True)


# ---- mu-law ---------------------------------------------------------------------------------------------
_INT_CODES = {np.dtype(np.int32): 2, np.dtype(np.int64): 3}


def _mulaw_call(x, mu, mode):
    """Run nnk_mulaw on x (array, tensor or scalar) with the reference's dtype chain of ``mode``."""
    import torch

    from .. import _device as dev
    from .._lib import NNK_F32, NNK_F64, check, lib
    mu = float(mu) if not isinstance(mu, numbers.Integral) else int(mu)
    is_t = dev.is_tensor(x)
    scalar = not is_t and np.isscalar(x)
    if not is_t and not scalar and not isinstance(x, np.ndarray):
        raise TypeError("expected a NumPy array, a scalar or a torch tensor, got %s" % type(x).__name__)
    if scalar and not isinstance(x, (numbers.Number, np.generic)):
        raise TypeError("expected a numeric scalar, got %s" % type(x).__name__)
    dt = dev.np_dtype(x) if not scalar else None
    if mode == 3:
        if is_t:
            if x.dtype == torch.bool or x.is_complex():
                raise TypeError("inv_mulaw_quantize: unsupported tensor dtype %s" % x.dtype)
            src = x if x.dtype in (torch.float32, torch.float64, torch.int32, torch.int64) else x.to(torch.int64)
            variant = 1
        elif scalar:
            src, variant = np.array([float(x)], np.float64), 2  # float(y), as the reference's _asfloat
        else:
            if dt.kind not in "iuf" or dt == np.uint64:
                raise TypeError("inv_mulaw_quantize: unsupported dtype %s" % dt)
            src = x if dt in (np.float32, np.float64) or dt in _INT_CODES else x.astype(np.int64)
            variant = 1
        out_np = np.float32 if variant == 1 else np.float64
    else:
        if scalar:
            if isinstance(x, np.floating) and x.dtype == np.float32:
                src, variant = np.array([x], np.float32), 0 if mode != 1 else 1
            elif isinstance(x, (bool, np.bool_)) or not isinstance(x, (numbers.Real, np.floating, np.integer)):
                raise TypeError("mu-law: unsupported scalar %r" % (x,))
            else:
                src, variant = np.array([float(x)], np.float64), 2
        else:
            if dt not in (np.float32, np.float64):
                raise TypeError("mu-law: x must be float32 or float64, got %s" % dt)
            src = x
            variant = 2 if dt == np.float64 else (1 if (is_t or mode == 1) else 0)
        if mode == 2:
            out_np = np.int64
        elif mode == 1:
            out_np = np.float32 if variant == 1 else np.float64
        else:
            out_np = np.float64 if variant in (0, 2) else np.float32
    dev.require_cuda()
    xt = dev.to_device(src).contiguous()
    code = {torch.float32: NNK_F32, torch.float64: NNK_F64, torch.int32: 2, torch.int64: 3}[xt.dtype]
    out = torch.empty(xt.shape, dtype=getattr(torch, np.dtype(out_np).name), device=xt.device)
    if xt.numel():
        check(lib.nnk_mulaw(xt.data_ptr(), code, out.data_ptr(), mode, variant, xt.numel(), float(mu),
                            dev.current_stream_ptr(xt.device)), "nnk_mulaw")
    res = dev.like_input(out, x)
    if scalar:
        v = res[0]
        return int(v) if mode == 2 else v
    return res


def mulaw(x, mu=256):
    """Mu-law companding ``sign(x) log(1 + mu |x|) / log(1 + mu)`` (preprocessing/generic.py:56)."""
    return _mulaw_call(x, mu, 0)


def inv_mulaw(y, mu=256):
    """Mu-law expansion ``sign(y) (1 / mu) ((1 + mu)^|y| - 1)`` (preprocessing/generic.py:86)."""
    return _mulaw_call(y, mu, 1)


def mulaw_quantize(x, mu=256):
    """Mu-law companding and quantisation to ``int((y + 1) / 2 * mu)`` (preprocessing/generic.py:108)."""
    return _mulaw_call(x, mu, 2)


def inv_mulaw_quantize(y, mu=256):
    """Inverse of ``mulaw_quantize``: ``inv_mulaw(2 float32(y) / mu - 1)`` (preprocessing/generic.py:148)."""
    return _mulaw_call(y, mu, 3)


__all__ = ["preemphasis", "inv_preemphasis", "mulaw", "inv_mulaw", "mulaw_quantize", "inv_mulaw_quantize"]
