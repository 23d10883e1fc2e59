"""Pre-processing pieces on the DTW hot path (drop-in for the names the aligners need from
``nnmnkwii.preprocessing``), corpus normalisation (``normalize``: meanvar / meanstd / minmax and the
scale family), F0 interpolation (``f0``), pre-emphasis and mu-law (``waveform``) and the frame-length
helpers; the modulation spectrum (``modspec``: modspec / modphase / inv_modspec / modspec_smoothing)."""
import numpy as np


def trim_zeros_frames(x, eps=1e-7, trim="b"):
    """Remove leading and/or trailing zeros frames (nnmnkwii/preprocessing/generic.py:291-332).

    Host-side utility with the reference's exact semantics; the aligners compute the same trailing
    lengths on the device (C ABI ``nnk_trim_lengths``) without touching the host.
    """
    assert trim in {"f", "b", "fb"}
    live = np.flatnonzero(np.sum(np.abs(x), axis=1) >= eps)  # frames that are not (numerically) zero
    if live.size == 0:
        return x[:0] if len(x) else x
    first = live[0] if "f" in trim else 0
    last = live[-1] + 1 if "b" in trim else len(x)
    return x if (first == 0 and last == len(x)) else x[first:last]


def _pad_end(x, n, kwargs):
    return np.pad(x, (0, n) if x.ndim == 1 else [(0, n), (0, 0)], **kwargs)


def adjust_frame_length(x, pad=True, divisible_by=1, **kwargs):
    """Pad (``pad=True``) or trim the end of a ``(T,)`` or ``(T, D)`` array so that its length is divisible
    by ``divisible_by`` (nnmnkwii/preprocessing/generic.py:359-414).  ``kwargs`` go to :func:`numpy.pad`
    (default ``mode="constant"``).  Host-side, NumPy only, the reference's semantics."""
    kwargs.setdefault("mode", "constant")
    assert x.ndim == 2 or x.ndim == 1
    Tx = x.shape[0]
    T = Tx
    if divisible_by > 1 and Tx % divisible_by:
        T = Tx + divisible_by - Tx % divisible_by if pad else Tx - Tx % divisible_by
    if T > Tx:
        return _pad_end(x, T - Tx, kwargs)
    return x[:T] if T < Tx else x


def adjust_frame_lengths(x, y, pad=True, ensure_even=False, divisible_by=1, **kwargs):
    """Give two ``(T, D)`` (or ``(T,)``) arrays the same length, divisible by ``divisible_by``, by padding
    both to the longer (``pad=True``) or trimming both to the shorter (nnmnkwii/preprocessing/generic.py:
    417-493).  ``ensure_even`` (deprecated) means ``divisible_by=2``.  Host-side, NumPy only."""
    assert x.ndim in [1, 2] and y.ndim in [1, 2]
    kwargs.setdefault("mode", "constant")
    Tx, Ty = x.shape[0], y.shape[0]
    if x.ndim == 2:
        assert x.shape[-1] == y.shape[-1]
    if ensure_even:
        divisible_by = 2
    if pad:
        T = max(Tx, Ty)
        if divisible_by > 1 and T % divisible_by:
            T += divisible_by - T % divisible_by
    else:
        T = min(Tx, Ty)
        if divisible_by > 1:
            T -= T % divisible_by
    x = _pad_end(x, T - Tx, kwargs) if Tx < T else x[:T] if Tx > T else x
    y = _pad_end(y, T - Ty, kwargs) if Ty < T else y[:T] if Ty > T else y
    return x, y


adjast_frame_length = adjust_frame_length  # deprecated spellings, kept by the reference
adjast_frame_lengths = adjust_frame_lengths


def delta_features(x, windows, lengths=None):
    """Compute delta features and combine them (nnmnkwii/preprocessing/generic.py:229-288).

    ``x`` is ``(T, D)`` static features (NumPy array or torch tensor); ``windows`` is a list of
    ``(l, u, coeff)`` triples (only ``coeff`` is used, as in the reference) or of plain coefficient
    arrays.  Returns ``(T, D * len(windows))`` in the dtype and form of ``x`` (a CPU tensor is computed on
    the GPU and comes back as a CPU tensor).  Additive: with ``lengths`` the
    rows of ``x`` are several utterances back to back and the deltas do not cross their boundaries.
    Runs on the GPU (C ABI ``nnk_delta_features``, csrc/nnk_delta.cu).
    """
    import ctypes

    import torch

    from .. import _device as dev
    from .. import _lib

    dev.require_cuda()
    assert len(windows) > 0
    coefs = [np.asarray(w[2] if isinstance(w, tuple) else w, dtype=np.float64).ravel() for w in windows]
    T, D = x.shape
    lens = np.asarray([T] if lengths is None else lengths, dtype=np.int64)
    assert int(lens.sum()) == T
    for c in coefs:
        if len(lens) and int(lens.min()) < len(c):
            raise ValueError("delta window longer than the utterance (np.correlate 'same' would change the length)")
    wc = _lib.make_windows([((len(c) - 1) // 2, len(c) - 1 - (len(c) - 1) // 2, c) for c in coefs])
    xd = dev.to_device(x)
    xd = (xd if xd.dtype in (torch.float32, torch.float64) else xd.to(torch.float64)).contiguous()
    device = xd.device
    out = torch.empty((T, D * len(coefs)), dtype=xd.dtype, device=device)
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)).to(device)
    if T and D:
        _lib.check(_lib.lib.nnk_delta_features(xd.data_ptr(), dev.torch_dtype_code(xd.dtype), D, D, off.data_ptr(), None, len(lens),
                                               int(lens.max()), ctypes.byref(wc), out.data_ptr(), D * len(coefs),
                                               dev.current_stream_ptr(device)), "nnk_delta_features")
    res = dev.like_input(out, x)
    if res.dtype == x.dtype:
        return res
    return res.to(x.dtype) if dev.is_tensor(x) else res.astype(x.dtype)


from .normalize import (inv_minmax_scale, inv_scale, meanstd, meanvar, minmax, minmax_scale,  # noqa: E402
                        minmax_scale_params, remove_zeros_frames, scale)
from .f0 import interp1d  # noqa: E402
from .waveform import (inv_mulaw, inv_mulaw_quantize, inv_preemphasis, mulaw, mulaw_quantize,  # noqa: E402
                       preemphasis)
from .modspec import inv_modspec, modphase, modspec, modspec_smoothing  # noqa: E402,F401

__all__ = ["trim_zeros_frames", "delta_features", "meanvar", "meanstd", "minmax", "scale", "inv_scale",
           "minmax_scale_params", "minmax_scale", "inv_minmax_scale", "remove_zeros_frames", "interp1d",
           "preemphasis", "inv_preemphasis", "mulaw", "inv_mulaw", "mulaw_quantize", "inv_mulaw_quantize",
           "adjust_frame_length", "adjust_frame_lengths", "adjast_frame_length", "adjast_frame_lengths", "modspec",
           "modphase", "inv_modspec", "modspec_smoothing"]
