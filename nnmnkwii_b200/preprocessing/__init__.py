"""Pre-processing pieces on the DTW hot path (drop-in for the names the aligners need from
``nnmnkwii.preprocessing``) and corpus normalisation (``normalize``: meanvar / meanstd / minmax and the
scale family)."""
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


def delta_features(x, windows, lengths=None):
    """Compute delta features and combine them (nnmnkwii/preprocessing/generic.py:229-288).

    ``x`` is ``(T, D)`` static features (NumPy array or torch CUDA tensor); ``windows`` is a list of
    ``(l, u, coeff)`` triples (only ``coeff`` is used, as in the reference) or of plain coefficient
    arrays.  Returns ``(T, D * len(windows))`` in the dtype of ``x``.  Additive: with ``lengths`` the
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
    is_t = type(x).__module__.startswith("torch")
    lens = np.asarray([T] if lengths is None else lengths, dtype=np.int64)
    assert int(lens.sum()) == T
    for c in coefs:
        if len(lens) and int(lens.min()) < len(c):
            raise ValueError("delta window longer than the utterance (np.correlate 'same' would change the length)")
    wc = _lib.make_windows([((len(c) - 1) // 2, len(c) - 1 - (len(c) - 1) // 2, c) for c in coefs])
    if is_t:
        xd = x if x.dtype in (torch.float32, torch.float64) else x.to(torch.float64)
    else:
        xn = np.ascontiguousarray(x)
        xd = torch.from_numpy(xn if xn.dtype in (np.float32, np.float64) else xn.astype(np.float64)).cuda()
    xd = xd.contiguous()
    device = xd.device
    out = torch.empty((T, D * len(coefs)), dtype=xd.dtype, device=device)
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)).to(device)
    if T and D:
        _lib.check(_lib.lib.nnk_delta_features(xd.data_ptr(), dev.torch_dtype_code(xd.dtype), D, D, off.data_ptr(), None, len(lens),
                                               int(lens.max()), ctypes.byref(wc), out.data_ptr(), D * len(coefs),
                                               dev.current_stream_ptr(device)), "nnk_delta_features")
    if is_t:
        return out if out.dtype == x.dtype else out.to(x.dtype)
    res = out.cpu().numpy()
    return res if res.dtype == x.dtype else res.astype(x.dtype)


from .normalize import (inv_minmax_scale, inv_scale, meanstd, meanvar, minmax, minmax_scale,  # noqa: E402
                        minmax_scale_params, remove_zeros_frames, scale)

__all__ = ["trim_zeros_frames", "delta_features", "meanvar", "meanstd", "minmax", "scale", "inv_scale",
           "minmax_scale_params", "minmax_scale", "inv_minmax_scale", "remove_zeros_frames"]
