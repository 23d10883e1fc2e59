"""Drop-in for ``nnmnkwii.util`` (nnmnkwii/util/__init__.py): the re-exported pre-processing names, the
per-slice helpers ``apply_each2d_trim`` / ``apply_each2d_padded`` and ``util.linalg``.

``func2d`` is an arbitrary callable, so the loop over slices stays on the host.  For a CUDA tensor ``X``
the slices, and the output, stay on the device: ``apply_each2d_trim`` takes every slice's trailing
length from one ``nnk_trim_lengths`` launch and one copy of ``N`` integers to the host (not ``N`` host
trims), and the output is a CUDA tensor in the dtype ``func2d`` returns.  Other input follows the
reference exactly: the output is a float64 NumPy array.

Deliberate difference: the reference calls ``func2d`` on slice 0 twice (once to learn the output width);
this port calls it once per slice.  ``util.files`` (the reference's example-data accessors, which need
its package data) is not ported.
"""
import numpy as np

from ..preprocessing import (adjust_frame_length, delta_features, meanstd, meanvar, minmax,  # noqa: F401
                             minmax_scale, remove_zeros_frames, scale, trim_zeros_frames)
from . import linalg  # noqa: F401

apply_delta_windows = delta_features


def _on_cuda(X):
    from .. import _device as dev
    return dev.is_tensor(X) and X.is_cuda


def _device_trim_lengths(X):
    """``len(trim_zeros_frames(X[i]))`` of every slice of a 3-D CUDA tensor, as host integers."""
    import torch

    from .. import _device as dev
    from .. import _lib

    N, T, D = X.shape
    Xd = X.detach().contiguous()
    lens = torch.zeros(N, dtype=torch.int32, device=Xd.device)
    if N and T and D:
        _lib.check(_lib.lib.nnk_trim_lengths(Xd.data_ptr(), dev.torch_dtype_code(Xd.dtype), T * D, D, T, D, 1e-7, N,
                                             lens.data_ptr(), dev.current_stream_ptr(Xd.device)), "nnk_trim_lengths")
    return lens.cpu().numpy()


def _apply_each(func2d, X, lens, args, kwargs):
    """``Y[i, :len(y_i)] = y_i`` with ``y_i = func2d(X[i][:lens[i]], ...)`` over a zero ``(N, T, D')`` output
    (float64 NumPy, or for a CUDA ``X`` a CUDA tensor of the dtype ``func2d`` returns)."""
    N, T = X.shape[0], X.shape[1]
    Y = None
    for idx in range(N):
        y = func2d(X[idx][: lens[idx]], *args, **kwargs)
        assert y.ndim == 2
        if Y is None:
            if _on_cuda(X):
                import torch
                Y = torch.zeros((N, T, y.shape[1]), dtype=y.dtype, device=y.device)
            else:
                Y = np.zeros((N, T, y.shape[1]))
        Y[idx][: len(y)] = y
    if Y is None:  # the reference needs slice 0 to exist too
        raise IndexError("apply_each2d: X has no slices")
    return Y


def apply_each2d_trim(func2d, X, *args, **kwargs):
    """Apply ``func2d`` to each ``(T, D)`` slice of ``X`` (``N x T x D``) with its trailing zero frames
    trimmed (``trim_zeros_frames``); returns ``N x T x D'`` with slice ``i`` in its first ``len(y_i)``
    rows and zeros after."""
    assert X.ndim == 3
    if _on_cuda(X):
        lens = _device_trim_lengths(X)
    else:
        lens = [len(trim_zeros_frames(X[idx])) for idx in range(X.shape[0])]
    return _apply_each(func2d, X, lens, args, kwargs)


def apply_each2d_padded(func2d, X, lengths, *args, **kwargs):
    """Apply ``func2d`` to ``X[i][:lengths[i]]`` for each slice of ``X`` (``N x T x D``); returns
    ``N x T x D'`` with slice ``i`` in its first ``len(y_i)`` rows and zeros after."""
    assert X.ndim == 3
    if _on_cuda(X) and hasattr(lengths, "is_cuda") and lengths.is_cuda:
        lengths = lengths.cpu()  # one copy instead of one per slice
    return _apply_each(func2d, X, lengths, args, kwargs)


__all__ = ["adjust_frame_length", "delta_features", "apply_delta_windows", "meanstd", "meanvar", "minmax",
           "minmax_scale", "remove_zeros_frames", "scale", "trim_zeros_frames", "apply_each2d_trim",
           "apply_each2d_padded", "linalg"]
