"""Modulation spectrum (MS) -- drop-in for ``nnmnkwii.preprocessing.modspec``, ``modphase``, ``inv_modspec`` and
``modspec_smoothing`` (nnmnkwii/preprocessing/modspec.py).

Runs on the GPU (C ABI ``nnk_modspec``, include/nnk_b200.h, csrc/nnk_modspec.cu): one CTA per (utterance,
feature column) zero-pads the column to ``n`` frames and runs the real FFT in shared memory.  Smoothing runs the
forward FFT, the band removal and the inverse FFT in the same CTA, so the spectrum never reaches global memory;
the gradient of ``autograd.ModSpec`` is the same kernel in its gradient mode.

Every function takes a ``(T, D)`` array or a padded ``(B, T, D)`` batch with ``lengths`` (frames of each
utterance).  Frames past an utterance's length are never read, and are written as 0 where the result has
frames, so nothing depends on what the padding holds.  Inputs are float32 / float64 CUDA tensors (the result
stays on their device, in their dtype) or NumPy arrays (uploaded; the result comes back as NumPy).  The phase is
complex64 / complex128 to match.

Deliberate differences from the reference:
  * ``n`` is 256, 512, 1024, 2048 or 4096, and ``modspec`` requires ``T <= n`` (``numpy.fft.rfft`` would crop);
  * a CPU tensor is refused: pass a CUDA tensor, or a NumPy array for the reference's host-array interface;
  * bins are kept as computed rather than passed through the reference's ``sqrt(exp(log(|X|^2)))`` round
    trip, and the phase is ``X / |X|``: results agree with the reference to rounding.
"""
import numpy as np

NS = (256, 512, 1024, 2048, 4096)


def _check_n(n):
    if n not in NS:
        raise ValueError("n must be one of %s, got %r" % (", ".join(map(str, NS)), n))


def _scales(norm, n):
    """(forward, inverse) scale of ``numpy.fft``'s ``norm``."""
    if norm is None or norm == "backward":
        return 1.0, 1.0 / n
    if norm == "ortho":
        return 1.0 / np.sqrt(n), 1.0 / np.sqrt(n)
    if norm == "forward":
        return 1.0 / n, 1.0
    raise ValueError('Invalid norm value %r; should be "backward", "ortho" or "forward".' % (norm,))


def _checked(a, name, kinds=(np.float32, np.float64)):
    """Refuse what the kernels cannot take, before anything touches the device."""
    from .. import _device as dev
    if dev.is_tensor(a):
        if not a.is_cuda:
            raise ValueError("%s is a CPU tensor: pass a CUDA tensor, or a NumPy array" % name)
    elif not isinstance(a, np.ndarray):
        raise TypeError("%s must be a CUDA tensor or a NumPy array, got %s" % (name, type(a).__name__))
    if dev.np_dtype(a) not in kinds:
        raise TypeError("%s must be %s, got %s" % (name, " or ".join(np.dtype(k).name for k in kinds), dev.np_dtype(a)))
    return a


def _batch(x, lengths, name="x", most=None):
    """(B, T, D, host lengths or None, longest utterance) of a (T, D) or padded (B, T, D) input; ``lengths`` may
    not exceed ``most`` (default: T)."""
    from .. import _device as dev
    if x.ndim == 2:
        if lengths is not None:
            raise ValueError("lengths needs a padded (B, T, D) %s" % name)
        return 1, int(x.shape[0]), int(x.shape[1]), None, int(x.shape[0])
    if x.ndim != 3:
        raise ValueError("%s must be (T, D) or (B, T, D), got %d-D" % (name, x.ndim))
    B, T, D = (int(s) for s in x.shape)
    lens = dev.check_lengths(lengths, B)
    if lens is None:
        return B, T, D, None, T if B else 0
    longest = int(lens.max()) if lens.size else 0
    most = T if most is None else most
    if longest > most:
        raise ValueError("lengths exceed the %d frames of %s" % (most, name))
    return B, T, D, lens, longest


def _device_input(x, B, T, D):
    from .. import _device as dev
    dev.require_cuda()
    return dev.to_device(x).reshape(B, T, D).contiguous()


def _launch(mode, n, inp, in2, out, out2, B, T_in, T_out, D, lens, fwd_scale, inv_scale, limit_bin=0,
            log_domain=False):
    """Enqueue nnk_modspec on the current stream of ``out``'s device."""
    import torch

    from .. import _device as dev
    from .. import _lib
    if not (B and D):
        return
    lt = dev.lengths_on(lens, out.device)
    rv = (lambda t: torch.view_as_real(t) if t.is_complex() else t)
    _lib.check(_lib.lib.nnk_modspec(mode, dev.torch_dtype_code(out.dtype), n, inp.data_ptr(),
                                    rv(in2).data_ptr() if in2 is not None else None, out.data_ptr(),
                                    rv(out2).data_ptr() if out2 is not None else None, B, T_in, T_out, D,
                                    lt.data_ptr() if lt is not None else None, fwd_scale, inv_scale, limit_bin,
                                    int(bool(log_domain)), dev.current_stream_ptr(out.device)), "nnk_modspec")


def _complex_of(dtype):
    import torch
    return torch.complex64 if dtype == torch.float32 else torch.complex128


def _out(t, x, two_d):
    from .. import _device as dev
    return dev.like_input(t[0] if two_d else t, x)


def modspec(x, n=4096, norm=None, return_phase=False, lengths=None):
    """Modulation spectrum: power of the DFT of each feature trajectory along time, ``|rfft(x, n, axis=0)|^2``
    (preprocessing/modspec.py:6).

    Args:
        x: ``(T, D)`` trajectory, or a padded ``(B, T, D)`` batch.
        n (int): DFT length, 256 .. 4096 (a power of two), at least the number of frames.
        norm: ``None`` / ``"backward"``, ``"ortho"`` or ``"forward"``, as in :func:`numpy.fft.rfft`.
        return_phase (bool): also return the phase ``exp(1j angle(X))``.
        lengths: with a ``(B, T, D)`` ``x``, frames of each utterance (default: ``T``).

    Returns:
        ``(n // 2 + 1, D)`` (or ``(B, n // 2 + 1, D)``) power, and the phase of the same shape if asked.
    """
    import torch

    from .._lib import NNK_MS_POWER
    _checked(x, "x")
    _check_n(n)
    fwd, _ = _scales(norm, n)
    B, T, D, lens, frames = _batch(x, lengths)
    if frames > n:
        raise ValueError("DFT length %d is shorter than the %d frames of x" % (n, frames))
    xt = _device_input(x, B, T, D)
    K = n // 2 + 1
    ms = torch.empty((B, K, D), dtype=xt.dtype, device=xt.device)
    ph = torch.empty((B, K, D), dtype=_complex_of(xt.dtype), device=xt.device) if return_phase else None
    _launch(NNK_MS_POWER, n, xt, None, ms, ph, B, T, 0, D, lens, fwd, 0.0)
    if return_phase:
        return _out(ms, x, x.ndim == 2), _out(ph, x, x.ndim == 2)
    return _out(ms, x, x.ndim == 2)


def modphase(x, n=4096, norm=None, lengths=None):
    """Phase of the modulation spectrum, ``modspec(x, n, norm, return_phase=True)[1]`` (modspec.py:57)."""
    return modspec(x, n, norm, return_phase=True, lengths=lengths)[1]


def inv_modspec(ms, phase, norm=None, lengths=None):
    """Trajectory from a modulation spectrum and its phase, ``irfft(sqrt(ms) * phase, n, axis=0)`` with
    ``n = 2 (len(ms) - 1)`` (preprocessing/modspec.py:61).

    Args:
        ms: ``(n // 2 + 1, D)`` power, or ``(B, n // 2 + 1, D)``.
        phase: complex (or real) phase of the same shape.
        norm: as in :func:`modspec`.
        lengths: with 3-D input, frames to return for each utterance.

    Returns:
        ``(n, D)`` (or ``(B, n, D)``) as the reference, the caller trims it; with ``lengths``,
        ``(B, max(lengths), D)`` with frames past each length set to 0.
    """
    import torch

    from .. import _device as dev
    from .._lib import NNK_MS_INVERSE
    _checked(ms, "ms")
    _checked(phase, "phase", (np.float32, np.float64, np.complex64, np.complex128))
    if tuple(ms.shape) != tuple(phase.shape):
        raise ValueError("ms %s and phase %s differ in shape" % (tuple(ms.shape), tuple(phase.shape)))
    n = 2 * (int(ms.shape[-2]) - 1) if ms.ndim in (2, 3) else 0
    B, K, D, lens, frames = _batch(ms, lengths, "ms", n)
    _check_n(n)
    _, inv = _scales(norm, n)
    T_out = n if lens is None else frames
    mt = _device_input(ms, B, K, D)
    pt = dev.to_device(phase, mt.device).resolve_conj().to(_complex_of(mt.dtype)).reshape(B, K, D).contiguous()
    out = torch.empty((B, T_out, D), dtype=mt.dtype, device=mt.device)
    _launch(NNK_MS_INVERSE, n, mt, pt, out, None, B, 0, T_out, D, lens, 1.0, inv)
    return _out(out, ms, ms.ndim == 2)


def modspec_smoothing(x, modfs, n=4096, norm=None, cutoff=50, log_domain=True, lengths=None):
    """Smooth trajectories by removing the high modulation-frequency bands of their MS
    (preprocessing/modspec.py:108).

    Bins at and above ``int(n * cutoff / modfs) + 1`` are set to 0 in the log-power domain
    (``log_domain=True``: they keep their phase at unit power) or in the power domain, then the trajectory is
    rebuilt and cut to its own length.

    Args:
        x: ``(T, D)`` trajectory, or a padded ``(B, T, D)`` batch with ``lengths``.
        modfs: sampling frequency of the MS domain (frames per second).
        n (int): DFT length, 256 .. 4096 (a power of two), at least the number of frames.
        norm: as in :func:`modspec`.
        cutoff (float): cut-off frequency in Hz, at most ``modfs // 2``; None keeps every band.
        log_domain (bool): remove the bands in the log-power domain.
        lengths: with a ``(B, T, D)`` ``x``, frames of each utterance (later frames of the result are 0).

    Returns:
        Smoothed trajectories, the shape of ``x``.
    """
    import torch

    from .._lib import NNK_MS_SMOOTH
    _checked(x, "x")
    if cutoff is not None and cutoff > modfs // 2:
        raise ValueError("cutoff frequency %s Hz is above the Nyquist frequency %s Hz of the modulation spectrum"
                         % (cutoff, modfs // 2))
    _check_n(n)
    fwd, inv = _scales(norm, n)
    B, T, D, lens, frames = _batch(x, lengths)
    if frames > n:
        raise RuntimeError("DFT length %d must be larger than time length %d" % (n, frames))
    K = n // 2 + 1
    limit = K if cutoff is None else int(n * cutoff / modfs) + 1
    if limit < 0:  # the reference's ms[limit:] = 0 counts a negative start from the end
        limit = max(0, K + limit)
    xt = _device_input(x, B, T, D)
    out = torch.empty_like(xt)
    _launch(NNK_MS_SMOOTH, n, xt, None, out, None, B, T, T, D, lens, fwd, inv, min(limit, K), log_domain)
    return _out(out, x, x.ndim == 2)


def _modspec_grad(y, grad_ms, n, norm, lengths=None):
    """dL/dy of L(modspec(y, n, norm)) for CUDA tensors: ``y`` (T, D) or (B, T, D), ``grad_ms`` the shape of the
    power spectrum.  Frames past ``lengths`` get 0."""
    import torch

    from .._lib import NNK_MS_GRAD
    B, T, D, lens, _ = _batch(y, lengths)
    fwd, _ = _scales(norm, n)
    yt = _device_input(y, B, T, D)
    g = grad_ms.detach().to(device=yt.device, dtype=yt.dtype).reshape(B, n // 2 + 1, D).contiguous()
    out = torch.empty_like(yt)
    _launch(NNK_MS_GRAD, n, yt, g, out, None, B, T, T, D, lens, fwd, 0.0)
    return out[0] if y.ndim == 2 else out


__all__ = ["modspec", "modphase", "inv_modspec", "modspec_smoothing"]
