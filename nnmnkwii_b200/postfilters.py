"""Merlin's mel-cepstral post-filter on the GPU (drop-in for ``nnmnkwii.postfilters``, without pysptk)."""
import numpy as np

__all__ = ["merlin_post_filter"]

_basis_cache = {}


def _basis(device, alpha, D, order, fftlen):
    """float64 basis of (device, alpha, D, order, fftlen), built once on the device (csrc/nnk_postfilter.cu).

    The build is synchronised before the basis enters the cache, so a later call on any stream may read it.
    The caller reads it on the current stream of ``device``; an eviction never recycles its block before
    that read has run."""
    import torch

    from . import _device as dev
    from . import _lib

    key = (str(device), float(alpha), D, order, fftlen)
    b = _basis_cache.get(key)
    if b is None:
        n = int(_lib.lib.nnk_postfilter_basis_elems(D, fftlen))
        if n == 0:
            raise NotImplementedError("merlin_post_filter: D = %d / fftlen = %d is not supported by the CUDA kernels "
                                      "(D <= 128, fftlen <= 8192)" % (D, fftlen))
        b = torch.empty(n, dtype=torch.float64, device=device)
        _lib.check(_lib.lib.nnk_postfilter_basis(float(alpha), D, order, fftlen, b.data_ptr(), n,
                                                 dev.current_stream_ptr(device)), "nnk_postfilter_basis")
        torch.cuda.current_stream(device).synchronize()
        if len(_basis_cache) >= 32:
            _basis_cache.clear()
        _basis_cache[key] = b
    return dev.keep_for_current_stream(b, device)


def merlin_post_filter(mgc, alpha, minimum_phase_order=511, fftlen=1024, coef=1.4, weight=None):
    """Post-filter used in Merlin (nnmnkwii/postfilters/__init__.py:7-62), computed on the GPU.

    ``mgc`` is ``(T, D)`` mel-generalized cepstrum, a NumPy array (copied to the device and back; NumPy
    is returned) or a torch CUDA tensor (processed on the current stream; a CUDA tensor is returned).
    Rows may be strided: a column slice such as ``y[:, :60]`` of an MLPG output is read in place.  The
    filter works frame by frame, so several utterances back to back are one call; an all-zero frame
    comes out exactly zero.  ``weight`` defaults to ``coef`` with 1 at indices 0 and 1, as in the
    reference; ``len(weight) != D`` raises ``AssertionError``.

    The result equals the reference's ``b2mc(mc2b(w * mgc) with coefficient 0 shifted by
    log(r0 / p_r0) / 2)`` (r0 = ``c2acr(freqt(mgc, minimum_phase_order, -alpha), 0, fftlen)``), computed
    in float64 as ``w * mgc`` with the shift added to column 0 (mc2b and b2mc are exact inverses
    elsewhere).  float32 input gives float32 output, float64 gives float64, any other dtype is computed
    and returned as float64.

    Raises ``ValueError`` before any device work when ``mgc`` is not 2-D, ``fftlen`` is not a power of
    two (SPTK's ``fftr`` refuses other lengths), ``minimum_phase_order < 0`` or
    ``minimum_phase_order + 1 > fftlen`` (``c2acr`` needs the coefficients to fit in its FFT buffer).
    These are this package's checks: pysptk's own argument checks are not restated.  ``D > 128`` or
    ``fftlen > 8192`` raises ``NotImplementedError``.  There is no CPU path.
    """
    import torch

    from . import _device as dev
    from . import _lib

    if mgc.ndim != 2:
        raise ValueError("merlin_post_filter: mgc must be 2-D (T, D), got %d-D" % mgc.ndim)
    T, D = (int(s) for s in mgc.shape)
    if weight is None:
        weight = np.ones(D) * coef
        weight[:2] = 1
    assert len(weight) == D
    fftlen, order = int(fftlen), int(minimum_phase_order)
    if fftlen < 1 or fftlen & (fftlen - 1):
        raise ValueError("merlin_post_filter: fftlen must be a power of two, got %d" % fftlen)
    if order < 0:
        raise ValueError("merlin_post_filter: minimum_phase_order must be >= 0, got %d" % order)
    if order + 1 > fftlen:
        raise ValueError("merlin_post_filter: minimum_phase_order + 1 (%d) exceeds fftlen (%d)" % (order + 1, fftlen))
    if dev.is_tensor(weight):
        weight = weight.detach().cpu().numpy()
    weight = np.ascontiguousarray(weight, dtype=np.float64).ravel()
    dev.require_cuda()

    if dev.is_tensor(mgc):
        if not mgc.is_cuda:
            raise ValueError("merlin_post_filter: a torch tensor must be on a CUDA device")
        x = mgc if mgc.dtype in (torch.float32, torch.float64) else mgc.to(torch.float64)
        if x.stride(1) != 1 or x.stride(0) < D:
            x = x.contiguous()
    else:
        xn = np.ascontiguousarray(mgc)
        x = torch.from_numpy(xn if xn.dtype in (np.float32, np.float64) else xn.astype(np.float64)).cuda()
    device = x.device
    out = torch.empty((T, D), dtype=x.dtype, device=device)
    if T and D:
        basis = _basis(device, alpha, D, order, fftlen)
        w = dev.constant_on_device(weight, device)
        _lib.check(_lib.lib.nnk_postfilter_apply(x.data_ptr(), dev.torch_dtype_code(x.dtype), T, D, max(x.stride(0), D),
                                                 w.data_ptr(), fftlen, basis.data_ptr(), basis.numel(), out.data_ptr(), D,
                                                 dev.current_stream_ptr(device)), "nnk_postfilter_apply")
    return dev.like_input(out, mgc)
