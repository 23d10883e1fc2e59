"""Post-filters on the GPU: Merlin's mel-cepstral post-filter (drop-in for ``nnmnkwii.postfilters``, without
pysptk) and the modulation-spectrum post-filter with its statistics (additive)."""
import numpy as np

__all__ = ["merlin_post_filter", "modspec_post_filter", "modspec_statistics"]

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


# ---- modulation-spectrum post-filter (Takamichi et al., ICASSP 2014), utterance level ----------------------------------
def _ms_input(x, n, lengths):
    """(B, T, D, host lengths) of a trajectory or padded batch the MS post-filter takes; argument errors only."""
    from .preprocessing.modspec import _batch, _check_n, _checked
    _checked(x, "x")
    _check_n(n)
    B, T, D, lens, frames = _batch(x, lengths)
    if frames > n:
        raise ValueError("DFT length %d is shorter than the %d frames of x" % (n, frames))
    return B, T, D, lens


def modspec_statistics(x, n=4096, lengths=None, segment=None):
    """Statistics of the log modulation spectrum over a set of utterances, for :func:`modspec_post_filter`.

    For each utterance and feature column, ``s_j = log(max(|rfft(x[:, d], n)_j|^2, tiny))`` (natural log; ``tiny``
    is the smallest normal number of ``x``'s dtype and only matters for bins of exactly zero power): the log of
    ``preprocessing.modspec`` with the default norm.  ``mean[j, d]`` and ``var[j, d]`` are the mean and the
    population variance of ``s_j`` across the utterances, accumulated in float64 in a fixed order (two passes).

    Runs on the GPU in two launches: the log power of every utterance into a temporary ``(B, n // 2 + 1, D)``
    array in ``x``'s dtype (``nnk_modspec``, csrc/nnk_modspec.cu), then its moments (``nnk_segment_moments``).  The
    temporary costs ``B * (n // 2 + 1) * D`` elements: about 250 MB for 512 float32 utterances at ``n = 4096``,
    ``D = 60``.  The statistics are not accumulated in chunks, so the whole set goes in one call.

    Pass the columns you will filter, typically ``mgc[:, 1:]``: the power coefficient (column 0) is usually left
    alone.  Compute the natural statistics on natural speech and the generated ones on the model's output for
    the same kind of utterances, with the same ``n`` (and the same ``segment``).

    **Segment level** (``segment=L``, the paper's other variant).  Each utterance of ``T`` frames is cut into
    ``J = ceil(T / H) + 1`` overlapping segments (none when ``T = 0``) with the hop ``H = L / 2``: segment ``j``
    starts at frame ``(j - 1) H`` and frames outside ``[0, T)`` are 0, so every frame lies in exactly two
    segments, and the first and last segments lie half outside the utterance (they count like any other).  Each
    segment is windowed with the periodic Hann window ``w_m = 0.5 - 0.5 cos(2 pi m / L)``, and ``s_j`` is the log
    power of ``rfft(w * segment, n)``.  ``mean`` and ``var`` are taken over all segments of all utterances, so
    utterances of any length count, and a corpus gives many more samples per bin than at the utterance level.
    The statistics have the same shape as utterance-level statistics of the same ``n``: nothing tells the two
    apart, so keep track of which kind you computed.  The temporary holds every segment's log power,
    ``S * (n // 2 + 1) * D`` elements for ``S`` segments in all.

    Args:
        x: ``(T, D)`` trajectory (one utterance) or a padded ``(B, T, D)`` batch; float32 / float64 CUDA tensor or
            NumPy array (a CPU tensor is refused).
        n (int): DFT length, 256, 512, 1024, 2048 or 4096, at least every utterance's length; with ``segment``,
            the per-segment DFT length, 32, 64, 128, 256 or 512.
        lengths: with a ``(B, T, D)`` ``x``, frames of each utterance (default: ``T``); frames past a length are
            never read.
        segment (int): ``None`` for the utterance level, or the segment length ``L``, even, ``4 <= L <= n``.

    Returns:
        ``(mean, var)``, each float64 of shape ``(n // 2 + 1, D)``: NumPy arrays for NumPy ``x``, tensors on
        ``x``'s device otherwise.

    Raises:
        ValueError: ``n`` not supported, an utterance longer than ``n``, no utterance, or an utterance of no
            frames (it has no modulation spectrum), all before any device work.  With ``segment``: an ``n`` or
            ``L`` not supported, or a set without a segment (zero-length utterances are skipped); a ``segment``
            that is not an int is a TypeError.
    """
    import torch

    from . import _device as dev
    from . import _lib
    from .preprocessing.modspec import _device_input, _launch
    if segment is not None:
        return _segment_statistics(x, n, lengths, segment)
    B, T, D, lens = _ms_input(x, n, lengths)
    if B == 0:
        raise ValueError("modspec_statistics needs at least one utterance")
    if (T if lens is None else int(lens.min())) < 1:
        raise ValueError("every utterance needs at least one frame (a zero-length utterance has no modulation "
                         "spectrum)")
    K = n // 2 + 1
    xt = _device_input(x, B, T, D)
    device = xt.device
    logms = torch.empty((B, K, D), dtype=xt.dtype, device=device)
    _launch(_lib.NNK_MS_LOGPOWER, n, xt, None, logms, None, B, T, 0, D, lens, 1.0, 0.0)
    mean = torch.empty((K, D), dtype=torch.float64, device=device)
    var = torch.empty((K, D), dtype=torch.float64, device=device)
    if D:  # one segment of B rows and K * D columns
        off = torch.tensor([0, B], dtype=torch.int64, device=device)
        _lib.check(_lib.lib.nnk_segment_moments(logms.data_ptr(), dev.torch_dtype_code(logms.dtype), K * D, K * D,
                                                off.data_ptr(), None, 1, mean.data_ptr(), var.data_ptr(),
                                                dev.current_stream_ptr(device)), "nnk_segment_moments")
    return dev.like_input(mean, x), dev.like_input(var, x)


def _ms_stats(pairs, K, D):
    """float64 host ``(mean, var)`` of each named statistics pair, checked: shape ``(K, D)``, finite means,
    finite non-negative variances.  Shapes and types of every pair are checked before any value is read."""
    from . import _device as dev
    from .preprocessing.modspec import _checked
    for name, pair in pairs:
        if not isinstance(pair, (tuple, list)) or len(pair) != 2:
            raise TypeError("%s must be a (mean, var) pair" % name)
        for a, what in zip(pair, ("mean", "var")):
            _checked(a, "%s %s" % (name, what))
            if tuple(a.shape) != (K, D):
                raise ValueError("%s %s is %s, expected (n // 2 + 1, D) = %s: statistics of another n or D?"
                                 % (name, what, tuple(a.shape), (K, D)))
    out = []
    for name, pair in pairs:
        m, v = (np.asarray(a.detach().cpu().numpy() if dev.is_tensor(a) else a, dtype=np.float64) for a in pair)
        if not np.isfinite(m).all():
            raise ValueError("%s mean is not finite" % name)
        if not np.isfinite(v).all() or (v < 0).any():
            raise ValueError("%s var must be finite and >= 0" % name)
        out.append((m, v))
    return out


def _ms_table(natural, generated, k, K, D, dtype):
    """The filter's ``(K, D, 2)`` table ``(a, c)``, ``s' = a s + c``, computed in float64 and stored in ``dtype``."""
    (mu_n, v_n), (mu_g, v_g) = _ms_stats([("natural", natural), ("generated", generated)], K, D)
    g = np.sqrt(np.divide(v_n, v_g, out=np.ones_like(v_n), where=v_g > 0))
    return np.stack([(1.0 - k) + k * g, k * (mu_n - g * mu_g)], axis=-1).astype(dtype)


def modspec_post_filter(x, natural, generated, k=1.0, n=4096, lengths=None, segment=None):
    """Modulation-spectrum (MS) post-filter of Takamichi et al., "A postfilter to modify the modulation spectrum
    in HMM-based speech synthesis", ICASSP 2014, at the utterance level, on the GPU.

    Generated trajectories are over-smoothed: their MS is too low at the higher modulation frequencies.  The
    filter moves each utterance's log MS towards the statistics of natural speech.  For one utterance of
    ``T <= n`` frames and one column, with ``Y = rfft(x[:, d], n)`` and ``s_j = log(max(|Y_j|^2, tiny))`` as in
    :func:`modspec_statistics`, every bin ``j >= 1`` of non-zero power becomes (statistics taken at bin ``j``,
    column ``d``; ``k`` is the emphasis weight)::

        g   = sqrt(v_N / v_G)                    (1 where v_G == 0)
        s'  = (1 - k) s_j + k (g (s_j - mu_G) + mu_N)
        C_j = Y_j / |Y_j| exp(s' / 2)

    and the result is ``irfft(C, n)[:T]``.  ``k = 0``, or equal natural and generated statistics, gives ``x``
    back to rounding.

    Deliberate choices:
      * utterance level by default: the filter sees each utterance's whole MS; ``segment=L`` selects the
        segment-level variant below;
      * bin 0 is not filtered (``C_0 = Y_0``): it is ``T`` times the column's mean, which the acoustic model sets,
        not modulation, so each column keeps its level.  A bin of zero power stays 0, so an all-zero column comes
        out all zero;
      * there is no ``norm`` argument: with one norm for the statistics and the filter, a norm shifts ``s``,
        ``mu_N`` and ``mu_G`` by the same constant and leaves the result unchanged;
      * ``k`` outside ``[0, 1]``, non-finite means and negative or non-finite variances raise ``ValueError``.

    Each utterance and column is filtered on its own; frames past an utterance's length are written as 0, and a
    zero-length utterance comes back as zeros.  Runs on the GPU (``nnk_modspec``, csrc/nnk_modspec.cu): one CTA
    per (utterance, column) does the forward FFT, the per-bin filter and the inverse FFT in shared memory.  The
    per-bin gain ``s' = a s + c`` is tabulated on the host in float64 from the statistics
    (``a = (1 - k) + k g``, ``c = k (mu_N - g mu_G)``); statistics given as CUDA tensors are copied to the host
    for that, which waits for the current stream.

    Pass the columns the statistics were computed on, typically ``mgc[:, 1:]`` (leave the power coefficient
    alone).

    **Segment level** (``segment=L``).  The utterance is cut into the windowed segments of
    :func:`modspec_statistics` (hop ``H = L / 2``, periodic Hann window ``w``, segment ``j`` from frame
    ``(j - 1) H``, ``J = ceil(T / H) + 1`` of them), each segment's spectrum ``Y_j = rfft(w * segment, n)`` is
    filtered bin by bin as above, and the result is overlap-added without a synthesis window::

        y_t = sum_j irfft(C_j, n)[t - (j - 1) H]     over the j with 0 <= t - (j - 1) H < L

    For this window ``w_m + w_{m + H} = 1``, so ``k = 0`` or equal statistics give ``x`` back to rounding.
    There is no limit on the utterance's length, and the cost grows with its frames, not with the longest
    utterance of the batch.  The first and last segments lie half outside the utterance and are filtered like
    the others.  Use statistics computed with the same ``n`` and ``segment``: segment-level and utterance-level
    statistics of one ``n`` have the same shape, so the shape check cannot tell them apart.  Runs on the GPU
    (``nnk_ms_segment``, csrc/nnk_ms_segment.cu): one CTA per (utterance, tile of frames, group of columns)
    filters every segment of its tile, one warp per (segment, column), and overlap-adds them in shared memory.

    Args:
        x: ``(T, D)`` trajectory or a padded ``(B, T, D)`` batch; float32 / float64 CUDA tensor or NumPy array (a
            CPU tensor is refused).
        natural: ``(mean, var)`` of natural speech from :func:`modspec_statistics`, each ``(n // 2 + 1, D)``,
            NumPy arrays or CUDA tensors.
        generated: ``(mean, var)`` of generated speech, likewise.
        k (float): emphasis weight in ``[0, 1]``; 1 replaces the MS statistics completely.
        n (int): DFT length, 256, 512, 1024, 2048 or 4096, at least every utterance's length; the ``n`` of the
            statistics.  With ``segment``: the per-segment DFT length, 32, 64, 128, 256 or 512.
        lengths: with a ``(B, T, D)`` ``x``, frames of each utterance (default: ``T``).
        segment (int): ``None`` for the utterance level, or the segment length ``L``, even, ``4 <= L <= n``.

    Returns:
        The filtered trajectories: ``x``'s shape and dtype, NumPy for NumPy ``x``, a tensor on ``x``'s device
        otherwise.

    Raises:
        ValueError: for any of the range checks above, an ``n`` not supported, an utterance longer than ``n``
            (utterance level only), a ``segment`` length not supported, or statistics of the wrong shape;
            TypeError for inputs that are not float arrays or a ``segment`` that is not an int.  Argument errors
            are raised before any device work.
    """
    import torch

    from . import _device as dev
    from . import _lib
    from .preprocessing.modspec import _device_input, _launch, _out
    if segment is not None:
        return _segment_post_filter(x, natural, generated, k, n, lengths, segment)
    B, T, D, lens = _ms_input(x, n, lengths)
    k = float(k)
    if not 0.0 <= k <= 1.0:
        raise ValueError("k must be in [0, 1], got %r" % k)
    table = _ms_table(natural, generated, k, n // 2 + 1, D, dev.np_dtype(x))
    xt = _device_input(x, B, T, D)
    out = torch.empty_like(xt)
    _launch(_lib.NNK_MS_POSTFILTER, n, xt, dev.to_device(table, xt.device), out, None, B, T, T, D, lens, 1.0,
            1.0 / n)
    return _out(out, x, x.ndim == 2)


# ---- segment level (csrc/nnk_ms_segment.cu) ------------------------------------------------------------------------
SEGMENT_NS = (32, 64, 128, 256, 512)


def _segment_input(x, n, lengths, segment):
    """(B, T, D, host lengths or None, L) of a segment-level call; argument errors only."""
    from .preprocessing.modspec import _batch, _checked
    _checked(x, "x")
    if n not in SEGMENT_NS:
        raise ValueError("with segment, n must be one of %s, got %r" % (", ".join(map(str, SEGMENT_NS)), n))
    if isinstance(segment, bool) or not isinstance(segment, (int, np.integer)):
        raise TypeError("segment must be an int (the segment length L) or None, got %s" % type(segment).__name__)
    L = int(segment)
    if L % 2 or not 4 <= L <= n:
        raise ValueError("segment length must be even with 4 <= L <= n = %d, got %d" % (n, L))
    B, T, D, lens, _ = _batch(x, lengths)
    return B, T, D, lens, L


def _segment_counts(lengths, L):
    """Segments ``ceil(T / (L / 2)) + 1`` of each length ``T`` (0 for ``T = 0``), int64."""
    lens = np.asarray(lengths, np.int64)
    H = L // 2
    return np.where(lens > 0, -(-lens // H) + 1, 0)


def _segment_launch(mode, n, L, xt, table, out, B, T, D, lens, seg_off=None):
    """Enqueue nnk_ms_segment on the current stream of ``out``'s device."""
    from . import _device as dev
    from . import _lib
    lt = dev.lengths_on(lens, out.device)
    _lib.check(_lib.lib.nnk_ms_segment(mode, dev.torch_dtype_code(xt.dtype), n, L, xt.data_ptr(),
                                       table.data_ptr() if table is not None else None, out.data_ptr(), B, T, D,
                                       lt.data_ptr() if lt is not None else None, seg_off.data_ptr() if seg_off is not None else None,
                                       dev.current_stream_ptr(out.device)), "nnk_ms_segment")


def _segment_statistics(x, n, lengths, segment):
    import torch

    from . import _device as dev
    from . import _lib
    from .preprocessing.modspec import _device_input
    B, T, D, lens, L = _segment_input(x, n, lengths, segment)
    J = _segment_counts(np.full(B, T) if lens is None else lens, L)
    S = int(J.sum())
    if S == 0:
        raise ValueError("modspec_statistics needs at least one segment (every utterance has zero frames)")
    K = n // 2 + 1
    xt = _device_input(x, B, T, D)
    device = xt.device
    mean = torch.empty((D, K), dtype=torch.float64, device=device)
    var = torch.empty((D, K), dtype=torch.float64, device=device)
    if D:
        logms = torch.empty((S, D, K), dtype=xt.dtype, device=device)
        seg_off = torch.as_tensor(np.concatenate([[0], np.cumsum(J)[:-1]]).astype(np.int64), device=device)
        _segment_launch(_lib.NNK_MSSEG_LOGPOWER, n, L, xt, None, logms, B, T, D, lens, seg_off)
        off = torch.tensor([0, S], dtype=torch.int64, device=device)  # one segment of S rows and D * K columns
        _lib.check(_lib.lib.nnk_segment_moments(logms.data_ptr(), dev.torch_dtype_code(logms.dtype), D * K, D * K,
                                                off.data_ptr(), None, 1, mean.data_ptr(), var.data_ptr(),
                                                dev.current_stream_ptr(device)), "nnk_segment_moments")
    return dev.like_input(mean.t().contiguous(), x), dev.like_input(var.t().contiguous(), x)


def _segment_post_filter(x, natural, generated, k, n, lengths, segment):
    import torch

    from . import _device as dev
    from . import _lib
    from .preprocessing.modspec import _device_input, _out
    B, T, D, lens, L = _segment_input(x, n, lengths, segment)
    k = float(k)
    if not 0.0 <= k <= 1.0:
        raise ValueError("k must be in [0, 1], got %r" % k)
    table = _ms_table(natural, generated, k, n // 2 + 1, D, dev.np_dtype(x))
    xt = _device_input(x, B, T, D)
    out = torch.empty_like(xt)
    _segment_launch(_lib.NNK_MSSEG_POSTFILTER, n, L, xt, dev.to_device(table, xt.device), out, B, T, D, lens)
    return _out(out, x, x.ndim == 2)
