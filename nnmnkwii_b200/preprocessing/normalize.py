"""Corpus normalisation -- drop-in for the statistics and scaling functions of
``nnmnkwii.preprocessing`` (nnmnkwii/preprocessing/generic.py:335-828).

``meanvar``, ``meanstd`` and ``minmax`` make one pass over the valid frames on the GPU (C ABI
``nnk_frame_stats``, csrc/nnk_stats.cu): count, mean, sum of squared deviations, min and max of every
column in float64, merged with Chan's pairwise formula in a fixed order (two identical calls are
bit-identical).  ``dataset`` may be

  (a) a sized, indexable or iterable set of ``(T, D)`` NumPy arrays (e.g. ``FileSourceDataset``):
      utterances, cut to ``lengths[idx]``, are packed back to back into a bounded page-locked staging
      buffer (``STAGING_BYTES``); one launch per full buffer, the running state stays on the device;
  (b) a 3-D NumPy array ``(B, T, D)``: the same staging path, no full-size device copy;
  (c) a 3-D CUDA tensor: read in place, one launch.

(a) and (b) return NumPy arrays of ``dataset[0].dtype``; (c) returns CUDA tensors of the tensor's dtype,
so ``inv_scale`` -> ``paramgen.mlpg_batch(variances=Y_var)`` stays on the device.  Inputs other than
float32 / float64 are computed in float64 and cast back, as the reference does.

``scale``, ``inv_scale``, ``minmax_scale`` and ``inv_minmax_scale`` run one per-column affine kernel
(``nnk_column_affine``) in ``numpy.result_type(x, params)`` with IEEE round-to-nearest operations and no
FMA contraction: bit-identical to the reference's NumPy expression.  The parameter arithmetic
(``minmax_scale_params``, zero ranges and zero standard deviations) is done on the D-vectors.

Deliberate differences from the reference:
  * a 2-D ``dataset`` raises ``ValueError`` (the reference iterates its rows);
  * ``lengths`` must have one entry per item, each >= 0 (``ValueError``); a length above T is clipped,
    as slicing does;
  * an empty utterance is skipped (in the reference it turns every variance into NaN);
  * ``minmax`` with no frames, and ``meanvar`` / ``meanstd`` with no frames and
    ``last_sample_count == 0``, raise ``ValueError``;
  * a NaN propagates into its column's mean, variance, min and max (scikit-learn's per-column NaN
    counts are not restated; the reference mixes them with a scalar count).
"""
import numpy as np

STAGING_BYTES = 256 << 20  # page-locked host staging for forms (a) and (b): two halves, double-buffered

_pinned = {}


def _handle_zeros_in_scale(scale, copy=True):
    """Zero scale -> 1 (preprocessing/generic.py:7-21); NumPy arrays, scalars or torch tensors."""
    if np.isscalar(scale):
        return 1.0 if scale == 0.0 else scale
    if isinstance(scale, np.ndarray):
        if copy:
            scale = scale.copy()
        scale[scale == 0.0] = 1.0
        return scale
    from .._device import is_tensor
    if is_tensor(scale):
        import torch
        return torch.where(scale == 0.0, torch.ones_like(scale), scale)
    return scale


def remove_zeros_frames(x, eps=1e-7):
    """Remove zeros frames (preprocessing/generic.py:335-356): host-side, the reference's semantics."""
    T, D = x.shape
    s = np.sum(np.abs(x), axis=1)
    s[s < eps] = 0.0
    return x[s > eps]


# ---- statistics ----------------------------------------------------------------------------------------
def _compute_dtype(dt):
    return np.float32 if np.dtype(dt) == np.float32 else np.float64


class _State:
    """The running device state [count, mean[D], m2[D], min[D], max[D]] (float64) of one pass."""

    def __init__(self, D, device, mean_, var_, count):
        import torch
        self.D = D
        self.device = device
        s = torch.empty(1 + 4 * D, dtype=torch.float64, device=device)
        s[0] = float(count)
        s[1:1 + D] = _vec_f64(mean_, D, device)
        s[1 + D:1 + 2 * D] = _vec_f64(var_, D, device) * float(count)  # var_ * count, as sklearn's last_unnormalized_variance
        s[1 + 2 * D:1 + 3 * D] = float("inf")
        s[1 + 3 * D:] = float("-inf")
        self.t = s

    def fold(self, x, ld, utt_off, lengths, n_utt, max_rows):
        """Enqueue nnk_frame_stats over the utterances of device matrix x (float32 / float64)."""
        from .. import _device as dev
        from .._lib import check, lib
        if n_utt == 0 or max_rows == 0:
            return
        need = int(lib.nnk_frame_stats_workspace_bytes(n_utt, max_rows, self.D))
        ws = dev.workspace(self.device, need)
        check(lib.nnk_frame_stats(x.data_ptr(), dev.torch_dtype_code(x.dtype), self.D, ld, utt_off.data_ptr(),
                                  lengths.data_ptr() if lengths is not None else None, n_utt, max_rows,
                                  self.t.data_ptr(), ws.data_ptr(), ws.numel(), dev.current_stream_ptr(self.device)),
              "nnk_frame_stats")


def _vec_f64(v, D, device):
    import torch

    from .._device import is_tensor
    if is_tensor(v):
        t = v.detach().to(device=device, dtype=torch.float64)
    else:
        t = torch.as_tensor(np.asarray(v, dtype=np.float64), device=device)
    if t.dim() > 1 or (t.dim() == 1 and t.numel() not in (1, D)):
        raise ValueError("initial statistics must be scalars or of shape (%d,)" % D)
    return t.reshape(-1).expand(D) if t.dim() == 1 else t.expand(D)


def _pinned_buffer(nbytes):
    import torch
    buf = _pinned.get(nbytes)
    if buf is None:
        _pinned.clear()
        buf = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        _pinned[nbytes] = buf
    return buf


def _stats_tensor(x, lens, mean_, var_, count):
    """Form (c): a 3-D CUDA tensor, read in place with one launch."""
    import torch

    from .. import _device as dev
    B, T, D = (int(s) for s in x.shape)
    if x.dtype not in (torch.float32, torch.float64):
        x = x.to(torch.float64)
    ld = int(x.stride(1)) if T > 1 else int(x.stride(0))
    if not (x.stride(2) == 1 and ld >= D and (B == 1 or x.stride(0) == T * ld)):
        x = x.contiguous()
        ld = D
    frames = B * T if lens is None else int(np.minimum(lens, T).sum())
    st = _State(D, x.device, mean_, var_, count)
    if frames:
        off = torch.arange(B + 1, dtype=torch.int64, device=x.device) * T  # padded batch: utterance b at row b * T
        st.fold(x, ld, off, dev.lengths_on(lens, x.device, T), B, T)
    return st, frames


def _stats_host(dataset, lens, mean_, var_, count):
    """Forms (a) and (b): pack utterances into page-locked staging, one launch per full buffer."""
    import torch

    from .. import _device as dev
    device = dev.cuda_device()
    stream = torch.cuda.current_stream(device)
    st = None
    dtype = None
    cdt = None
    half = STAGING_BYTES // 2
    slots, events, dev_bufs = None, [None, None], [None, None]
    slot, fill, frames, cap = 0, 0, 0, 0

    def flush():
        nonlocal slot, fill
        if fill == 0:
            return
        host = slots[slot][:fill * st.D * np.dtype(cdt).itemsize]
        d = dev_bufs[slot]
        d[:host.numel()].copy_(host, non_blocking=True)
        x = d[:host.numel()].view(torch.float32 if cdt == np.float32 else torch.float64)
        off = torch.tensor([0, fill], dtype=torch.int64).to(device, non_blocking=True)
        st.fold(x, st.D, off, None, 1, fill)
        ev = torch.cuda.Event()
        ev.record(stream)
        events[slot] = ev
        slot, fill = 1 - slot, 0
        if events[slot] is not None:
            events[slot].synchronize()  # the other half's copy has finished: it can be refilled

    for idx, x in enumerate(dataset):
        if dev.is_tensor(x):
            x = x.detach().cpu().numpy()
        x = np.asarray(x)
        if x.ndim != 2:
            raise ValueError("every item of dataset must be a (T, D) array, item %d has shape %s" % (idx, x.shape))
        if st is None:
            dtype = x.dtype
            cdt = _compute_dtype(dtype)
            D = int(x.shape[1])
            if D < 1:
                raise ValueError("dataset has no columns")
            st = _State(D, device, mean_, var_, count)
            esz = np.dtype(cdt).itemsize
            cap = max(1, half // (D * esz))
            buf = _pinned_buffer(2 * cap * D * esz)
            slots = [buf[:cap * D * esz], buf[cap * D * esz:]]
            dev_bufs = [torch.empty(cap * D * esz, dtype=torch.uint8, device=device) for _ in range(2)]
        elif x.shape[1] != st.D:
            raise ValueError("item %d has %d columns, item 0 has %d" % (idx, x.shape[1], st.D))
        if lens is not None:
            x = x[:lens[idx]]
        done = 0
        while done < len(x):
            k = min(cap - fill, len(x) - done)
            view = slots[slot].numpy().view(cdt).reshape(cap, st.D)
            np.copyto(view[fill:fill + k], x[done:done + k], casting="unsafe")
            fill += k
            done += k
            frames += k
            if fill == cap:
                flush()
    if st is None:
        raise ValueError("dataset is empty")
    flush()
    return st, frames, dtype


def _run_stats(dataset, lengths, mean_=0.0, var_=0.0, count=0, allow_empty=False):
    """-> (state, frames, result dtype or None for CUDA results).  Argument errors come before any launch."""
    from .. import _device as dev
    T = None
    if isinstance(dataset, np.ndarray) or dev.is_tensor(dataset):
        if len(dataset.shape) != 3:
            raise ValueError("an array dataset must be (B, T, D), got %d-D" % len(dataset.shape))
        T = int(dataset.shape[1])
        if int(dataset.shape[2]) < 1:
            raise ValueError("dataset has no columns")
    n_items = None
    try:
        n_items = len(dataset)
    except TypeError:
        pass
    lens = dev.check_lengths(lengths, n_items)
    if n_items == 0:
        raise ValueError("dataset is empty")
    if not allow_empty and (T == 0 or (lens is not None and int(lens.sum()) == 0)):
        raise ValueError("no frames: every length is 0")
    dev.require_cuda()
    if dev.is_tensor(dataset) and dataset.is_cuda:
        st, frames = _stats_tensor(dataset, lens, mean_, var_, count)
        return st, frames, None
    return _stats_host(dataset, lens, mean_, var_, count)


def _finish_meanvar(st, dtype, ref):
    """mean, var (= m2 / count) in the result dtype; `ref` is the input tensor of form (c) or None."""
    D = st.D
    if dtype is None:
        n = st.t[0]
        mean = st.t[1:1 + D]
        var = st.t[1 + D:1 + 2 * D] / n
        return mean.to(ref.dtype), var.to(ref.dtype)
    s = st.t.cpu().numpy()
    return s[1:1 + D].astype(dtype), (s[1 + D:1 + 2 * D] / s[0]).astype(dtype)


def _meanvar(dataset, lengths, mean_, var_, last_sample_count):
    count = int(last_sample_count)
    if count < 0:
        raise ValueError("last_sample_count must be >= 0")
    st, frames, dtype = _run_stats(dataset, lengths, mean_, var_, count, allow_empty=count > 0)
    if frames == 0 and count == 0:
        raise ValueError("meanvar: no frames (all lengths are 0) and last_sample_count == 0")
    m, v = _finish_meanvar(st, dtype, dataset if dtype is None else None)
    return m, v, count + frames


def meanvar(dataset, lengths=None, mean_=0.0, var_=0.0, last_sample_count=0, return_last_sample_count=False):
    """Mean and variance of every column over a dataset (preprocessing/generic.py:496-549).

    Args:
        dataset: forms (a), (b) or (c) of the module docstring.
        lengths (list): frame lengths of the items (padded data); one entry per item, each >= 0.
        mean_, var_ (array or scalar): incoming statistics, merged first.
        last_sample_count (int): frames behind ``mean_`` / ``var_``.
        return_last_sample_count (bool): also return the total frame count (a Python int).
    """
    m, v, n = _meanvar(dataset, lengths, mean_, var_, last_sample_count)
    return (m, v, n) if return_last_sample_count else (m, v)


def meanstd(dataset, lengths=None, mean_=0.0, var_=0.0, last_sample_count=0, return_last_sample_count=False):
    """Mean and standard deviation (zero -> 1) of every column (preprocessing/generic.py:552-602)."""
    from .._device import is_tensor
    m, v, n = _meanvar(dataset, lengths, mean_, var_, last_sample_count)
    if is_tensor(v):
        import torch
        s = _handle_zeros_in_scale(torch.sqrt(v))
    else:
        s = _handle_zeros_in_scale(np.sqrt(v))
    return (m, s, n) if return_last_sample_count else (m, s)


def minmax(dataset, lengths=None):
    """Min and max of every column over a dataset (preprocessing/generic.py:605-636)."""
    st, frames, dtype = _run_stats(dataset, lengths)
    if frames == 0:
        raise ValueError("minmax: no frames (zero-size reduction)")
    D = st.D
    if dtype is None:
        return st.t[1 + 2 * D:1 + 3 * D].to(dataset.dtype), st.t[1 + 3 * D:].to(dataset.dtype)
    s = st.t.cpu().numpy()
    return s[1 + 2 * D:1 + 3 * D].astype(dtype), s[1 + 3 * D:].astype(dtype)


# ---- per-column affine maps ----------------------------------------------------------------------------
def _affine(x, a, b, form):
    """form 0: (x - a) / b, form 1: x * b + a, per column of the last axis, on the GPU."""
    import torch

    from .. import _device as dev
    from .._lib import check, lib
    dev.require_cuda()
    if len(x.shape) == 0:
        raise ValueError("x must have at least one dimension")
    D = int(x.shape[-1])
    params = [p if np.isscalar(p) and not isinstance(p, np.generic) else dev.np_dtype(p) for p in (a, b)]
    cdt = np.result_type(dev.np_dtype(x), *params)  # a Python scalar parameter stays weak, as in NumPy's promotion
    if cdt not in (np.float32, np.float64):
        raise TypeError("scaling computes in float32 or float64, numpy.result_type gives %s" % cdt)
    tcdt = torch.float32 if cdt == np.float32 else torch.float64
    xt = dev.to_device(x)
    device = xt.device
    if xt.dtype not in (torch.float32, torch.float64) or (xt.dtype == torch.float64 and tcdt == torch.float32):
        xt = xt.to(tcdt)
    xt = xt.contiguous()

    def vec(p):
        if dev.is_tensor(p):
            t = p.detach().to(device=device, dtype=tcdt)
        else:
            t = torch.as_tensor(np.asarray(p, dtype=cdt), device=device)
        if t.numel() not in (1, D) or t.dim() > 1:
            raise ValueError("scaling parameters must be scalars or of shape (%d,), got %s" % (D, tuple(t.shape)))
        return t.reshape(-1).expand(D).contiguous()
    av, bv = vec(a), vec(b)
    out = torch.empty(xt.shape, dtype=tcdt, device=device)
    rows = xt.numel() // D if D else 0
    if rows and D:
        check(lib.nnk_column_affine(xt.data_ptr(), dev.torch_dtype_code(xt.dtype), dev.torch_dtype_code(tcdt), rows, D,
                                    av.data_ptr(), bv.data_ptr(), form, out.data_ptr(), dev.current_stream_ptr(device)),
              "nnk_column_affine")
    return dev.like_input(out, x)


def scale(x, data_mean, data_std):
    """``(x - data_mean) / data_std`` with zero std -> 1 (preprocessing/generic.py:639-665)."""
    return _affine(x, data_mean, _handle_zeros_in_scale(data_std, copy=True), 0)


def inv_scale(x, data_mean, data_std):
    """``data_std * x + data_mean`` (preprocessing/generic.py:668-684)."""
    return _affine(x, data_mean, data_std, 1)


def _minmax_scale_factor(data_min, data_max, feature_range):
    data_range = data_max - data_min
    return (feature_range[1] - feature_range[0]) / _handle_zeros_in_scale(data_range, copy=False)


def minmax_scale_params(data_min, data_max, feature_range=(0, 1)):
    """``(min_, scale_)`` with ``x * scale_ + min_`` the min/max scaling (preprocessing/generic.py:695-731).
    Host arithmetic on the D-vectors (NumPy arrays or tensors); no GPU needed for NumPy inputs."""
    scale_ = _minmax_scale_factor(data_min, data_max, feature_range)
    min_ = feature_range[0] - data_min * scale_
    return min_, scale_


def _minmax_params(data_min, data_max, feature_range, scale_, min_, what):
    if (scale_ is None or min_ is None) and (data_min is None or data_max is None):
        raise ValueError("`data_min` and `data_max` or `scale_` and `min_` must be specified to perform %s" % what)
    if scale_ is None:
        scale_ = _minmax_scale_factor(data_min, data_max, feature_range)
    if min_ is None:
        min_ = feature_range[0] - data_min * scale_
    return min_, scale_


def minmax_scale(x, data_min=None, data_max=None, feature_range=(0, 1), scale_=None, min_=None):
    """``x * scale_ + min_`` (preprocessing/generic.py:734-786); ValueError without
    (``data_min``, ``data_max``) or (``scale_``, ``min_``)."""
    min_, scale_ = _minmax_params(data_min, data_max, feature_range, scale_, min_, "minmax scale")
    return _affine(x, min_, scale_, 1)


def inv_minmax_scale(x, data_min=None, data_max=None, feature_range=(0, 1), scale_=None, min_=None):
    """``(x - min_) / scale_`` (preprocessing/generic.py:789-828)."""
    min_, scale_ = _minmax_params(data_min, data_max, feature_range, scale_, min_, "inverse of minmax scale")
    return _affine(x, min_, scale_, 0)


__all__ = ["meanvar", "meanstd", "minmax", "scale", "inv_scale", "minmax_scale_params", "minmax_scale",
           "inv_minmax_scale", "remove_zeros_frames"]
