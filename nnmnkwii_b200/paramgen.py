"""Parameter generation (MLPG) -- drop-in for ``nnmnkwii.paramgen`` on an H100.

Same names, argument order, defaults, return types and error behaviour as the reference
(nnmnkwii/paramgen/_mlpg.py, ``__init__.py:1-17``):

    build_win_mats(windows, T)                          _mlpg.py:13-50
    mlpg(mean_frames, variance_frames, windows)         _mlpg.py:92-199
    mlpg_grad(mean_frames, variance_frames, windows, grad_output)   _mlpg.py:202-281
    full_window_mat(win_mats, T)                        _mlpg.py:284-294 (mlpg_helper.pyx:10-32)
    unit_variance_mlpg_matrix(windows, T)               _mlpg.py:297-373
    reshape_means(means, static_dim)                    _mlpg.py:376-405

All arithmetic runs in the sm_90a kernels of libnnk_b200 (csrc/nnk_mlpg.cu) through the C ABI in
include/nnk_b200.h.  NumPy inputs go through the host-buffer entry points (copies included); torch
CUDA tensors are used in place on the current stream and a CUDA tensor comes back.  There is no CPU
fallback: without the library / a GPU these functions raise.

Additive, batched entry points (the reference has none -- its notebooks loop over utterances and
streams in Python): :class:`StreamLayout`, :func:`merlin_layout`, :func:`mlpg_batch`.

Additive, parameter generation considering global variance (Toda, Black & Tokuda 2007, Sec. IV):
:func:`mlpg_gv`, :func:`mlpg_gv_batch` and the GV statistics :func:`global_variance`,
:func:`gv_statistics` (csrc/nnk_mlpg.cu ``nnk_mlpg_gv``, csrc/nnk_stats.cu ``nnk_segment_moments``).

Additive, parameter generation considering the modulation spectrum (DESIGN.md 3.18): :func:`mlpg_ms`,
:func:`mlpg_ms_batch` (csrc/nnk_ms_gen.cu ``nnk_mlpg_ms``; with ``segment=L`` ``nnk_mlpg_ms_segment``).

Additive, parameter generation from per-frame mixture outputs over all components (DESIGN.md 3.19):
:func:`mlpg_mixture`, :func:`mlpg_mixture_batch` (csrc/nnk_mix_gen.cu ``nnk_mix_gen``).

Additive, the log-likelihood of target trajectories under the trajectory model of the MLPG inputs (DESIGN.md
3.20): :func:`trajectory_log_likelihood`, :func:`trajectory_log_likelihood_batch` (csrc/nnk_mlpg.cu
``nnk_mlpg_traj_ll``).

Additive, samples from that trajectory model with counter-based noise (DESIGN.md 3.21): :func:`trajectory_sample`,
:func:`trajectory_sample_batch` (csrc/nnk_mlpg.cu ``nnk_mlpg_traj_sample``).

Additive, the gradient of :func:`mlpg_batch` in its means and its variances for minimum-generation-error training
(DESIGN.md 3.22): :func:`mlpg_vjp_batch` (csrc/nnk_mlpg.cu ``nnk_mlpg_vjp``).
"""
import ctypes

import numpy as np

from . import _lib
from .bandmat import BandMat

__all__ = [
    "mlpg_grad_batch",
    "build_win_mats", "mlpg", "mlpg_grad", "full_window_mat", "unit_variance_mlpg_matrix", "reshape_means",
    "StreamLayout", "merlin_layout", "mlpg_batch",
    "mlpg_gv", "mlpg_gv_batch", "global_variance", "gv_statistics",
    "mlpg_ms", "mlpg_ms_batch", "mlpg_mixture", "mlpg_mixture_batch",
    "trajectory_log_likelihood", "trajectory_log_likelihood_batch", "trajectory_sample", "trajectory_sample_batch",
    "mlpg_vjp_batch",
]


def build_win_mats(windows, T):
    """Builds a window matrix of a given size for each window in a collection (_mlpg.py:13-50).

    Returns a list of ``T x T`` Toeplitz :class:`~nnmnkwii_b200.bandmat.BandMat` (lower bandwidth
    ``l``, upper bandwidth ``u``, ``transposed=True`` exactly like the reference's
    ``bm.band_c_bm(u, l, win_coeffs).T``).  Host-side only: the kernels take the window
    coefficients directly and never build these matrices.
    """
    win_mats = []
    for ll, u, win_coeff in windows:
        assert ll >= 0 and u >= 0
        assert len(win_coeff) == ll + u + 1
        win_coeffs = np.tile(np.reshape(win_coeff, (ll + u + 1, 1)), T)
        win_mats.append(BandMat(u, ll, win_coeffs.copy()).T)
    return win_mats


def full_window_mat(win_mats, T):
    """Dense ``(T * num_windows, T)`` float64 stack of the window matrices (_mlpg.py:284-294)."""
    mat_full = np.zeros((T * len(win_mats), T))
    for win_index, win_mat in enumerate(win_mats):
        mat_full[win_index * T:(win_index + 1) * T, :] = win_mat.full()
    return mat_full


def reshape_means(means, static_dim):
    """Reshape means (``T x D``) to (``T*num_windows x static_dim``); no-op if already reshaped
    (_mlpg.py:376-405)."""
    T, D = means.shape
    if D == static_dim:
        return means
    from ._device import is_tensor
    if is_tensor(means):
        return means.reshape(T, -1, static_dim).transpose(0, 1).reshape(-1, static_dim)
    return means.reshape(T, -1, static_dim).transpose(1, 0, 2).reshape(-1, static_dim)


# ---------------------------------------------------------------------------------------------------
# layouts (additive)
# ---------------------------------------------------------------------------------------------------
class StreamLayout(object):
    """Where the streams of a ``(T, D)`` frame matrix live.

    ``streams`` is a list of ``(in_col, static_dim)`` for smoothed streams (window ``w`` of static
    dimension ``d`` is column ``in_col + w * static_dim + d``, as in the reference) or
    ``(in_col, static_dim, "copy")`` for columns that are passed through (e.g. Merlin's vuv flag).
    Output columns are assigned consecutively in the order given.
    """

    def __init__(self, D_in, streams):
        self.D_in = int(D_in)
        rows = []
        out_col = 0
        self.slices = []
        for s in streams:
            in_col, sd = int(s[0]), int(s[1])
            copy = len(s) > 2 and s[2] == "copy"
            for d in range(sd):
                rows.append((in_col + d, 0 if copy else sd, out_col + d, 1 if copy else 0))
            self.slices.append((out_col, out_col + sd))
            out_col += sd
        self.D_out = out_col
        self.chains = np.array(rows, dtype=_lib.CHAIN_DTYPE) if rows else np.zeros(0, dtype=_lib.CHAIN_DTYPE)
        self.n_chain = len(rows)

    @classmethod
    def single(cls, D, num_windows):
        """One stream occupying the whole matrix: ``static_dim = D // num_windows`` (_mlpg.py:172)."""
        return cls(D, [(0, D // num_windows)])


def merlin_layout():
    """The 187-column Merlin / slt_arctic acoustic layout of the gallery notebooks: mgc 180 (static
    60), lf0 3 (static 1), vuv 1 (copied), bap 3 (static 1) -> 63 output columns."""
    return StreamLayout(187, [(0, 60), (180, 1), (183, 1, "copy"), (184, 1)])


def _offsets_from(lengths=None, offsets=None, n_rows=None):
    if offsets is not None:
        off = np.asarray(offsets, dtype=np.int64)
    elif lengths is not None:
        off = np.concatenate([[0], np.cumsum(np.asarray(lengths, dtype=np.int64))])
    else:
        off = np.array([0, n_rows], dtype=np.int64)
    return np.ascontiguousarray(off)


def _utterance_table(lengths, offsets, n_rows, padded=None):
    """Host table of the utterances of a batch: ``(offsets, lengths, order, max_T, n_utt)`` with ``order``
    longest first.  ``padded=(B, Tmax)``: utterance b has ``lengths[b] <= Tmax`` frames from row
    ``b * Tmax``; otherwise ``lengths`` / ``offsets`` (default: one utterance) cover the ``n_rows`` rows
    back to back.  The kernels index rows, ``order`` and lengths from this table: it is checked here."""
    from ._device import is_tensor
    lengths, offsets = (a.cpu().numpy() if is_tensor(a) else a for a in (lengths, offsets))
    if padded:
        B, Tmax = padded
        lens = np.asarray(lengths, dtype=np.int64)
        assert len(lens) == B and lens.max(initial=0) <= Tmax
        off = np.arange(B + 1, dtype=np.int64) * Tmax
    else:
        off = _offsets_from(lengths, offsets, n_rows)
        assert off[0] == 0 and off[-1] == n_rows
        lens = np.diff(off)
    return off, lens, np.argsort(-lens, kind="stable").astype(np.int32), int(lens.max(initial=0)), len(lens)


def mlpg_batch(means, variances, windows, lengths=None, offsets=None, layout=None, check=True, out=None):
    """Batched MLPG over many utterances and streams in one call (additive API).

    Args:
        means: flat ``(sum_T, D)`` frame matrix holding the utterances back to back (give ``lengths``
            or ``offsets``), or a zero-padded ``(B, Tmax, D)`` batch (give ``lengths``).
            NumPy array (host path, copies included) or torch CUDA tensor (in place, current stream).
        variances: same shape as ``means`` (per-frame) or ``(D,)`` (global).
        windows: list of ``(l, u, coeff)`` triples shared by all smoothed streams.
        layout: :class:`StreamLayout`; default = one stream covering all columns.
        out: optional preallocated ``(sum_T, D_out)`` NumPy result buffer of the input dtype (flat
            host form only); pass page-locked memory to keep the device-to-host copy asynchronous.

    Returns:
        ``(sum_T, D_out)`` (or ``(B, Tmax, D_out)``) array / tensor of the input dtype.
    """
    from ._device import is_tensor, torch_dtype_code
    padded = means.ndim == 3
    D = means.shape[-1]
    if layout is None:
        layout = StreamLayout.single(D, len(windows))
    assert layout.D_in == D
    if padded:
        assert lengths is not None, "padded (B, Tmax, D) input needs lengths"
        B, Tmax = means.shape[0], means.shape[1]
    if is_tensor(means):
        return _mlpg_batch_device(means, variances, windows, lengths, offsets, layout, padded, check)

    dtype = means.dtype
    work_dtype = dtype if (dtype in (np.float32, np.float64) and np.asarray(variances).dtype == dtype) else np.float64
    m = np.ascontiguousarray(means, dtype=work_dtype)
    v = np.ascontiguousarray(variances, dtype=work_dtype)
    var1d = v.ndim == 1
    if var1d:
        assert v.shape[0] >= D
    else:
        assert m.shape == v.shape
    wc = _lib.make_windows(windows)
    if padded:
        # zero-padded batch: run on the flat view, one "utterance" per row block
        lens = _utterance_table(lengths, None, None, (B, Tmax))[1]
        keep = np.concatenate([np.arange(b * Tmax, b * Tmax + lens[b]) for b in range(B)]) if B else np.zeros(0, np.int64)
        flat_m = m.reshape(B * Tmax, D)[keep]
        flat_v = v if var1d else v.reshape(B * Tmax, D)[keep]
        y = mlpg_batch(flat_m, flat_v, windows, lengths=lens, layout=layout, check=check)
        out = np.zeros((B * Tmax, layout.D_out), dtype=dtype)
        out[keep] = y
        return out.reshape(B, Tmax, layout.D_out)
    n_rows = m.shape[0]
    off = _utterance_table(lengths, offsets, n_rows)[0]
    if out is not None and (out.shape != (n_rows, layout.D_out) or out.dtype != work_dtype or not out.flags.c_contiguous):
        raise ValueError("out must be a C-contiguous (%d, %d) array of dtype %s" % (n_rows, layout.D_out, work_dtype))
    if out is None:
        out = np.empty((n_rows, layout.D_out), dtype=work_dtype)
    st = _lib.NnkStatus()
    chains = np.ascontiguousarray(layout.chains)
    rc = _lib.lib.nnk_mlpg_batch_host(
        m.ctypes.data, v.ctypes.data, int(var1d), torch_dtype_code(work_dtype), n_rows, D, layout.D_out,
        off.ctypes.data, len(off) - 1, chains.ctypes.data, layout.n_chain, ctypes.byref(wc), out.ctypes.data,
        ctypes.byref(st))
    _lib.check(rc, "nnk_mlpg_batch_host")
    return out if out.dtype == dtype else out.astype(dtype)


def _mlpg_batch_device(means, variances, windows, lengths, offsets, layout, padded, check, gv=None):
    import torch

    from . import _device as dev

    dev.require_cuda()
    assert means.is_cuda, "torch inputs must be CUDA tensors (no CPU fallback)"
    n_rows = means.shape[0] * means.shape[1] if padded else means.shape[0]
    off, lens, order, max_T, n_utt = _utterance_table(lengths, offsets, n_rows, means.shape[:2] if padded else None)
    device = means.device
    dtype = means.dtype
    if dtype not in (torch.float32, torch.float64) or variances.dtype != dtype:
        work = torch.float64
    else:
        work = dtype
    m = means.to(work).contiguous()
    v = variances.to(device=device, dtype=work)
    var1d = v.dim() == 1
    D = m.shape[-1]
    if not var1d:
        v = v.expand_as(m).contiguous() if v.shape != m.shape else v.contiguous()
    else:
        v = v.contiguous()
    out = torch.zeros((n_rows, layout.D_out), dtype=work, device=device)
    if n_utt and max_T and layout.n_chain:
        if gv is not None:
            gv = (torch.from_numpy(gv[0]).to(device), torch.from_numpy(gv[1]).to(device)) + tuple(gv[2:])
        dev.run_mlpg(
            "fwd" if gv is None else "gv", means=m, variances=v, rhs=None, out=out,
            offsets=torch.from_numpy(off).to(device), lengths=dev.lengths_on(lens, device) if padded else None,
            order=torch.from_numpy(order).to(device), chains=dev.chains_on_device(layout.chains, device),
            n_chain=layout.n_chain, max_T=max_T, windows_c=_lib.make_windows(windows),
            in_ld=D, var_ld=0 if var1d else D, go_ld=0, out_ld=layout.D_out,
            dtype_code=dev.torch_dtype_code(work), go_f64=0, n_utt=n_utt, device=device, check=check, gv=gv)
    if padded:
        out = out.reshape(m.shape[0], m.shape[1], layout.D_out)
    return out if work == dtype else out.to(dtype)


# ---------------------------------------------------------------------------------------------------
# global variance (additive)
# ---------------------------------------------------------------------------------------------------
def _host_vector(x, name):
    from ._device import is_tensor
    if is_tensor(x):
        x = x.detach().cpu().numpy()
    try:
        return np.ascontiguousarray(np.asarray(x, dtype=np.float64).ravel())
    except (TypeError, ValueError):
        raise ValueError("%s must be a sequence of numbers" % name)


def _gv_args(gv_mean, gv_var, layout, n_iter, step, weight):
    """Checked GV parameters ``(gv_mean, gv_var, n_iter, step, weight)`` (float64 host vectors of
    ``layout.D_out`` entries; ``weight`` 0 = the default ``1 / (nw T)``).  Entries of copied columns
    are not used and not checked."""
    gm, gvv = _host_vector(gv_mean, "gv_mean"), _host_vector(gv_var, "gv_var")
    for name, a in (("gv_mean", gm), ("gv_var", gvv)):
        if a.shape != (layout.D_out,):
            raise ValueError("%s must have one entry per output column (%d), got %d" % (name, layout.D_out, a.size))
    used = layout.chains["out_col"][layout.chains["flags"] == 0]
    if not np.all(np.isfinite(gm[used])) or np.any(gm[used] < 0):
        raise ValueError("gv_mean must be finite and >= 0")
    if not np.all(np.isfinite(gvv[used]) & (gvv[used] > 0)):
        raise ValueError("gv_var must be finite and > 0")
    if isinstance(n_iter, bool) or int(n_iter) != n_iter or n_iter < 0:
        raise ValueError("n_iter must be an integer >= 0, got %r" % (n_iter,))
    if not (np.isfinite(step) and step > 0):
        raise ValueError("step must be finite and > 0, got %r" % (step,))
    if weight is not None and not (np.isfinite(weight) and weight > 0):
        raise ValueError("weight must be finite and > 0 (or None), got %r" % (weight,))
    gm, gvv = gm.copy(), gvv.copy()
    gm[np.setdiff1d(np.arange(layout.D_out), used)] = 0.0  # copied columns: never read
    gvv[np.setdiff1d(np.arange(layout.D_out), used)] = 1.0
    return gm, gvv, int(n_iter), float(step), 0.0 if weight is None else float(weight)


def mlpg_gv_batch(means, variances, windows, gv_mean, gv_var, lengths=None, offsets=None, layout=None, n_iter=20,
                  step=1.0, weight=None, check=True, out=None):
    r"""Batched parameter generation considering global variance (additive API).

    Per utterance and smoothed output column, starting from the :func:`mlpg_batch` trajectory
    :math:`c_m = P^{-1} b`, maximises

    .. math:: F(c) = \omega (b^T c - \tfrac12 c^T P c) - \tfrac{1}{2 \sigma^2} (v(c) - \mu)^2

    with :math:`v(c)` the population variance of :math:`c` over the utterance's frames (Toda, Black &
    Tokuda 2007, Sec. IV, diagonal GV covariance).  The start point rescales :math:`c_m` to variance
    :math:`\mu`; each of the ``n_iter`` trials takes the step ``alpha * ((c_m - c) + P^-1 g / omega)``
    (``g`` the gradient of the GV term) and keeps it when :math:`F` does not decrease, otherwise halves
    ``alpha`` (which starts at ``step``).  See DESIGN.md 3.15.

    Args:
        means, variances, windows, lengths, offsets, layout, check: as :func:`mlpg_batch` (flat or padded,
            per-frame or global ``(D,)`` variances, NumPy arrays or torch CUDA tensors).
        gv_mean, gv_var: target GV :math:`\mu` (``>= 0``) and its variance :math:`\sigma^2` (``> 0``), one
            entry per output column (``layout.D_out``), e.g. from :func:`gv_statistics`; copied columns
            (Merlin's vuv) ignore theirs.
        n_iter: trials (``>= 0``; 0 returns the rescaled start point).
        step: initial step ``alpha`` (``> 0``).
        weight: :math:`\omega` (``> 0``); default ``1 / (num_windows * T)`` per utterance.
        out: optional ``(sum_T, D_out)`` NumPy buffer of the working dtype (flat host form only).

    Returns:
        Trajectories shaped and typed like :func:`mlpg_batch`'s.  Arithmetic is float64.
    """
    import torch

    from . import _device as dev
    padded = means.ndim == 3
    D = means.shape[-1]
    if layout is None:
        layout = StreamLayout.single(D, len(windows))
    if layout.D_in != D:
        raise ValueError("layout covers %d input columns, means have %d" % (layout.D_in, D))
    if padded and lengths is None:
        raise ValueError("padded (B, Tmax, D) input needs lengths")
    gv = _gv_args(gv_mean, gv_var, layout, n_iter, step, weight)
    if dev.is_tensor(means):
        return _mlpg_batch_device(means, variances, windows, lengths, offsets, layout, padded, check, gv=gv)
    dtype = np.asarray(means).dtype
    v_np = np.asarray(variances)
    work = dtype if (dtype in (np.float32, np.float64) and v_np.dtype == dtype) else np.dtype(np.float64)
    dev.require_cuda()
    device = dev.cuda_device()
    m = torch.from_numpy(np.ascontiguousarray(means, dtype=work)).to(device)
    v = torch.from_numpy(np.ascontiguousarray(v_np, dtype=work)).to(device)
    y = _mlpg_batch_device(m, v, windows, lengths, offsets, layout, padded, check, gv=gv).cpu().numpy()
    if out is not None:
        if padded or out.shape != y.shape or out.dtype != work or not out.flags.c_contiguous:
            raise ValueError("out must be a C-contiguous %s array of dtype %s" % (y.shape, work))
        out[...] = y
        y = out
    return y if y.dtype == dtype else y.astype(dtype)


def mlpg_gv(mean_frames, variance_frames, windows, gv_mean, gv_var, n_iter=20, step=1.0, weight=None):
    """Parameter generation considering global variance for one utterance, ``(T, D) -> (T, static_dim)``:
    :func:`mlpg`'s arguments plus the GV parameters of :func:`mlpg_gv_batch` (``gv_mean`` / ``gv_var`` of
    length ``static_dim``).  NumPy in, NumPy out (a CUDA tensor stays a CUDA tensor)."""
    T, D = mean_frames.shape
    return mlpg_gv_batch(mean_frames, variance_frames, windows, gv_mean, gv_var, lengths=[T], n_iter=n_iter,
                         step=step, weight=weight)


def _moments(x, lengths, offsets, want_mean):
    """Per-utterance column mean (optional) and population variance on the device, float64 tensors
    ``(n_utt, D)``; ``(T, D)`` input is one utterance."""
    import torch

    from . import _device as dev
    shape = tuple(x.shape)
    if len(shape) == 3:
        if lengths is None:
            raise ValueError("padded (B, Tmax, D) input needs lengths")
        B, Tmax, D = shape
        lens = dev.check_lengths(lengths, B)
        if lens.size and int(lens.max()) > Tmax:
            raise ValueError("lengths exceed Tmax = %d" % Tmax)
        off = np.arange(B + 1, dtype=np.int64) * Tmax
    elif len(shape) == 2:
        n_rows, D = shape
        if offsets is not None:
            off = np.asarray(dev.check_lengths(offsets, len(offsets)), dtype=np.int64)
            if len(off) < 1 or off[0] != 0 or off[-1] != n_rows or np.any(np.diff(off) < 0):
                raise ValueError("offsets must rise from 0 to %d" % n_rows)
        elif lengths is not None:
            lens = dev.check_lengths(lengths, len(lengths))
            off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
            if off[-1] != n_rows:
                raise ValueError("lengths sum to %d, x has %d rows" % (off[-1], n_rows))
        else:
            off = np.array([0, n_rows], dtype=np.int64)
        lens = np.diff(off)
    else:
        raise ValueError("x must be (T, D), (sum_T, D) or (B, Tmax, D)")
    if lens.size and int(lens.min()) < 1:
        raise ValueError("every utterance needs at least one frame (a zero-length utterance has no variance)")
    dev.require_cuda()
    xt = dev.to_device(x)
    if xt.dtype not in (torch.float32, torch.float64):
        xt = xt.to(torch.float64)
    xt = xt.contiguous()
    n_utt = len(lens)
    device = xt.device
    var = torch.empty((n_utt, D), dtype=torch.float64, device=device)
    mean = torch.empty((n_utt, D), dtype=torch.float64, device=device) if want_mean else None
    if n_utt and D:
        off_t = torch.from_numpy(off).to(device)
        len_t = dev.lengths_on(lens, device)
        _lib.check(_lib.lib.nnk_segment_moments(
            xt.data_ptr(), dev.torch_dtype_code(xt.dtype), D, D, off_t.data_ptr(), len_t.data_ptr(), n_utt,
            mean.data_ptr() if want_mean else None, var.data_ptr(), dev.current_stream_ptr(device)),
            "nnk_segment_moments")
    return mean, var


def global_variance(x, lengths=None, offsets=None):
    """Global variance (per-utterance, per-column population variance over frames), float64.

    Args:
        x: ``(T, D)`` (one utterance), a padded ``(B, Tmax, D)`` batch with ``lengths``, or a flat
            ``(sum_T, D)`` batch with ``offsets`` (or ``lengths``).  NumPy array or torch tensor,
            float32 / float64 (accumulated in float64, two passes, fixed order).

    Returns:
        ``(D,)`` for ``(T, D)`` input without ``lengths`` / ``offsets``, otherwise ``(B, D)``; a NumPy
        array for NumPy input, a tensor on the input's device for a tensor.  A zero-length utterance
        raises ``ValueError``.
    """
    from . import _device as dev
    _, var = _moments(x, lengths, offsets, False)
    if x.ndim == 2 and lengths is None and offsets is None:
        var = var[0]
    return dev.like_input(var, x)


def gv_statistics(x, lengths=None, offsets=None):
    """``(gv_mean, gv_var)``: mean and population variance over utterances of :func:`global_variance`
    (same arguments), each ``(D,)`` float64 -- the GV model :func:`mlpg_gv_batch` takes."""
    from . import _device as dev
    _, gv = _moments(x, lengths, offsets, False)
    mean, var = _moments(gv, None, None, True)
    return dev.like_input(mean[0], x), dev.like_input(var[0], x)


# ---------------------------------------------------------------------------------------------------
# modulation spectrum (additive)
# ---------------------------------------------------------------------------------------------------
_MS_GEN_N = (256, 512, 1024, 2048, 4096)
_MS_SEG_N = (32, 64, 128, 256, 512)  # the segment level's DFT lengths (postfilters.SEGMENT_NS)


def _ms_args(ms_mean, ms_var, layout, n_iter, step, weight, segment=None):
    """Checked MS parameters ``(ms_mean, ms_var, n, n_iter, step, weight)``: float64 host ``(K, layout.D_out)``
    arrays (``weight`` 0 = the default ``1 / (nw T)``).  Columns of copied chains are not used and not checked;
    they are set to ``(0, inf)``.  With ``segment`` (the segment length L), n is one of the segment level's."""
    from ._device import is_tensor
    if segment is not None and (isinstance(segment, bool) or not isinstance(segment, (int, np.integer))):
        raise TypeError("segment must be an int (the segment length L) or None, got %s" % type(segment).__name__)
    arrs = []
    for name, a in (("ms_mean", ms_mean), ("ms_var", ms_var)):
        if is_tensor(a):
            a = a.detach().cpu().numpy()
        try:
            a = np.array(a, dtype=np.float64)
        except (TypeError, ValueError):
            raise ValueError("%s must be an array of numbers" % name)
        if a.ndim != 2 or a.shape[1] != layout.D_out:
            raise ValueError("%s must be (n // 2 + 1, %d), got shape %s" % (name, layout.D_out, a.shape))
        arrs.append(a)
    mm, mv = arrs
    if mm.shape != mv.shape:
        raise ValueError("ms_mean and ms_var differ in shape: %s, %s" % (mm.shape, mv.shape))
    n = 2 * (mm.shape[0] - 1)
    if segment is not None:
        if n not in _MS_SEG_N:
            raise ValueError("ms_mean / ms_var have %d bins: with segment, n = 2 (K - 1) = %d must be one of 32, 64, "
                             "128, 256, 512" % (mm.shape[0], n))
        if int(segment) % 2 or not 4 <= int(segment) <= n:
            raise ValueError("segment length must be even with 4 <= L <= n = %d, got %d" % (n, int(segment)))
    elif n not in _MS_GEN_N:
        raise ValueError("ms_mean / ms_var have %d bins: n = 2 (K - 1) = %d must be one of 256, 512, 1024, 2048, "
                         "4096" % (mm.shape[0], n))
    used = np.unique(layout.chains["out_col"][layout.chains["flags"] == 0])
    unused = np.setdiff1d(np.arange(layout.D_out), used)
    v, m = mv[:, used], mm[:, used]
    if np.any(np.isnan(v)) or np.any(v <= 0):
        raise ValueError("ms_var must be > 0 (inf exempts a bin), not NaN")
    if not np.all(np.isfinite(m[np.isfinite(v)])):
        raise ValueError("ms_mean must be finite where ms_var is finite")
    if isinstance(n_iter, bool) or int(n_iter) != n_iter or n_iter < 0:
        raise ValueError("n_iter must be an integer >= 0, got %r" % (n_iter,))
    if not (np.isfinite(step) and step > 0):
        raise ValueError("step must be finite and > 0, got %r" % (step,))
    if weight is not None and not (np.isfinite(weight) and weight > 0):
        raise ValueError("weight must be finite and > 0 (or None), got %r" % (weight,))
    mm[:, unused] = 0.0
    mv[:, unused] = np.inf
    return mm, mv, n, int(n_iter), float(step), 0.0 if weight is None else float(weight)


def _ms_lengths(means, lengths, offsets, padded):
    """Host frame counts of the utterances of a batch (argument errors as ``ValueError``)."""
    from . import _device as dev
    if padded:
        lens = dev.check_lengths(lengths, means.shape[0])
        if lens.size and int(lens.max()) > means.shape[1]:
            raise ValueError("lengths exceed Tmax = %d" % means.shape[1])
        return lens
    n_rows = means.shape[0]
    if offsets is not None:
        off = np.asarray(offsets.cpu().numpy() if dev.is_tensor(offsets) else offsets, dtype=np.int64)
        if off.ndim != 1 or len(off) < 1 or off[0] != 0 or off[-1] != n_rows or np.any(np.diff(off) < 0):
            raise ValueError("offsets must rise from 0 to %d" % n_rows)
        return np.diff(off)
    if lengths is not None:
        lens = dev.check_lengths(lengths, len(lengths))
        if int(lens.sum()) != n_rows:
            raise ValueError("lengths sum to %d, means have %d rows" % (lens.sum(), n_rows))
        return lens
    return np.array([n_rows], dtype=np.int64)


def mlpg_ms_batch(means, variances, windows, ms_mean, ms_var, lengths=None, offsets=None, layout=None, n_iter=20,
                  step=1.0, weight=None, check=True, out=None, segment=None):
    r"""Batched parameter generation considering the modulation spectrum (additive API).

    Per utterance and smoothed output column ``s``, with ``Y = rfft(c, n)`` and
    :math:`s_k(c) = \log \max(|Y_k|^2, \mathrm{tiny})` (what :func:`~nnmnkwii_b200.postfilters.modspec_statistics`
    averages), maximises

    .. math:: F(c) = \omega (b^T c - \tfrac12 c^T P c) - \tfrac12 \sum_{k=1}^{n/2} q_k (s_k(c) - \nu_k)^2,
              \quad \nu_k = \mathrm{ms\_mean}[k, s], \; q_k = 1 / \mathrm{ms\_var}[k, s]

    from the :func:`mlpg_batch` trajectory :math:`c_m = P^{-1} b`.  Each of the ``n_iter`` trials takes the
    step ``alpha * ((c_m - c) + P^-1 g / omega)`` (``g`` the gradient of the MS term) and keeps it when
    :math:`F` does not decrease, otherwise halves ``alpha`` (which starts at ``step``), so ``F`` never falls
    below :math:`F(c_m)` and ``n_iter = 0`` is plain MLPG.  Bin 0 has no term (the model sets the level); a bin
    with ``ms_var = inf`` has none either, which is how a column (e.g. the power coefficient) is left alone.
    This follows the idea of Takamichi et al. (ICASSP 2015) with the project's own step rule (DESIGN.md 3.18);
    nobody has measured the output quality at the default ``n_iter`` and ``step``.

    Args:
        means, variances, windows, lengths, offsets, layout, check: as :func:`mlpg_batch` (flat or padded,
            per-frame or global ``(D,)`` variances, NumPy arrays or torch CUDA tensors).
        ms_mean, ms_var: ``(K, layout.D_out)`` statistics of the log modulation spectrum, e.g.
            :func:`~nnmnkwii_b200.postfilters.modspec_statistics` of natural static trajectories; the DFT length
            ``n = 2 (K - 1)`` is 256, 512, 1024, 2048 or 4096 and at least every utterance's length.
            ``ms_var > 0`` (``inf`` exempts the bin); ``ms_mean`` finite where ``ms_var`` is.  Copied columns
            (Merlin's vuv) ignore theirs.
        n_iter: trials (``>= 0``).
        step: initial step ``alpha`` (``> 0``).
        weight: :math:`\omega` (``> 0``); default ``1 / (num_windows * T)`` per utterance.
        out: optional ``(sum_T, D_out)`` NumPy buffer of the working dtype (flat host form only).
        segment: ``None`` (the utterance level above) or the segment length ``L`` of the segment-level term:
            with hop ``H = L / 2``, a periodic Hann window ``w`` and the ``J = ceil(T / H) + 1`` segments of
            :func:`~nnmnkwii_b200.postfilters.modspec_statistics` ``(segment=L)`` (segment ``j`` starts at frame
            ``(j - 1) H``, frames outside the utterance are 0), the MS term becomes the mean over the segments,
            :math:`-\tfrac{1}{2J} \sum_j \sum_{k=1}^{n/2} q_k (s_{j,k}(c) - \nu_k)^2` with
            :math:`s_{j,k}` the log power of ``rfft(w * c[segment j], n)``.  ``ms_mean`` / ``ms_var`` are then
            ``(n // 2 + 1, D_out)`` statistics with ``n`` 32, 64, 128, 256 or 512, e.g.
            ``modspec_statistics(natural_static, n=n, segment=L)``; ``L`` is even with ``4 <= L <= n``, and
            utterances may have any length.  Nobody has measured the output quality of this variant at the
            default ``n_iter`` and ``step`` either.

    Returns:
        Trajectories shaped and typed like :func:`mlpg_batch`'s.  Arithmetic is float64 (float32 inputs are
        widened once on the device).  Every argument error is raised before any launch: a ``segment`` that is
        not an int is a ``TypeError``, every other one a ``ValueError``.
    """
    import torch

    from . import _device as dev
    if means.ndim not in (2, 3):
        raise ValueError("means must be (sum_T, D) or (B, Tmax, D)")
    padded = means.ndim == 3
    D = means.shape[-1]
    if layout is None:
        layout = StreamLayout.single(D, len(windows))
    if layout.D_in != D:
        raise ValueError("layout covers %d input columns, means have %d" % (layout.D_in, D))
    if padded and lengths is None:
        raise ValueError("padded (B, Tmax, D) input needs lengths")
    ms = _ms_args(ms_mean, ms_var, layout, n_iter, step, weight, segment)
    lens = _ms_lengths(means, lengths, offsets, padded)
    if segment is None and lens.size and int(lens.max()) > ms[2]:
        raise ValueError("an utterance of %d frames is longer than the DFT length n = %d" % (lens.max(), ms[2]))
    L = None if segment is None else int(segment)
    if dev.is_tensor(means):
        return _mlpg_ms_device(means, variances, windows, lengths, offsets, layout, padded, check, ms, L)
    dtype = np.asarray(means).dtype
    v_np = np.asarray(variances)
    work = dtype if (dtype in (np.float32, np.float64) and v_np.dtype == dtype) else np.dtype(np.float64)
    dev.require_cuda()
    device = dev.cuda_device()
    m = torch.from_numpy(np.ascontiguousarray(means, dtype=work)).to(device)
    v = torch.from_numpy(np.ascontiguousarray(v_np, dtype=work)).to(device)
    y = _mlpg_ms_device(m, v, windows, lengths, offsets, layout, padded, check, ms, L).cpu().numpy()
    if out is not None:
        if padded or out.shape != y.shape or out.dtype != work or not out.flags.c_contiguous:
            raise ValueError("out must be a C-contiguous %s array of dtype %s" % (y.shape, work))
        out[...] = y
        y = out
    return y if y.dtype == dtype else y.astype(dtype)


def _mlpg_ms_device(means, variances, windows, lengths, offsets, layout, padded, check, ms, L=None):
    import torch

    from . import _device as dev

    dev.require_cuda()
    assert means.is_cuda, "torch inputs must be CUDA tensors (no CPU fallback)"
    dev.poll_errors()
    n_rows = means.shape[0] * means.shape[1] if padded else means.shape[0]
    off, lens, order, max_T, n_utt = _utterance_table(lengths, offsets, n_rows, means.shape[:2] if padded else None)
    device = means.device
    dtype = means.dtype
    m = means.to(torch.float64).contiguous()  # float32 inputs are widened once; all arithmetic is float64
    v = variances.to(device=device, dtype=torch.float64)
    var1d = v.dim() == 1
    D = m.shape[-1]
    v = v.contiguous() if var1d else (v.expand_as(m).contiguous() if v.shape != m.shape else v.contiguous())
    out = torch.zeros((n_rows, layout.D_out), dtype=torch.float64, device=device)
    if n_utt and max_T and layout.n_chain:
        wc = _lib.make_windows(windows)
        need = _lib.lib.nnk_mlpg_ms_workspace_bytes(n_utt, layout.n_chain, max_T, n_rows, layout.D_out,
                                                    ctypes.byref(wc))
        if need == 0:
            raise NotImplementedError("window set not supported by the CUDA kernels")
        ws = dev.workspace(device, need)
        status = torch.zeros(1, dtype=torch.int64, device=device)
        offsets_d = torch.from_numpy(off).to(device)
        lengths_d = dev.lengths_on(lens, device) if padded else None
        order_d = torch.from_numpy(order).to(device)
        chains_d = dev.chains_on_device(layout.chains, device)
        mean_d = torch.from_numpy(np.ascontiguousarray(ms[0])).to(device)
        var_d = torch.from_numpy(np.ascontiguousarray(ms[1])).to(device)
        a = _lib.NnkMlpgArgs()
        a.means, a.vars, a.grad_out, a.out = m.data_ptr(), v.data_ptr(), None, out.data_ptr()
        a.dtype, a.n_utt = _lib.NNK_F64, n_utt
        a.in_ld, a.var_ld, a.go_ld, a.out_ld = D, 0 if var1d else D, 0, layout.D_out
        a.utt_off, a.utt_len, a.order = offsets_d.data_ptr(), lengths_d.data_ptr() if padded else None, order_d.data_ptr()
        a.chains, a.n_chain, a.max_T, a.go_f64, a.win = chains_d.data_ptr(), layout.n_chain, max_T, 0, wc
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
        a.status_word, a.out_off = status.data_ptr(), None
        p = _lib.NnkMlpgMs()
        p.ms_mean, p.ms_var, p.n, p.n_iter, p.step, p.weight = (mean_d.data_ptr(), var_d.data_ptr(), ms[2], ms[3],
                                                                ms[4], ms[5])
        p.n_rows = n_rows
        if L is None:
            _lib.check(_lib.lib.nnk_mlpg_ms(ctypes.byref(a), ctypes.byref(p), dev.current_stream_ptr(device)),
                       "nnk_mlpg_ms")
        else:
            _lib.check(_lib.lib.nnk_mlpg_ms_segment(ctypes.byref(a), ctypes.byref(p), L,
                                                    dev.current_stream_ptr(device)), "nnk_mlpg_ms_segment")
        if check == "deferred":
            dev._defer_check(status, device)
        elif check:
            dev.raise_if_failed(status)
    if padded:
        out = out.reshape(m.shape[0], m.shape[1], layout.D_out)
    return out if dtype == torch.float64 else out.to(dtype)


def mlpg_ms(mean_frames, variance_frames, windows, ms_mean, ms_var, n_iter=20, step=1.0, weight=None,
            segment=None):
    """Parameter generation considering the modulation spectrum for one utterance, ``(T, D) -> (T, static_dim)``:
    :func:`mlpg`'s arguments plus the MS parameters of :func:`mlpg_ms_batch` (``ms_mean`` / ``ms_var`` of shape
    ``(n // 2 + 1, static_dim)``; ``segment=L`` for the segment-level term).  NumPy in, NumPy out (a CUDA tensor
    stays a CUDA tensor)."""
    T, D = mean_frames.shape
    return mlpg_ms_batch(mean_frames, variance_frames, windows, ms_mean, ms_var, lengths=[T], n_iter=n_iter,
                         step=step, weight=weight, segment=segment)


# ---------------------------------------------------------------------------------------------------
# mixture outputs (additive)
# ---------------------------------------------------------------------------------------------------
_MIX_DATA_ERRORS = {1: "a NaN or +inf log-weight", 2: "every log-weight is -inf",
                    3: "a variance that is not positive and finite"}


def _mix_column_map(layout, nw):
    """int32 ``(D_in,)`` column map of nnk_mix_gen (include/nnk_b200.h): ``-1`` for a column no chain reads,
    ``out_col << 3`` for a copied column, ``(out_col << 3) | (w + 1)`` for window ``w`` of a smoothed one."""
    cmap = np.full(layout.D_in, -1, dtype=np.int32)
    for in_col, stride, out_col, flags in layout.chains.tolist():
        for w in range(1 if flags & 1 else nw):
            col = in_col + w * stride
            if not 0 <= col < layout.D_in or cmap[col] != -1:
                raise ValueError("layout: column %d is outside the %d input columns or read by two chains"
                                 % (col, layout.D_in))
            cmap[col] = (out_col << 3) | (0 if flags & 1 else w + 1)
    return cmap


def _mix_check(log_weights, means, variances, windows, lengths, offsets, layout, n_iter):
    """Checked arguments of :func:`mlpg_mixture_batch`, all raised before any launch:
    ``(padded, lens, layout, column map, n_iter, arrays)``."""
    from . import _device as dev
    if isinstance(n_iter, (bool, np.bool_)) or not isinstance(n_iter, (int, np.integer)) or n_iter < 0:
        raise ValueError("n_iter must be an integer >= 0, got %r" % (n_iter,))
    arrs = (log_weights, means, variances)
    tensors = [dev.is_tensor(a) for a in arrs]
    if any(tensors) and not all(tensors):
        raise ValueError("log_weights, means and variances must all be CUDA tensors or all NumPy arrays")
    if all(tensors):
        if not all(a.is_cuda for a in arrs):
            raise ValueError("torch inputs must be CUDA tensors (no CPU fallback)")
    else:
        arrs = tuple(np.asarray(a) for a in arrs)
    for name, a in zip(("log_weights", "means", "variances"), arrs):
        if dev.np_dtype(a) not in (np.float32, np.float64):
            raise ValueError("%s must be float32 or float64, got %s" % (name, dev.np_dtype(a)))
    means = arrs[1]
    if means.ndim not in (3, 4):
        raise ValueError("means must be (sum_T, M, D) or (B, Tmax, M, D), got shape %s" % (tuple(means.shape),))
    if tuple(arrs[2].shape) != tuple(means.shape):
        raise ValueError("variances must have the shape of means %s, got %s" % (tuple(means.shape),
                                                                                 tuple(arrs[2].shape)))
    if tuple(arrs[0].shape) != tuple(means.shape[:-1]):
        raise ValueError("log_weights must be %s, got %s" % (tuple(means.shape[:-1]), tuple(arrs[0].shape)))
    padded = means.ndim == 4
    M, D = int(means.shape[-2]), int(means.shape[-1])
    if not 1 <= M <= _lib.NNK_MIX_GEN_MAX_M:
        raise ValueError("mlpg_mixture supports 1 .. %d components, got %d" % (_lib.NNK_MIX_GEN_MAX_M, M))
    if not 1 <= D <= _lib.NNK_MIX_GEN_MAX_D:
        raise ValueError("mlpg_mixture supports 1 .. %d columns, got %d" % (_lib.NNK_MIX_GEN_MAX_D, D))
    if not windows:
        raise ValueError("windows must not be empty")
    _lib.make_windows(windows)
    if layout is None:
        layout = StreamLayout.single(D, len(windows))
    if layout.D_in != D:
        raise ValueError("layout covers %d input columns, means have %d" % (layout.D_in, D))
    if padded and lengths is None:
        raise ValueError("padded (B, Tmax, M, D) input needs lengths")
    lens = _ms_lengths(means, lengths, offsets, padded)
    return padded, lens, layout, _mix_column_map(layout, len(windows)), int(n_iter), arrs


def mlpg_mixture_batch(log_weights, means, variances, windows, lengths=None, offsets=None, layout=None, n_iter=5,
                       return_log_likelihood=False):
    r"""Batched parameter generation from per-frame Gaussian mixtures, over all components (additive API).

    Frame ``t`` has ``M`` diagonal Gaussian components with log-weights ``lw[t, m]``, means ``mu[t, m]`` and
    variances ``s2[t, m]`` in the column layout of :func:`mlpg_batch`'s ``(T, D)`` rows, e.g. the output of a
    mixture density network.  With ``Y = W c`` the static and dynamic sequence of trajectory ``c`` (windows
    never cross an utterance), the trajectory maximises

    .. math:: L(c) = \sum_t \log \sum_m \exp(lw_{t,m} + \log N(Y_t; \mu_{t,m}, \mathrm{diag}\,\sigma^2_{t,m}))

    over the columns that count at ``t``: on the first and last ``H = max(l, u)`` frames of an utterance (every
    frame when ``H = 0``) only the static and copied columns, as :func:`mlpg` gives the dynamic windows zero
    precision there; elsewhere every column a chain reads.  EM (Tokuda et al., ICASSP 2000): ``c_0`` is
    :func:`mlpg_batch` of each frame's most probable component (the lowest index on ties, as ``np.argmax``); each
    iteration takes the posteriors ``gamma[t, m]`` of the current trajectory and solves with precisions
    ``P_t = sum_m gamma / s2`` and means ``(sum_m gamma mu / s2) / P_t``, so ``L`` never decreases.  See
    DESIGN.md 3.19.  Nobody has measured whether the result sounds better than the most-probable collapse.

    Args:
        log_weights: flat ``(sum_T, M)`` or padded ``(B, Tmax, M)``; need not be normalised, may be ``-inf``
            (a log-softmax output goes in as it is).
        means, variances: flat ``(sum_T, M, D)`` or padded ``(B, Tmax, M, D)``; ``variances`` positive and
            finite wherever a chain reads.  The three are CUDA tensors or NumPy arrays, float32 or float64.
        windows, lengths, offsets, layout: as :func:`mlpg_batch` (``merlin_layout()`` included: a copied column
            counts like a static one).
        n_iter: EM iterations (``>= 0``); 0 returns :func:`mlpg_batch` of the most probable components.
        return_log_likelihood: also return ``L(c_0) .. L(c_n_iter)`` per utterance.

    Returns:
        The trajectories, flat ``(sum_T, D_out)`` or padded ``(B, Tmax, D_out)`` with zero rows beyond each
        length, of the form and dtype of ``means`` (computed in float64; a float32 result is the float64 result of
        the widened inputs, rounded); with ``return_log_likelihood`` also an ``(n_utt, n_iter + 1)`` float64 NumPy
        array.  Argument errors (shapes, dtypes, more than 64 components or 256 columns, ``n_iter``) raise
        ``ValueError`` before any launch.  A data error (a NaN or ``+inf`` log-weight, a frame whose log-weights
        are all ``-inf``, a variance that is not positive and finite) is found on the device and raises
        ``ValueError`` when the result comes back.
    """
    import torch

    from . import _device as dev
    padded, lens, layout, cmap, n_iter, arrs = _mix_check(log_weights, means, variances, windows, lengths, offsets,
                                                          layout, n_iter)
    on_device = dev.is_tensor(arrs[1])
    if not on_device:
        dev.require_cuda()
        device = dev.cuda_device()
        arrs = tuple(torch.from_numpy(np.ascontiguousarray(a)).to(device) for a in arrs)
    y, L = _mlpg_mixture_device(*arrs, windows, lens, layout, cmap, padded, n_iter, return_log_likelihood)
    if y.dtype != arrs[1].dtype:
        y = y.to(arrs[1].dtype)
    if not on_device:
        y = y.cpu().numpy()
    return (y, L) if return_log_likelihood else y


def _mlpg_mixture_device(lw, mu, s2, windows, lens, layout, cmap, padded, n_iter, want_ll):
    """The device part of :func:`mlpg_mixture_batch` on checked CUDA tensors: float64 ``(y, L or None)``."""
    import math

    import torch

    from . import _device as dev
    device = mu.device
    dev.poll_errors()
    if not (lw.dtype == mu.dtype == s2.dtype):
        lw, mu, s2 = (a.to(torch.float64) for a in (lw, mu, s2))
    lw, mu, s2 = (a.contiguous() for a in (lw, mu, s2))
    M, D = mu.shape[-2], mu.shape[-1]
    n_rows = mu.shape[0] * mu.shape[1] if padded else mu.shape[0]
    n_utt = len(lens)
    off = (np.arange(n_utt + 1, dtype=np.int64) * mu.shape[1] if padded
           else np.concatenate([[0], np.cumsum(lens)]).astype(np.int64))
    y = torch.zeros((n_rows, layout.D_out), dtype=torch.float64, device=device)
    L = np.zeros((n_utt, n_iter + 1)) if want_ll else None
    if not (n_utt and int(lens.max(initial=0)) and layout.n_chain):
        return (y.reshape(mu.shape[0], mu.shape[1], layout.D_out) if padded else y), L
    order = np.argsort(-lens, kind="stable").astype(np.int32)
    max_T = int(lens.max())
    tiles = -(-lens // _lib.NNK_MIX_GEN_TILE)
    tile_off = np.concatenate([[0], np.cumsum(tiles)]).astype(np.int32)
    n_tiles = int(tile_off[-1])

    def up(a):  # asynchronous upload: nothing below waits for the device until the results come back
        return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(device, non_blocking=True)
    tables = up(np.concatenate([off[:-1].astype(np.int32), lens.astype(np.int32), tile_off, order, cmap]))
    utt_off_d, len_d = tables[:n_utt], tables[n_utt:2 * n_utt]
    tile_d, order_d = tables[2 * n_utt:3 * n_utt + 1], tables[3 * n_utt + 1:4 * n_utt + 1]
    cmap_d = tables[4 * n_utt + 1:]
    offsets_d = up(off)
    chains = dev.chains_on_device(layout.chains, device)
    win = _lib.make_windows(windows)
    status = torch.zeros(2, dtype=torch.int64, device=device)  # [0] the solves' pivots, [1] the data errors

    def solve(E, V):  # the kernels and arguments of mlpg_batch(E, V, windows, lengths, layout=layout)
        out = torch.zeros((n_rows, layout.D_out), dtype=torch.float64, device=device)
        dev.run_mlpg("fwd", means=E, variances=V, rhs=None, out=out, offsets=offsets_d,
                     lengths=len_d if padded else None, order=order_d, chains=chains, n_chain=layout.n_chain,
                     max_T=max_T, windows_c=win, in_ld=D, var_ld=D, go_ld=0, out_ld=layout.D_out,
                     dtype_code=_lib.NNK_F64, go_f64=0, n_utt=n_utt, device=device, check=False, status=status[0:1])
        return out

    E = torch.empty((n_rows, D), dtype=torch.float64, device=device)
    V = torch.empty((n_rows, D), dtype=torch.float64, device=device)
    lnorm = torch.empty((n_rows, M), dtype=torch.float64, device=device)
    ll = torch.zeros((n_iter + 1, n_tiles), dtype=torch.float64, device=device) if want_ll else None
    a = _lib.NnkMixGenArgs()
    a.log_weights, a.means, a.vars = lw.data_ptr(), mu.data_ptr(), s2.data_ptr()
    a.dtype, a.M, a.D, a.n_utt = dev.torch_dtype_code(mu.dtype), M, D, n_utt
    a.utt_off, a.utt_len, a.tile_off, a.n_tiles = utt_off_d.data_ptr(), len_d.data_ptr(), tile_d.data_ptr(), n_tiles
    a.col_map, a.win = cmap_d.data_ptr(), win
    a.c_ld, a.c_cols = layout.D_out, layout.D_out
    a.lnorm, a.E, a.V = lnorm.data_ptr(), E.data_ptr(), V.data_ptr()
    a.status_word = status[1:2].data_ptr()
    stream = dev.current_stream_ptr(device)

    def launch(mode, c, k):
        a.mode = mode
        a.c = c.data_ptr() if c is not None else None
        a.ll_part = ll[k].data_ptr() if (want_ll and mode != _lib.NNK_MIX_GEN_SELECT) else None
        _lib.check(_lib.lib.nnk_mix_gen(ctypes.byref(a), stream), "nnk_mix_gen")

    launch(_lib.NNK_MIX_GEN_SELECT, None, 0)
    y = solve(E, V)
    for k in range(n_iter):
        launch(_lib.NNK_MIX_GEN_ESTEP, y, k)
        y = solve(E, V)
    if want_ll:
        launch(_lib.NNK_MIX_GEN_OBJECTIVE, y, n_iter)
    # the one host synchronisation: status words and objective partials come back together
    host_status = torch.empty(2, dtype=torch.int64).pin_memory()
    host_status.copy_(status, non_blocking=True)
    if want_ll:
        host_ll = torch.empty(ll.shape, dtype=torch.float64).pin_memory()
        host_ll.copy_(ll, non_blocking=True)
    torch.cuda.current_stream(device).synchronize()
    word = int(host_status[1]) & 0xFFFFFFFFFFFFFFFF
    if word:
        key = ~word & 0xFFFFFFFFFFFFFFFF
        row, kind = key >> 2, key & 3
        u = int(np.searchsorted(off, row, side="right")) - 1
        raise ValueError("mlpg_mixture: %s at frame %d of utterance %d" % (_MIX_DATA_ERRORS[kind], row - off[u], u))
    dev._raise_word(int(host_status[0]))
    if want_ll:
        parts = host_ll.numpy()
        L = np.array([[math.fsum(parts[k, tile_off[u]:tile_off[u + 1]]) for k in range(n_iter + 1)]
                      for u in range(n_utt)])
    if padded:
        y = y.reshape(mu.shape[0], mu.shape[1], layout.D_out)
    return y, L


def mlpg_mixture(log_weights, means, variances, windows, n_iter=5, return_log_likelihood=False):
    """Parameter generation from per-frame mixtures for one utterance: ``log_weights (T, M)``, ``means`` and
    ``variances (T, M, D)`` -> ``(T, static_dim)``, see :func:`mlpg_mixture_batch`.  With
    ``return_log_likelihood`` also ``L(c_0) .. L(c_n_iter)``, ``(n_iter + 1,)`` float64.  NumPy in, NumPy out (a
    CUDA tensor stays a CUDA tensor)."""
    if len(means.shape) != 3:
        raise ValueError("means must be (T, M, D), got shape %s" % (tuple(means.shape),))
    out = mlpg_mixture_batch(log_weights, means, variances, windows, lengths=[means.shape[0]], n_iter=n_iter,
                             return_log_likelihood=return_log_likelihood)
    return (out[0], out[1][0]) if return_log_likelihood else out


# ---------------------------------------------------------------------------------------------------
# reference signatures
# ---------------------------------------------------------------------------------------------------
def mlpg(mean_frames, variance_frames, windows):
    r"""Maximum Likelihood Parameter Generation, ``f: (T, D) -> (T, static_dim)`` (_mlpg.py:92-199).

    .. math:: y = (\sum_l W_l^T P_l W_l)^{-1} \sum_l W_l^T P_l \mu_l

    Args:
        mean_frames (2darray): means, static + dynamic features, ``(T, D)``.
        variance_frames (2d or 1darray): per-frame ``(T, D)`` or global ``(D,)`` variances.
        windows (list): ``(l, u, win_coeff)`` triples.

    Returns:
        Generated static features ``(T, D // len(windows))`` in the dtype of ``mean_frames``.
    """
    from ._device import is_tensor, torch_dtype_code
    if is_tensor(mean_frames):
        T, D = mean_frames.shape
        if variance_frames.dim() == 1 and variance_frames.shape[0] == D:
            pass
        else:
            assert mean_frames.shape == variance_frames.shape
        return mlpg_batch(mean_frames, variance_frames, windows, lengths=[T])
    mean_frames = np.asarray(mean_frames)
    variance_frames = np.asarray(variance_frames)
    dtype = mean_frames.dtype
    T, D = mean_frames.shape
    var1d = variance_frames.ndim == 1 and variance_frames.shape[0] == D
    if not var1d:
        assert mean_frames.shape == variance_frames.shape
    work_dtype = dtype if (dtype in (np.float32, np.float64) and variance_frames.dtype == dtype) else np.float64
    m = np.ascontiguousarray(mean_frames, dtype=work_dtype)
    v = np.ascontiguousarray(variance_frames, dtype=work_dtype)
    wc = _lib.make_windows(windows)
    static_dim = D // len(windows)
    y = np.zeros((T, static_dim), dtype=work_dtype)
    bad = ctypes.c_int32(0)
    rc = _lib.lib.nnk_mlpg_host(m.ctypes.data, v.ctypes.data, int(var1d), torch_dtype_code(work_dtype),
                                T, D, ctypes.byref(wc), y.ctypes.data, ctypes.byref(bad))
    _lib.check(rc, "nnk_mlpg_host")
    return y if y.dtype == dtype else y.astype(dtype)


def mlpg_grad(mean_frames, variance_frames, windows, grad_output, check=True):
    r"""MLPG gradient (_mlpg.py:202-281): returns ``(T, D)`` float32,

    .. math:: g_{d,l} = P_{d,l} \, W_l (\sum_l W_l^T P_{d,l} W_l)^{-1} o_d

    evaluated as one banded solve + one stencil per static dimension (the reference solves a
    dense ``T x T`` right-hand side per (dimension, window)).
    """
    import torch

    from . import _device as dev

    dev.require_cuda()
    device = dev.cuda_device(mean_frames)
    T, D = mean_frames.shape
    v = dev.to_device(variance_frames, device).to(device)
    if v.dtype not in (torch.float32, torch.float64):
        v = v.to(torch.float64)
    if v.dim() == 2 and v.shape[0] > 1 and v.stride(0) == 0:
        v = v[0]  # v.expand(T, D) of a global variance (tests/test_autograd.py:191): keep it 1-D
    var1d = v.dim() == 1
    v = v.contiguous()
    go = dev.to_device(grad_output, device).to(device)
    if go.dtype not in (torch.float32, torch.float64):
        go = go.to(torch.float32)
    go = go.contiguous()
    nw = len(windows)
    static_dim = D // nw
    out = torch.zeros((T, D), dtype=torch.float32, device=device)
    if T and static_dim:
        chains = dev.simple_chains(static_dim)
        dev.run_mlpg(
            "grad", means=None, variances=v, rhs=go, out=out,
            offsets=torch.tensor([0, T], dtype=torch.int64, device=device), lengths=None, order=None,
            chains=dev.chains_on_device(chains, device), n_chain=static_dim, max_T=T,
            windows_c=_lib.make_windows(windows), in_ld=D, var_ld=0 if var1d else D, go_ld=go.shape[1], out_ld=D,
            dtype_code=dev.torch_dtype_code(v.dtype), go_f64=int(go.dtype == torch.float64), n_utt=1,
            device=device, check=check)
    return out if dev.is_tensor(mean_frames) else out.cpu().numpy()


def mlpg_grad_batch(variances, windows, grad_output, lengths, layout=None, check=True):
    """Batched :func:`mlpg_grad` on the device (additive API): the gradients of
    ``mlpg_batch(means, variances, windows, lengths, layout=layout)`` with respect to ``means`` for
    every utterance of the batch in ONE launch of ``nnk_mlpg_grad``.

    Args:
        variances: CUDA tensor, flat ``(sum_T, D)`` / padded ``(B, Tmax, D)`` per-frame variances,
            or ``(D,)`` global.
        grad_output: CUDA tensor ``(sum_T, D_out)`` / ``(B, Tmax, D_out)``, the gradient with respect
            to the generated trajectories.
        lengths: frames per utterance.

    Returns:
        float32 CUDA tensor shaped like the means (``(sum_T, D)`` or ``(B, Tmax, D)``); rows beyond
        an utterance's length (padded form) are zero.
    """
    import torch

    from . import _device as dev

    dev.require_cuda()
    assert dev.is_tensor(grad_output) and grad_output.is_cuda, "device tensors only (no CPU fallback)"
    device = grad_output.device
    padded = grad_output.dim() == 3
    go = grad_output.detach()
    if go.dtype not in (torch.float32, torch.float64):
        go = go.to(torch.float32)
    go = go.contiguous()
    v = variances.detach().to(device)
    if v.dtype not in (torch.float32, torch.float64):
        v = v.to(torch.float64)
    var1d = v.dim() == 1
    D = v.shape[-1]
    if layout is None:
        layout = StreamLayout.single(D, len(windows))
    assert layout.D_in == D and go.shape[-1] == layout.D_out
    n_rows = go.shape[0] * go.shape[1] if padded else go.shape[0]
    off, lens, order, max_T, n_utt = _utterance_table(lengths, None, n_rows, go.shape[:2] if padded else None)
    if not var1d:
        v = v.expand(*go.shape[:-1], D)
    v = v.contiguous()  # materialises stride-0 expanded variances
    out = torch.zeros((n_rows, D), dtype=torch.float32, device=device)
    if n_utt and max_T and layout.n_chain:
        # the gradient kernel indexes grad_output by chain: chain c reads column c, so route the
        # layout's output columns to chain order (identity for a single stream)
        out_cols = torch.from_numpy(layout.chains["out_col"].astype(np.int64)).to(device)
        go2 = go.reshape(n_rows, layout.D_out)
        if not np.array_equal(layout.chains["out_col"], np.arange(layout.n_chain)):
            go2 = go2.index_select(1, out_cols).contiguous()
        dev.run_mlpg(
            "grad", means=None, variances=v, rhs=go2, out=out,
            offsets=torch.from_numpy(off).to(device), lengths=dev.lengths_on(lens, device) if padded else None,
            order=torch.from_numpy(order).to(device),
            chains=dev.chains_on_device(layout.chains, device), n_chain=layout.n_chain, max_T=max_T,
            windows_c=_lib.make_windows(windows), in_ld=D, var_ld=0 if var1d else D, go_ld=layout.n_chain, out_ld=D,
            dtype_code=dev.torch_dtype_code(v.dtype), go_f64=int(go2.dtype == torch.float64), n_utt=n_utt,
            device=device, check=check)
    return out.reshape(go.shape[0], go.shape[1], D) if padded else out


def unit_variance_mlpg_matrix(windows, T):
    r"""MLPG matrix for unit-variance inputs, ``R = (W^T W)^{-1} W^T`` with the reference's edge
    rule for dynamic windows; ``(T, num_windows * T)`` float32 (_mlpg.py:297-373).

    Built on the GPU as ``num_windows * T`` banded solves (one chain per column of
    :math:`\tilde W^T`) instead of the reference's dense ``O(T^2)`` banded inverse followed by a
    dense ``(T x T)(T x 3T)`` product.
    """
    import torch

    from . import _device as dev

    dev.require_cuda()
    device = dev.cuda_device()
    nw = len(windows)
    win_mats = build_win_mats(windows, T)
    max_win_width = int(np.max([max(w.l, w.u) for w in win_mats]))
    # right-hand sides = columns of Wtilde^T: row r of window w, edge rows of dynamic windows zeroed
    mask = np.zeros(T)
    if max_win_width > 0:  # precisions.data[:, m:-m] += 1.0 (_mlpg.py:354); m == 0 -> empty slice
        mask[max_win_width:T - max_win_width] = 1.0
    rhs = np.zeros((T, nw * T))
    for w, (l, u, c) in enumerate(windows):
        c = np.asarray(c, dtype=np.float64)
        rows = np.arange(T)
        scale = np.ones(T) if w == 0 else mask
        for k in range(-l, u + 1):
            cols = rows + k
            ok = (cols >= 0) & (cols < T)
            rhs[cols[ok], w * T + rows[ok]] = scale[ok] * c[l + k]
    n_chain = nw * T
    chains = np.zeros(n_chain, dtype=_lib.CHAIN_DTYPE)  # in_col = win_stride = 0: all read variance[0] == 1
    chains["out_col"] = np.arange(n_chain)
    out = torch.zeros((T, n_chain), dtype=torch.float64, device=device)
    if T:
        dev.run_mlpg(
            "solve", means=None, variances=torch.ones(max(1, nw), dtype=torch.float64, device=device),
            rhs=torch.from_numpy(rhs).to(device), out=out,
            offsets=torch.tensor([0, T], dtype=torch.int64, device=device), lengths=None, order=None,
            chains=dev.chains_on_device(chains, device), n_chain=n_chain, max_T=T,
            windows_c=_lib.make_windows(windows), in_ld=1, var_ld=0, go_ld=n_chain, out_ld=n_chain,
            dtype_code=_lib.NNK_F64, go_f64=1, n_utt=1, device=device, check=True)
    return out.to(torch.float32).cpu().numpy()


# ---------------------------------------------------------------------------------------------------
# trajectory-model log-likelihood (additive)
# ---------------------------------------------------------------------------------------------------
def _traj_ll_check(targets, means, variances, windows, lengths, offsets, layout):
    """Checked shapes of :func:`trajectory_log_likelihood_batch`'s arguments: ``(layout, padded, on_device)``.
    Raises ValueError for every argument error, before anything touches the device.  With ``targets=None`` it
    checks the means, variances, windows, lengths and layout alone (:func:`trajectory_sample_batch`)."""
    from ._device import is_tensor
    arrays = tuple(a for a in (targets, means, variances) if a is not None)
    kinds = [is_tensor(a) for a in arrays]
    if any(kinds) and not all(kinds):
        raise ValueError("targets, means and variances must all be NumPy arrays or all torch tensors")
    on_device = all(kinds)
    if on_device and not all(a.is_cuda for a in arrays):
        raise ValueError("torch inputs must be CUDA tensors (there is no CPU fallback)")
    if not on_device:
        targets, means, variances = (None if a is None else np.asarray(a) for a in (targets, means, variances))
    dts = [str(a.dtype).replace("torch.", "") for a in (targets, means, variances) if a is not None]
    if len(set(dts)) != 1 or dts[0] not in ("float32", "float64"):
        raise ValueError("targets, means and variances must share one dtype, float32 or float64 (got %s)" % ", ".join(dts))
    if means.ndim not in (2, 3):
        raise ValueError("means must be (sum_T, D) or (B, Tmax, D), got shape %s" % (tuple(means.shape),))
    padded = means.ndim == 3
    D = means.shape[-1]
    if padded and lengths is None:
        raise ValueError("padded (B, Tmax, D) input needs lengths")
    if not (variances.ndim == 1 and variances.shape[0] == D) and tuple(variances.shape) != tuple(means.shape):
        raise ValueError("variances must have the shape of means or be (D,) = (%d,), got %s"
                         % (D, tuple(variances.shape)))
    if not isinstance(windows, (list, tuple)) or not 1 <= len(windows) <= _lib.NNK_MAX_WIN:
        raise ValueError("windows must be a list of 1 to %d (l, u, coeff) triples" % _lib.NNK_MAX_WIN)
    for w in windows:
        l, u, c = w
        if not (0 <= int(l) <= _lib.NNK_MAX_HALF and 0 <= int(u) <= _lib.NNK_MAX_HALF) or \
                np.asarray(c).size != int(l) + int(u) + 1:
            raise ValueError("window %r: need 0 <= l, u <= %d and l + u + 1 coefficients" % (w, _lib.NNK_MAX_HALF))
    if layout is None:
        layout = StreamLayout.single(D, len(windows))
    if layout.D_in != D:
        raise ValueError("layout covers %d input columns, means have %d" % (layout.D_in, D))
    want = tuple(means.shape[:-1]) + (layout.D_out,)
    if targets is not None and tuple(targets.shape) != want:
        raise ValueError("targets must have the shape mlpg_batch returns, %s, got %s" % (want, tuple(targets.shape)))
    n_rows = means.shape[0] * means.shape[1] if padded else means.shape[0]
    try:
        lens = np.asarray(lengths.cpu().numpy() if is_tensor(lengths) else lengths) if lengths is not None else None
        if padded:
            if lens.ndim != 1 or len(lens) != means.shape[0] or np.any(lens < 0) or np.any(lens > means.shape[1]):
                raise ValueError
        else:
            off = _offsets_from(lens, offsets, n_rows)
            if off.ndim != 1 or off[0] != 0 or off[-1] != n_rows or np.any(np.diff(off) < 0):
                raise ValueError
    except (ValueError, TypeError, AttributeError):
        raise ValueError("lengths / offsets do not describe the %d rows of the batch" % n_rows)
    return layout, padded, on_device


def _traj_ll_device(targets, means, variances, windows, lengths, offsets, layout, padded, grad):
    """One launch of ``nnk_mlpg_traj_ll`` on checked CUDA tensors, on the current stream, with one host
    synchronisation (the status word).  Returns ``(ll (n_utt, n_chain) float64, lens, grads)``; ``grads`` is
    ``(g_means, g_vars, g_targets)`` in the layouts of nnk_mlpg_traj_ll in include/nnk_b200.h (``g_vars`` float64
    ``(n_utt, D)`` partials for ``(D,)`` variances), or None."""
    import torch

    from . import _device as dev
    device = means.device
    dev.poll_errors()
    m, v, x = means.contiguous(), variances.contiguous(), targets.contiguous()
    D = m.shape[-1]
    n_rows = m.shape[0] * m.shape[1] if padded else m.shape[0]
    table = _utterance_table(lengths, offsets, n_rows, m.shape[:2] if padded else None)
    _, lens, _, max_T, n_utt = table
    var1d = v.dim() == 1
    ll = torch.zeros((n_utt, layout.n_chain), dtype=torch.float64, device=device)
    grads = None
    if grad:
        grads = (torch.zeros_like(m), torch.zeros((n_utt, D), dtype=torch.float64, device=device) if var1d
                 else torch.zeros_like(v), torch.zeros_like(x))
    if not (n_utt and max_T and layout.n_chain):
        return ll, lens, grads
    a, keep, status = _traj_args(m, v, windows, table, layout, padded, _lib.lib.nnk_mlpg_traj_ll_workspace_bytes)
    t = _lib.NnkTrajLl()
    t.targets, t.tgt_ld, t.ll, t.grad = x.data_ptr(), layout.D_out, ll.data_ptr(), int(bool(grad))
    if grad:
        t.grad_means, t.gm_ld = grads[0].data_ptr(), D
        t.grad_vars, t.gv_ld = grads[1].data_ptr(), D
        t.grad_targets, t.gx_ld = grads[2].data_ptr(), layout.D_out
    _lib.check(_lib.lib.nnk_mlpg_traj_ll(ctypes.byref(a), ctypes.byref(t), dev.current_stream_ptr(device)),
               "nnk_mlpg_traj_ll")
    dev.raise_if_failed(status)
    return ll, lens, grads


def _traj_args(m, v, windows, table, layout, padded, sizing):
    """``(args, keep, status)``: the nnk_mlpg_args_t of contiguous CUDA means and variances and the batch table
    ``table`` of :func:`_utterance_table`, with a workspace sized by ``sizing`` (``nnk_mlpg_traj_*_workspace_bytes``,
    capped at ``_device.WORKSPACE_CAP_BYTES`` but never below one utterance) and a zeroed status word.  ``keep``
    holds the device tables the launch reads."""
    import torch

    from . import _device as dev
    device = m.device
    off, lens, order, max_T, n_utt = table
    D = m.shape[-1]
    win = _lib.make_windows(windows)
    a = _lib.NnkMlpgArgs()
    a.means, a.vars = m.data_ptr(), v.data_ptr()
    a.dtype, a.n_utt = dev.torch_dtype_code(m.dtype), n_utt
    a.in_ld, a.var_ld = D, 0 if v.dim() == 1 else D
    offsets_d = torch.from_numpy(off).to(device)
    order_d = torch.from_numpy(order).to(device)
    lens_d = dev.lengths_on(lens, device) if padded else None
    a.utt_off, a.order = offsets_d.data_ptr(), order_d.data_ptr()
    a.utt_len = lens_d.data_ptr() if lens_d is not None else None
    chains = dev.chains_on_device(layout.chains, device)
    a.chains, a.n_chain, a.max_T, a.win = chains.data_ptr(), layout.n_chain, max_T, win
    need = sizing(n_utt, layout.n_chain, max_T, ctypes.byref(win))
    if need == 0:
        raise NotImplementedError("window set not supported by the CUDA kernels")
    per_utt = need // n_utt
    ws = dev.workspace(device, max(per_utt, min(need, max(dev.WORKSPACE_CAP_BYTES, per_utt))))
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    status = torch.zeros(1, dtype=torch.int64, device=device)
    a.status_word = status.data_ptr()
    return a, (offsets_d, order_d, lens_d, chains, ws), status


def _traj_ll_scatter(ll, layout):
    """(n_utt, n_chain) per-chain log-likelihoods -> (n_utt, D_out), zero in columns no chain solves."""
    import torch
    out = torch.zeros((ll.shape[0], layout.D_out), dtype=torch.float64, device=ll.device)
    if layout.n_chain:
        out[:, torch.from_numpy(layout.chains["out_col"].astype(np.int64)).to(ll.device)] = ll
    return out


def trajectory_log_likelihood_batch(targets, means, variances, windows, lengths=None, offsets=None, layout=None):
    r"""Log-likelihood of target trajectories under the trajectory model of the MLPG inputs (additive API).

    Per utterance and smoothed output column, with ``P`` and ``b`` exactly as :func:`mlpg_batch` builds them
    (its edge rule included) and :math:`\bar c = P^{-1} b` the trajectory it returns, the target static
    trajectory :math:`x` scores

    .. math:: \ell = \tfrac12 \log\det P - \tfrac12 (x - \bar c)^T P (x - \bar c) - \tfrac T2 \log 2\pi,

    the log-density of :math:`N(x; \bar c, P^{-1})` (Zen, Tokuda & Kitamura 2007).  Use it as an objective
    measure of an acoustic model or, through :func:`nnmnkwii_b200.autograd.trajectory_log_likelihood`, as a
    training loss.  See DESIGN.md 3.20.

    Args:
        targets: natural static trajectories, shaped like :func:`mlpg_batch`'s result (``(sum_T, D_out)`` or
            ``(B, Tmax, D_out)``); copied columns are not read.
        means, variances, windows, lengths, offsets, layout: as :func:`mlpg_batch` (flat or padded, per-frame
            or global ``(D,)`` variances).  All three arrays are NumPy arrays or all CUDA tensors, of one dtype.

    Returns:
        ``(n_utt, D_out)`` float64 log-likelihoods, zero in copied columns; NumPy for NumPy input, a CUDA
        tensor for tensors (computed on the current stream).  Arithmetic is float64.  Targets and means are not
        checked: non-finite values give NaN.  A variance that makes a pivot of ``P`` non-positive raises
        ``numpy.linalg.LinAlgError`` as :func:`mlpg_batch` does.
    """
    import torch

    from . import _device as dev
    layout, padded, on_device = _traj_ll_check(targets, means, variances, windows, lengths, offsets, layout)
    dev.require_cuda()
    if not on_device:
        device = dev.cuda_device()
        targets, means, variances = (torch.from_numpy(np.ascontiguousarray(a)).to(device)
                                     for a in (targets, means, variances))
    ll, _, _ = _traj_ll_device(targets, means, variances, windows, lengths, offsets, layout, padded, False)
    out = _traj_ll_scatter(ll, layout)
    return out if on_device else out.cpu().numpy()


def trajectory_log_likelihood(targets, mean_frames, variance_frames, windows):
    """:func:`trajectory_log_likelihood_batch` of one utterance: ``targets (T, static_dim)``, :func:`mlpg`'s
    ``(T, D)`` means and variances (or ``(D,)``); returns the ``(static_dim,)`` float64 log-likelihoods."""
    return trajectory_log_likelihood_batch(targets, mean_frames, variance_frames, windows,
                                           lengths=[mean_frames.shape[0]])[0]


# ---------------------------------------------------------------------------------------------------
# sampling from the trajectory model (additive)
# ---------------------------------------------------------------------------------------------------
def _is_int(x):
    return isinstance(x, (int, np.integer)) and not isinstance(x, (bool, np.bool_))


def _traj_sample_check(n_samples, seed, keys, scale, n_utt):
    """Checked ``(n_samples, seed, keys (uint32 array or None), scale)`` of :func:`trajectory_sample_batch`; raises
    ValueError for every argument error."""
    from ._device import is_tensor
    if not _is_int(n_samples) or not 1 <= int(n_samples) < 2 ** 31:
        raise ValueError("n_samples must be an int in [1, 2^31), got %r" % (n_samples,))
    if not _is_int(seed) or not 0 <= int(seed) < 2 ** 64:
        raise ValueError("seed must be an int in [0, 2^64), got %r" % (seed,))
    if keys is not None:
        k = np.asarray(keys.detach().cpu().numpy() if is_tensor(keys) else keys)
        if k.shape != (n_utt,) or (k.size and (not np.issubdtype(k.dtype, np.integer) or k.min() < 0
                                               or int(k.max()) >= 2 ** 32)):
            raise ValueError("keys must be %d integers in [0, 2^32), one per utterance" % n_utt)
        keys = k.astype(np.uint32)
    try:
        scale = float(scale)
    except (TypeError, ValueError):
        raise ValueError("scale must be a finite number >= 0, got %r" % (scale,))
    if not (np.isfinite(scale) and scale >= 0.0):
        raise ValueError("scale must be a finite number >= 0, got %r" % (scale,))
    return int(n_samples), int(seed), keys, scale


def _traj_sample_device(means, variances, windows, table, layout, padded, n_samples, seed, keys, scale):
    """One launch of ``nnk_mlpg_traj_sample`` per workspace wave on checked CUDA tensors, on the current stream,
    with one host synchronisation (the status word).  Returns the ``(n_samples,) + mlpg_batch`` shaped samples."""
    import torch

    from . import _device as dev
    device = means.device
    dev.poll_errors()
    m, v = means.contiguous(), variances.contiguous()
    _, _, _, max_T, n_utt = table
    out = torch.zeros((n_samples,) + tuple(m.shape[:-1]) + (layout.D_out,), dtype=m.dtype, device=device)
    if not (n_utt and max_T and layout.n_chain):
        return out
    a, keep, status = _traj_args(m, v, windows, table, layout, padded, _lib.lib.nnk_mlpg_traj_sample_workspace_bytes)
    a.out, a.out_ld = out.data_ptr(), layout.D_out
    keys_d = torch.from_numpy(keys.view(np.int32)).to(device) if keys is not None else None
    t = _lib.NnkTrajSample()
    t.sample_stride, t.n_samples, t.seed, t.scale = out[0].numel(), n_samples, seed, scale
    t.keys = keys_d.data_ptr() if keys_d is not None else None
    _lib.check(_lib.lib.nnk_mlpg_traj_sample(ctypes.byref(a), ctypes.byref(t), dev.current_stream_ptr(device)),
               "nnk_mlpg_traj_sample")
    dev.raise_if_failed(status)
    return out


def trajectory_sample_batch(means, variances, windows, n_samples=1, seed=0, keys=None, scale=1.0, lengths=None,
                            offsets=None, layout=None):
    r"""Samples from the trajectory model of the MLPG inputs (additive API).

    Per utterance and smoothed output column, with ``P`` and ``b`` exactly as :func:`mlpg_batch` builds them (its
    edge rule included) and :math:`\bar c = P^{-1} b` the trajectory it returns, each sample is a draw of
    :math:`N(\bar c, \mathrm{scale}^2 P^{-1})` (Zen, Tokuda & Kitamura 2007): the static trajectories the model
    that :func:`trajectory_log_likelihood_batch` scores spreads around its mode.  ``scale = 0`` gives
    :func:`mlpg_batch`'s result in every sample.  See DESIGN.md 3.21.

    The noise is counter-based (Philox4x32-10, Box-Muller; the comment of nnk_mlpg_traj_sample in include/nnk_b200.h
    defines it bit for bit): a draw is a pure function of ``(seed, key, sample index, frame, output column)``.  It
    does not depend on the batch around an utterance, its padding, the dtype or ``n_samples``: the first ``k`` of 16
    samples are the ``k`` samples of ``n_samples = k``.

    Args:
        means, variances, windows, lengths, offsets, layout: as :func:`mlpg_batch` (flat or padded, per-frame or
            global ``(D,)`` variances).  Both arrays are NumPy arrays or both CUDA tensors, of one dtype.
        n_samples: samples per utterance, an int in [1, 2^31).
        seed: an int in [0, 2^64).
        keys: ``n_utt`` integers in [0, 2^32), the key of each utterance's noise (for example its index in the
            dataset, so that a draw does not depend on how the batch was shuffled).  Default: the utterance's
            index in the batch (the order of ``offsets``, or the batch index of padded input).
        scale: multiplies the standard deviation; finite and >= 0.

    Returns:
        ``(n_samples,) + mlpg_batch's result shape`` in the input dtype: NumPy for NumPy input, a CUDA tensor
        for tensors (computed on the current stream).  Copied columns repeat the means in every sample; padded
        tail rows are zero.  Arithmetic is float64.  A variance that makes a pivot of ``P`` non-positive raises
        ``numpy.linalg.LinAlgError`` as :func:`mlpg_batch` does.
    """
    import torch

    from . import _device as dev
    layout, padded, on_device = _traj_ll_check(None, means, variances, windows, lengths, offsets, layout)
    if not on_device:
        means, variances = np.asarray(means), np.asarray(variances)
    n_rows = means.shape[0] * means.shape[1] if padded else means.shape[0]
    table = _utterance_table(lengths, offsets, n_rows, tuple(means.shape[:2]) if padded else None)
    n_samples, seed, keys, scale = _traj_sample_check(n_samples, seed, keys, scale, table[4])
    dev.require_cuda()
    if not on_device:
        device = dev.cuda_device()
        means, variances = (torch.from_numpy(np.ascontiguousarray(a)).to(device) for a in (means, variances))
    out = _traj_sample_device(means, variances, windows, table, layout, padded, n_samples, seed, keys, scale)
    return out if on_device else out.cpu().numpy()


def trajectory_sample(mean_frames, variance_frames, windows, n_samples=1, seed=0, scale=1.0):
    """:func:`trajectory_sample_batch` of one utterance (key 0): :func:`mlpg`'s ``(T, D)`` means and variances
    (or ``(D,)``); returns the ``(n_samples, T, static_dim)`` samples."""
    return trajectory_sample_batch(mean_frames, variance_frames, windows, n_samples=n_samples, seed=seed,
                                   scale=scale, lengths=[mean_frames.shape[0]])


# ---------------------------------------------------------------------------------------------------
# gradient of MLPG in means and variances (additive)
# ---------------------------------------------------------------------------------------------------
def _mlpg_vjp_device(means, variances, windows, grad_output, table, layout, padded):
    """One launch of ``nnk_mlpg_vjp`` per workspace wave on checked CUDA tensors, on the current stream, with one
    host synchronisation (the status word).  Returns ``(grad_means, grad_variances)`` shaped like the inputs, in
    their dtype; ``(D,)`` variances get the per-utterance float64 partials summed over the batch."""
    import torch

    from . import _device as dev
    device = means.device
    dev.poll_errors()
    m, v, go = means.contiguous(), variances.contiguous(), grad_output.contiguous()
    _, _, _, max_T, n_utt = table
    D = m.shape[-1]
    var1d = v.dim() == 1
    g_m = torch.zeros_like(m)
    g_v = torch.zeros((n_utt, D), dtype=torch.float64, device=device) if var1d else torch.zeros_like(v)
    if n_utt and max_T and layout.n_chain:
        a, keep, status = _traj_args(m, v, windows, table, layout, padded, _lib.lib.nnk_mlpg_vjp_workspace_bytes)
        t = _lib.NnkMlpgVjp()
        t.grad_out, t.go_ld = go.data_ptr(), layout.D_out
        t.grad_means, t.gm_ld = g_m.data_ptr(), D
        t.grad_vars, t.gv_ld = g_v.data_ptr(), D
        _lib.check(_lib.lib.nnk_mlpg_vjp(ctypes.byref(a), ctypes.byref(t), dev.current_stream_ptr(device)),
                   "nnk_mlpg_vjp")
        dev.raise_if_failed(status)
    if var1d:
        g_v = g_v.sum(dim=0).to(m.dtype)
    return g_m, g_v


def mlpg_vjp_batch(means, variances, windows, grad_output, lengths=None, offsets=None, layout=None):
    r"""Gradient of :func:`mlpg_batch` in its means and its variances (additive API), for minimum generation error
    training through MLPG (Wu & Wang 2006; Wu & King 2015).

    Per utterance and smoothed output column, with ``P``, ``b`` and :math:`\bar c = P^{-1} b` exactly as
    :func:`mlpg_batch` builds them (its edge rule included), :math:`o = \partial L / \partial \bar c` the
    matching column of ``grad_output`` and :math:`g = P^{-1} o`:

    .. math::
        \partial L / \partial \mu_{t,w} = \tau_{t,w} (W_w g)_t, \qquad
        \partial L / \partial \sigma^2_{t,w} = -\tau_{t,w}^2 (W_w g)_t (\mu_{t,w} - (W_w \bar c)_t),

    with :math:`\tau = 1 / \sigma^2`.  Both are 0 where the edge rule sets the precision to zero.  Copied columns
    pass the gradient through to their mean and get a zero variance gradient.  The mean gradient is what
    :func:`mlpg_grad_batch` returns, here in the input dtype.  See DESIGN.md 3.22.

    Args:
        means, variances, windows, lengths, offsets, layout: as :func:`mlpg_batch` (flat or padded, per-frame or
            global ``(D,)`` variances).
        grad_output: the gradient with respect to :func:`mlpg_batch`'s result, of its shape.  All three arrays are
            NumPy arrays or all CUDA tensors, of one dtype (float32 or float64).

    Returns:
        ``(grad_means, grad_variances)`` shaped like ``means`` and ``variances``, in their dtype: NumPy for NumPy
        input, CUDA tensors for tensors (computed on the current stream, one kernel launch).  Padded rows get zero.
        For ``(D,)`` variances the per-frame gradients are summed over every frame of the batch.  Arithmetic is
        float64.  A variance that makes a pivot of ``P`` non-positive raises ``numpy.linalg.LinAlgError`` as
        :func:`mlpg_batch` does.
    """
    import torch

    from . import _device as dev
    layout, padded, on_device = _traj_ll_check(grad_output, means, variances, windows, lengths, offsets, layout)
    if not on_device:
        means, variances, grad_output = (np.asarray(a) for a in (means, variances, grad_output))
    n_rows = means.shape[0] * means.shape[1] if padded else means.shape[0]
    table = _utterance_table(lengths, offsets, n_rows, tuple(means.shape[:2]) if padded else None)
    dev.require_cuda()
    if not on_device:
        device = dev.cuda_device()
        means, variances, grad_output = (torch.from_numpy(np.ascontiguousarray(a)).to(device)
                                         for a in (means, variances, grad_output))
    g_m, g_v = _mlpg_vjp_device(means, variances, windows, grad_output, table, layout, padded)
    return (g_m, g_v) if on_device else (g_m.cpu().numpy(), g_v.cpu().numpy())
