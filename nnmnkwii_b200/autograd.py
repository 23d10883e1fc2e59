"""Autograd functions -- drop-in for the MLPG part of ``nnmnkwii.autograd``
(nnmnkwii/autograd/_impl/mlpg.py): ``MLPG``, ``UnitVarianceMLPG``, ``mlpg``, ``unit_variance_mlpg``.

Differences that are additions, not signature changes:
  * ``MLPG`` works on CUDA tensors in place (the reference "cannot run on CUDA", mlpg.py:33) and
    moves CPU tensors to the GPU and back; its backward is one banded solve + stencil per static
    dimension instead of the reference's dense ``T x T`` solve per (dimension, window).
  * ``UnitVarianceMLPG`` keeps the ``(means, R)`` signature; the dense ``R`` (``T x nw*T``) is
    reduced once to its numerical band and applied as a banded stencil sweep
    (csrc/nnk_uvmlpg.cu) instead of two dense GEMMs that multiply ~95 % zeros.

Additive: ``TrajectoryLogLikelihood`` / ``trajectory_log_likelihood``, the log-likelihood of
target trajectories under the trajectory model of the MLPG inputs, differentiable in targets, means and variances.
``MLPGWithVariances`` / ``mlpg_with_variances``: MLPG differentiable in its means and its variances, for minimum
generation error training of models that predict variances.

The modulation-spectrum part (nnmnkwii/autograd/_impl/modspec.py): ``ModSpec`` and ``modspec``, plus the batched
``ModSpecBatch`` / ``modspec_batch``, on csrc/nnk_modspec.cu.
"""
import numpy as np
import torch
from torch.autograd import Function

from . import _device as dev
from . import paramgen as G
from . import preprocessing as P
from .preprocessing.modspec import _modspec_grad


def _global_variance(variances):
    """A global ``(D,)`` variance -- given as such or as ``v.expand(T, D)`` (stride 0 over frames, what
    the reference's ``autograd.mlpg`` builds, mlpg.py:196-197) -- as a 1-D tensor; anything else unchanged."""
    if variances.dim() == 2 and variances.shape[0] > 1 and variances.stride(0) == 0:
        return variances[0]
    return variances


class MLPG(Function):
    """Generic MLPG as an autograd function, ``f : (T, D) -> (T, static_dim)`` (mlpg.py:8-67).

    Forward = :func:`nnmnkwii_b200.paramgen.mlpg`, backward = :func:`nnmnkwii_b200.paramgen.mlpg_grad`;
    returns float32 like the reference (mlpg.py:53); gradients for ``variances`` / ``windows`` are None.
    """

    @staticmethod
    def forward(ctx, means, variances, windows):
        assert means.dim() == 2  # we cannot do MLPG on minibatch (mlpg.py:44)
        ctx.windows = windows
        variances = _global_variance(variances)  # (D,) or a stride-0 expansion of it -> 1-D (16*sd B/frame path)
        ctx.save_for_backward(means, variances)
        assert variances.dim() == 1 or means.size() == variances.size()
        dev.require_cuda()
        device = dev.cuda_device(means)
        m = means.detach().to(device)
        v = variances.detach().to(device)
        # CUDA inputs: non-blocking status check (surfaces at the next call); CPU inputs (the reference's
        # use) synchronise on the copy back anyway, so the check is immediate
        ctx.check = "deferred" if means.is_cuda else True
        y = G.mlpg_batch(m, v, windows, lengths=[m.shape[0]], check=ctx.check).to(torch.float32)
        return y.to(means.device)

    @staticmethod
    def backward(ctx, grad_output):
        means, variances = ctx.saved_tensors
        dev.require_cuda()
        device = dev.cuda_device(means)
        g = G.mlpg_grad(means.detach().to(device), variances.detach().to(device), ctx.windows,
                        grad_output.detach().to(device), check=ctx.check)
        return g.to(means.device), None, None


class MLPGBatch(Function):
    """Additive: :class:`MLPG` over a whole mini-batch -- ``(B, Tmax, D)`` zero-padded or flat
    ``(sum_T, D)`` means with per-utterance ``lengths`` -- one forward and one backward kernel launch
    for all utterances (the reference's ``MLPG`` is 2-D only and is looped over the batch).
    Per-frame variances of the same shape, or global ``(D,)``.  Returns float32."""

    @staticmethod
    def forward(ctx, means, variances, windows, lengths):
        assert means.dim() in (2, 3)
        ctx.windows = windows
        ctx.lengths = [int(n) for n in (lengths.tolist() if torch.is_tensor(lengths) else lengths)]
        ctx.save_for_backward(means, variances)
        dev.require_cuda()
        device = dev.cuda_device(means)
        ctx.check = "deferred" if means.is_cuda else True
        y = G.mlpg_batch(means.detach().to(device), variances.detach().to(device), windows, lengths=ctx.lengths,
                         check=ctx.check)
        return y.to(torch.float32).to(means.device)

    @staticmethod
    def backward(ctx, grad_output):
        means, variances = ctx.saved_tensors
        dev.require_cuda()
        device = dev.cuda_device(means)
        g = G.mlpg_grad_batch(variances.detach().to(device), ctx.windows, grad_output.detach().to(device), ctx.lengths,
                              check=ctx.check)
        return g.to(means.device), None, None, None


class UnitVarianceMLPG(Function):
    r"""MLPG for unit-variance inputs, ``y = R \mu`` (mlpg.py:70-172).

    ``f : (T x D) -> (T, static_dim)`` or ``f : (T*num_windows, static_dim) -> (T, static_dim)``,
    2-D or 3-D (batched) ``means``; ``R`` from :func:`nnmnkwii_b200.paramgen.unit_variance_mlpg_matrix`.

    The band tables of ``R`` are cached on its storage pointer and torch's version counter.  Changing ``R``
    in place through torch bumps that counter; changing it through a NumPy view or ``R.data`` does not, and
    the stale tables are then used.  Pass a new tensor after such a change.
    """

    @staticmethod
    def forward(ctx, means, R):
        from . import _uvmlpg as uv

        ctx.save_for_backward(means, R)
        ctx.num_windows = R.shape[-1] // R.shape[0]
        T = R.shape[0]
        dim = means.dim()
        if dim == 2:
            T_, D = means.shape
            B = 1
            means3 = means.reshape(B, T_, D)
        else:
            B, T_, D = means.shape
            means3 = means
        reshaped = not (T == T_)  # mlpg.py:123: input already (T*nw, static_dim)?
        dev.require_cuda()
        device = dev.cuda_device(means)
        band = uv.band_of(R, device)
        out = uv.apply_forward(band, means3.detach().to(device), reshaped).to(means.device)
        ctx.reshaped = reshaped
        if dim == 2:
            return out.view(-1, out.shape[-1])
        return out

    @staticmethod
    def backward(ctx, grad_output):
        from . import _uvmlpg as uv

        means, R = ctx.saved_tensors
        T = R.shape[0]
        dim = means.dim()
        if dim == 2:
            T_, D = means.shape
            B = 1
            grad_output = grad_output.reshape(B, T, -1)
        else:
            B, T_, D = means.shape
        dev.require_cuda()
        device = dev.cuda_device(means)
        band = uv.band_of(R, device)
        grad = uv.apply_backward(band, grad_output.detach().to(device), ctx.reshaped, D).to(means.device)
        if dim == 2:
            return grad.view(-1, D), None
        return grad, None


class ModSpec(Function):
    """Modulation spectrum as an autograd function, ``f : (T, D) -> (n // 2 + 1, D)`` (modspec.py:9-60).

    Forward = :func:`nnmnkwii_b200.preprocessing.modspec`.  Backward is the adjoint of the power spectrum,
    ``dL/dy_t = 2 Re(sum_k dL/dP_k conj(Y_k) e^{-2 pi i k t / n})``, the same kernel in its gradient mode: an
    inverse FFT per column instead of the reference's dense ``(n // 2 + 1) x T`` cosine and sine tables.  Takes
    CUDA tensors only and keeps their dtype (the reference takes CPU tensors and returns float32 gradients).
    """

    @staticmethod
    def forward(ctx, y, n, norm):
        assert y.dim() == 2
        ctx.n, ctx.norm = n, norm
        ctx.save_for_backward(y)
        return P.modspec(y.detach(), n=n, norm=norm)

    @staticmethod
    def backward(ctx, grad_output):
        (y,) = ctx.saved_tensors
        return _modspec_grad(y, grad_output, ctx.n, ctx.norm), None, None


class ModSpecBatch(Function):
    """Additive: :class:`ModSpec` over a padded ``(B, T, D)`` batch with per-utterance ``lengths``, one kernel
    launch forward and one backward; ``f : (B, T, D) -> (B, n // 2 + 1, D)``.  Frames past an utterance's length
    take no part and get a zero gradient."""

    @staticmethod
    def forward(ctx, y, n, norm, lengths):
        assert y.dim() == 3
        ctx.n, ctx.norm = n, norm
        ctx.lengths = [int(v) for v in (lengths.tolist() if torch.is_tensor(lengths) else lengths)]
        ctx.save_for_backward(y)
        return P.modspec(y.detach(), n=n, norm=norm, lengths=ctx.lengths)

    @staticmethod
    def backward(ctx, grad_output):
        (y,) = ctx.saved_tensors
        return _modspec_grad(y, grad_output, ctx.n, ctx.norm, ctx.lengths), None, None, None


def modspec(y, n=2048, norm=None):
    """Modulation spectrum of a ``(T, D)`` CUDA tensor, differentiable (modspec.py:63-72)."""
    return ModSpec.apply(y, n, norm)


def modspec_batch(y, lengths, n=2048, norm=None):
    """Additive: batched :func:`modspec` (see :class:`ModSpecBatch`)."""
    return ModSpecBatch.apply(y, n, norm, lengths)


class TrajectoryLogLikelihood(Function):
    """Additive: the trajectory-model log-likelihood of :func:`nnmnkwii_b200.paramgen.trajectory_log_likelihood_batch`
    as an autograd function, ``f : (targets, means, variances) -> (B, D_out)`` float64, differentiable in all three
    (:class:`MLPGWithVariances` gives the variance gradient of a generation error).  CUDA tensors, flat
    ``(sum_T, D)`` or zero-padded ``(B, Tmax, D)`` with ``lengths``; variances per frame or global ``(D,)``;
    ``targets`` shaped like :func:`mlpg_batch`'s result.  The forward is one kernel launch, with the gradients
    computed in the same launch only when an input needs them; the backward scales them by ``grad_output[u, column]``
    with elementwise ops (and, for ``(D,)`` variances, a sum over utterances in a fixed order).  Gradients have each
    input's shape and dtype; padded frames and copied columns get zero."""

    @staticmethod
    def forward(ctx, targets, means, variances, windows, lengths, layout=None):
        layout, padded, on_device = G._traj_ll_check(targets, means, variances, windows, lengths, None, layout)
        if not on_device:
            raise ValueError("TrajectoryLogLikelihood takes CUDA tensors")
        grad = any(ctx.needs_input_grad[:3])
        ll, lens, grads = G._traj_ll_device(targets.detach(), means.detach(), variances.detach(), windows, lengths,
                                            None, layout, padded, grad)
        ctx.padded, ctx.lens, ctx.layout, ctx.nw = padded, lens, layout, len(windows)
        ctx.shapes = (targets.shape, means.shape, variances.shape)
        if grad:
            ctx.save_for_backward(*grads)
        return G._traj_ll_scatter(ll, layout)

    @staticmethod
    def backward(ctx, grad_output):
        g_m, g_v, g_x = ctx.saved_tensors
        layout, lens = ctx.layout, ctx.lens
        device = g_m.device
        go = grad_output.to(torch.float64)
        D = g_m.shape[-1]
        # scale of input column i of utterance u: grad_output[u, out_col of the chain that reads i], 0 if none
        col_out = np.full(D, layout.D_out, dtype=np.int64)  # D_out: a zero column appended to grad_output
        for c in layout.chains[layout.chains["flags"] == 0]:
            col_out[int(c["in_col"]) + np.arange(ctx.nw) * int(c["win_stride"])] = int(c["out_col"])
        go_ext = torch.cat([go, torch.zeros((go.shape[0], 1), dtype=torch.float64, device=device)], dim=1)
        s_in = go_ext[:, torch.from_numpy(col_out).to(device)]  # (B, D)
        s_out = go  # (B, D_out)
        if ctx.padded:
            rows_in, rows_out = s_in[:, None, :], s_out[:, None, :]
        else:
            reps = torch.from_numpy(np.asarray(lens, dtype=np.int64)).to(device)
            rows_in = torch.repeat_interleave(s_in, reps, dim=0, output_size=int(np.sum(lens)))
            rows_out = torch.repeat_interleave(s_out, reps, dim=0, output_size=int(np.sum(lens)))
        gm = (g_m.to(torch.float64) * rows_in).to(g_m.dtype) if ctx.needs_input_grad[1] else None
        if ctx.needs_input_grad[2]:
            if len(ctx.shapes[2]) == 1:
                gv = (g_v * s_in).sum(dim=0).to(g_m.dtype)
            else:
                gv = (g_v.to(torch.float64) * rows_in).to(g_v.dtype)
        else:
            gv = None
        gx = (g_x.to(torch.float64) * rows_out).to(g_x.dtype) if ctx.needs_input_grad[0] else None
        return gx, gm, gv, None, None, None


def trajectory_log_likelihood(targets, means, variances, windows, lengths, layout=None):
    """Additive: differentiable trajectory-model log-likelihood (see :class:`TrajectoryLogLikelihood`)."""
    return TrajectoryLogLikelihood.apply(targets, means, variances, windows, lengths, layout)


class MLPGWithVariances(Function):
    """Additive: MLPG differentiable in its means and its variances, ``f : (means, variances) -> mlpg_batch(...)``,
    for minimum generation error training (Wu & Wang 2006) of models that predict variances.  :class:`MLPG` and
    :class:`MLPGBatch` return no variance gradient.

    CUDA tensors only, of one dtype (float32 or float64): flat ``(sum_T, D)`` with ``lengths`` (a 2-D input without
    ``lengths`` is one utterance) or zero-padded ``(B, Tmax, D)`` with ``lengths``; variances per frame or global
    ``(D,)``; any :class:`~nnmnkwii_b200.paramgen.StreamLayout`.  The forward is
    :func:`nnmnkwii_b200.paramgen.mlpg_batch` (the same bits) in the means' dtype; the backward is one kernel launch
    of :func:`nnmnkwii_b200.paramgen.mlpg_vjp_batch`.  A stride-0 ``v.expand(T, D)`` is materialised and gets true
    per-frame gradients, which autograd sums back through the expand."""

    @staticmethod
    def forward(ctx, means, variances, windows, lengths, layout=None):
        layout, padded, on_device = G._traj_ll_check(None, means, variances, windows, lengths, None, layout)
        if not on_device:
            raise ValueError("MLPGWithVariances takes CUDA tensors")
        m, v = means.detach(), variances.detach().contiguous()
        ctx.windows, ctx.lengths, ctx.layout = windows, lengths, layout
        ctx.save_for_backward(m, v)
        return G.mlpg_batch(m, v, windows, lengths=lengths, layout=layout)

    @staticmethod
    def backward(ctx, grad_output):
        m, v = ctx.saved_tensors
        g_m, g_v = G.mlpg_vjp_batch(m, v, ctx.windows, grad_output.to(m.dtype), lengths=ctx.lengths,
                                    layout=ctx.layout)
        return (g_m if ctx.needs_input_grad[0] else None), (g_v if ctx.needs_input_grad[1] else None), None, None, None


def mlpg_with_variances(means, variances, windows, lengths=None, layout=None):
    """Additive: MLPG differentiable in means and variances (see :class:`MLPGWithVariances`)."""
    return MLPGWithVariances.apply(means, variances, windows, lengths, layout)


def mlpg(means, variances, windows):
    """Maximum Likelihood Parameter Generation on tensors (mlpg.py:175-199).

    ``variances`` may be ``(T, D)`` or global ``(D,)`` (expanded over frames).
    """
    T, D = means.size()
    if not (variances.dim() == 1 and variances.shape[0] == D):  # a global (D,) variance stays 1-D
        assert means.size() == variances.size()
    return MLPG.apply(means, variances, windows)


def mlpg_batch(means, variances, windows, lengths):
    """Additive: batched :func:`mlpg` (see :class:`MLPGBatch`)."""
    return MLPGBatch.apply(means, variances, windows, lengths)


def unit_variance_mlpg(R, means):
    """Special case of MLPG assuming unit variances (mlpg.py:202-217).  NB argument order
    ``(R, means)`` here, ``(means, R)`` for ``UnitVarianceMLPG.apply`` -- as in the reference."""
    return UnitVarianceMLPG.apply(means, R)


__all__ = ["MLPG", "MLPGBatch", "UnitVarianceMLPG", "mlpg", "mlpg_batch", "unit_variance_mlpg", "ModSpec",
           "ModSpecBatch", "modspec", "modspec_batch", "TrajectoryLogLikelihood", "trajectory_log_likelihood",
           "MLPGWithVariances", "mlpg_with_variances"]
_ = np  # numpy is part of the reference module's namespace
