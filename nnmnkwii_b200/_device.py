"""Device-side plumbing shared by the Python host layer: PyTorch owns allocation and streams,
libnnk_b200 (C ABI) does the arithmetic.  No numerical work happens in this file."""
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import CHAIN_DTYPE, NnkMlpgArgs, NnkStatus, lib

_const_cache = {}

WORKSPACE_CAP_BYTES = 2 << 30  # the launcher splits a batch into waves if it needs more


def require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError(
            "nnmnkwii_b200 needs a CUDA device (H100, sm_90a): there is no CPU fallback. "
            "torch.cuda.is_available() is False.")


# ---- the array boundary: caller's NumPy arrays / tensors <-> device tensors -----------------------------
def is_tensor(x):
    return type(x).__module__.startswith("torch")


def np_dtype(x):
    """NumPy dtype of an array or tensor."""
    return np.dtype(str(x.dtype).replace("torch.", "")) if is_tensor(x) else np.asarray(x).dtype


def cuda_device(x=None):
    """The CUDA device of tensor ``x`` if it is on one, otherwise the current device."""
    if is_tensor(x) and x.is_cuda:
        return x.device
    return torch.device("cuda", torch.cuda.current_device())


def to_device(x, device=None):
    """``x`` as a device tensor of its own dtype, not copied where it can be avoided: a tensor is detached (a
    CUDA tensor stays on its device, a CPU tensor goes to ``device`` or the current device); an array is
    made contiguous and uploaded."""
    if is_tensor(x):
        return x.detach() if x.is_cuda else x.detach().to(device or cuda_device())
    return torch.from_numpy(np.ascontiguousarray(x)).to(device or cuda_device())


def like_input(out, x):
    """Device result ``out`` in the form of input ``x``: CUDA tensor, CPU tensor or NumPy array."""
    if is_tensor(x):
        return out if x.is_cuda else out.cpu()
    return out.cpu().numpy()


def check_lengths(lengths, n_items):
    if lengths is None:
        return None
    if is_tensor(lengths):
        lengths = lengths.detach().cpu().numpy()
    lens = np.asarray(lengths)
    if lens.ndim != 1 or (lens.size and not np.issubdtype(lens.dtype, np.integer)):
        raise ValueError("lengths must be a 1-D sequence of integers")
    lens = lens.astype(np.int64)
    if n_items is None:
        raise ValueError("lengths needs a sized dataset (len(dataset))")
    if len(lens) != n_items:
        raise ValueError("lengths has %d entries for %d items" % (len(lens), n_items))
    if lens.size and int(lens.min()) < 0:
        raise ValueError("lengths must be >= 0")
    return lens


def lengths_on(lens, device, T=None):
    """Host lengths as an int32 device tensor, clipped to ``T`` when given; None stays None."""
    if lens is None:
        return None
    lens = np.asarray(lens)
    return torch.as_tensor((lens if T is None else np.minimum(lens, T)).astype(np.int32), device=device)


def current_stream_ptr(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def workspace(device, nbytes):
    """Scratch for ONE call: a uint8 tensor from torch's caching allocator.

    The allocator is stream-aware -- a block freed after a launch on stream A is only handed out again
    to stream A (or after A has been synchronised) -- so concurrent streams / threads never share a
    factor scratch, and a steady-state loop gets the same block back without a cudaMalloc.  That holds
    because the scratch is allocated on, and only used by, the current stream of ``device``; a tensor
    kept beyond one call and read from other streams needs ``keep_for_current_stream``.  The block is
    not cleared: it holds whatever an earlier call left in it."""
    return torch.empty(int(max(nbytes, 256)), dtype=torch.uint8, device=device)


def simple_chains(static_dim):
    """Chain table of a single stream laid out like the reference: window w of static dim d lives
    in column w * static_dim + d (paramgen/_mlpg.py:187)."""
    ch = np.zeros(static_dim, dtype=CHAIN_DTYPE)
    ch["in_col"] = np.arange(static_dim)
    ch["win_stride"] = static_dim
    ch["out_col"] = np.arange(static_dim)
    return ch


def keep_for_current_stream(t, device):
    """Mark cached tensor ``t`` as used by the work about to be enqueued on the current stream of ``device``.

    A cache entry's block belongs to the stream that was current when it was made.  When the cache drops
    the entry, the allocator may hand that block to the next allocation on that stream at once, even if a
    kernel on another stream has yet to read it.  ``record_stream`` makes the allocator wait for the work
    enqueued so far on the current stream before it reuses the block (a no-op on the owning stream)."""
    t.record_stream(torch.cuda.current_stream(device))
    return t


def constant_on_device(a, device):
    """Device copy of a small host constant (chain table, filter weights), kept in a bounded cache.  The
    caller enqueues its reads on the current stream of ``device``; an eviction never recycles the block
    before they have run (see keep_for_current_stream)."""
    key = (a.tobytes(), a.dtype.str, a.shape, str(device))
    t = _const_cache.get(key)
    if t is None:
        t = torch.from_numpy(a.copy()).to(device)
        if len(_const_cache) >= 64:
            _const_cache.clear()
        _const_cache[key] = t
    return keep_for_current_stream(t, device)


def chains_on_device(chains_np, device):
    return constant_on_device(chains_np.view(np.int32).reshape(-1, 4), device)


def torch_dtype_code(dt):
    """C-ABI dtype code of a torch or NumPy dtype."""
    if dt in (torch.float32, np.float32):
        return _lib.NNK_F32
    if dt in (torch.float64, np.float64):
        return _lib.NNK_F64
    raise TypeError("CUDA kernels support float32 / float64, got %s" % dt)


def _raise_word(word):
    word = int(word) & 0xFFFFFFFFFFFFFFFF
    if word:
        st = NnkStatus()
        lib.nnk_status_decode(ctypes.c_uint64(word), ctypes.byref(st))
        raise np.linalg.LinAlgError(
            "%d-th leading minor not positive definite (utterance %d, chain %d)" % (st.frame, st.utt, st.chain))


def raise_if_failed(status_word_tensor):
    """Synchronising check of the device status word -> numpy.linalg.LinAlgError like the reference
    (scipy.linalg.LinAlgError is the same class; _bandmat/linalg.pyx:79-82)."""
    _raise_word(status_word_tensor.item())


# ---- deferred (non-blocking) status checks -------------------------------------------------------
# check="deferred": the status word is copied to a pinned host slot behind the kernel and an event is
# recorded; nothing waits.  The slot is examined -- and LinAlgError raised -- at the next nnmnkwii_b200
# call that finds the event complete, or by poll_errors(block=True).  Same contract as CUDA's own
# asynchronous error reporting: the error surfaces at a later call, never silently.
_DEFER_SLOTS = 64
_defer = {"host": None, "pending": [], "next": 0}


def poll_errors(block=False):
    """Raise the LinAlgError of any completed deferred check (``block=True`` waits for all of them)."""
    pend = _defer["pending"]
    while pend:
        ev, slot = pend[0]
        if not ev.query():
            if not block:
                return
            ev.synchronize()
        pend.pop(0)
        word = int(_defer["host"][slot])
        if word:
            pend.clear()
            _raise_word(word)


def _defer_check(status, device):
    if torch.cuda.is_current_stream_capturing():
        return  # inside CUDA-graph capture: the caller reads `status` itself after replay
    if _defer["host"] is None:
        _defer["host"] = torch.zeros(_DEFER_SLOTS, dtype=torch.int64).pin_memory()
    if len(_defer["pending"]) >= _DEFER_SLOTS - 1:
        poll_errors(block=True)
    slot = _defer["next"]
    _defer["next"] = (slot + 1) % _DEFER_SLOTS
    _defer["host"][slot:slot + 1].copy_(status, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(device))
    _defer["pending"].append((ev, slot))


def run_mlpg(mode, *, means, variances, rhs, out, offsets, lengths, order, chains, n_chain, max_T, windows_c,
             in_ld, var_ld, go_ld, out_ld, dtype_code, go_f64, n_utt, device, check=True, out_offsets=None, status=None,
             gv=None):
    """Fill nnk_mlpg_args_t and enqueue nnk_mlpg_{fwd,grad,solve,gv} on torch's current stream of
    ``device`` (the C ABI switches to the device that owns ``out`` for the launch).  Mode "gv" takes
    ``gv = (gv_mean, gv_var, n_iter, step, weight)`` with float64 device tensors indexed by output column
    and ``weight`` 0 for 1 / (nw T).
    ``check``: True = synchronising status check, "deferred" = non-blocking (see poll_errors), False = none."""
    poll_errors()
    a = NnkMlpgArgs()
    a.means = means.data_ptr() if means is not None else None
    a.vars = variances.data_ptr()
    a.grad_out = rhs.data_ptr() if rhs is not None else None
    a.out = out.data_ptr()
    a.dtype = dtype_code
    a.n_utt = n_utt
    a.in_ld, a.var_ld, a.go_ld, a.out_ld = in_ld, var_ld, go_ld, out_ld
    a.utt_off = offsets.data_ptr()
    a.utt_len = lengths.data_ptr() if lengths is not None else None
    a.order = order.data_ptr() if order is not None else None
    a.out_off = out_offsets.data_ptr() if out_offsets is not None else None
    a.chains = chains.data_ptr()
    a.n_chain = n_chain
    a.max_T = max_T
    a.go_f64 = go_f64
    a.win = windows_c
    sizing = lib.nnk_mlpg_gv_workspace_bytes if mode == "gv" else lib.nnk_mlpg_workspace_bytes
    need = sizing(n_utt, n_chain, max_T, ctypes.byref(windows_c))
    if need == 0 and n_utt and n_chain and max_T:
        raise NotImplementedError("window set not supported by the CUDA kernels")
    per_utt = need // max(1, n_utt)
    nbytes = max(per_utt, min(need, max(WORKSPACE_CAP_BYTES, per_utt)))
    ws = workspace(device, max(nbytes, 256))
    a.workspace = ws.data_ptr()
    a.workspace_bytes = ws.numel()
    if status is None:  # a caller-owned word accumulates the first failure over several launches
        status = torch.zeros(1, dtype=torch.int64, device=device)
    a.status_word = status.data_ptr()
    if mode == "gv":
        g = _lib.NnkMlpgGv()
        g.gv_mean, g.gv_var = gv[0].data_ptr(), gv[1].data_ptr()
        g.n_iter, g.step, g.weight = int(gv[2]), float(gv[3]), float(gv[4])
        rc = lib.nnk_mlpg_gv(ctypes.byref(a), ctypes.byref(g), current_stream_ptr(device))
    else:
        fn = {"fwd": lib.nnk_mlpg_fwd, "grad": lib.nnk_mlpg_grad, "solve": lib.nnk_mlpg_solve}[mode]
        rc = fn(ctypes.byref(a), current_stream_ptr(device))
    _lib.check(rc, "nnk_mlpg_" + mode)
    if check == "deferred":
        _defer_check(status, device)
    elif check:
        raise_if_failed(status)
    return status
