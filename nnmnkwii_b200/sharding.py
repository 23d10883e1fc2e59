"""Utterance sharding across the GPUs of one box (SURVEY.md section 8e, BASELINE.json configs[4]).

Every utterance is independent, so the data path has NO collective: the batch is dealt to ranks by
cost (frames), each rank solves its slice with the single-GPU kernels, and the trajectories are
all-gathered so that every rank ends up with the full result.  One process per GPU;
``torch.distributed`` (NCCL over NVLink on the GPUs, gloo in the CPU tests) is only the plumbing.

Layout (``ShardPlan``): the utterances are first dealt into ``n_buckets`` groups of equal frame
count, and every group is split over the ranks by a longest-first greedy rule.  Bucket ``b`` of rank
``r`` occupies rows ``[goff[b] + r * cap[b], ... + n[b][r])`` of ONE flat ``(rows_total, D_out)``
result buffer (``cap[b]`` = largest per-rank frame count of the bucket, so the dead rows are at most
one utterance per bucket and rank -- no per-utterance padding).  The MLPG kernel writes straight into
that slot (``nnk_mlpg_args_t.out_off``) and the all-gather of bucket ``b`` moves the contiguous region
``[goff[b] + r * cap[b], ...)`` of every rank ``r`` to every other rank.  Two transports:

* ``"peer"`` (default on GPUs): the result buffers are cudaMalloc allocations shared between the per-GPU
  processes by CUDA IPC; as soon as bucket ``b`` is solved every rank PUSHES its slot into its peers'
  buffers with copy-engine DMA over NVLink (``nnk_peer_copy``, one side stream per peer).  No SMs are
  involved, so the transfer really overlaps the solve of bucket ``b + 1`` (an NCCL all-gather kernel has
  to wait for SM slots that the solve kernel holds).  One tiny NCCL
  all-reduce at the end of the pass is the "everything has landed everywhere" barrier.
* ``"nccl"`` / gloo: in-place ``all_gather_into_tensor`` of the bucket region, issued on a side stream.

The result stays in shard order with a row table (``ShardedResult.row_start``) and is only re-ordered
on request (``to_utterance_order``: one segment-copy kernel, no host indexing).
"""
import ctypes

import numpy as np


def partition(costs, world_size):
    """Greedy longest-processing-time partition.  Returns a list (one entry per rank) of index arrays,
    each sorted ascending; deterministic, identical on every rank."""
    costs = np.asarray(costs, dtype=np.int64)
    order = np.argsort(-costs, kind="stable")
    load = np.zeros(world_size, dtype=np.int64)
    buckets = [[] for _ in range(world_size)]
    for i in order:
        r = int(np.argmin(load))
        buckets[r].append(int(i))
        load[r] += costs[i]
    return [np.array(sorted(b), dtype=np.int64) for b in buckets]


class ShardPlan(object):
    """Deterministic host-side plan (identical on every rank) of who solves what and where it lands.

    Attributes:
        members[b][r]: utterance ids (longest first) of bucket ``b`` on rank ``r``.
        cap[b]:        rows reserved per rank in bucket ``b`` (max over ranks of the frame count).
        goff[b]:       first row of bucket ``b`` in the gathered result; ``rows_total`` = its extent.
        loff[b]:       first row of bucket ``b`` in a rank's LOCAL input buffers (``rows_local`` rows).
        row_start[u]:  first row of utterance ``u`` in the gathered result (shard order).
    """

    def __init__(self, lengths, world_size, n_buckets=4):
        self.lengths = np.asarray(lengths, dtype=np.int64)
        self.world = int(world_size)
        n = len(self.lengths)
        nb = max(1, min(int(n_buckets), max(1, n // max(1, self.world))))
        self.n_buckets = nb
        # deal utterances (longest first) round-robin into buckets: equal frames and the same length mix
        order = np.argsort(-self.lengths, kind="stable")
        groups = [order[b::nb] for b in range(nb)]
        self.members, self.cap, self.goff, self.loff = [], [], [], []
        self.row_start = np.zeros(n, dtype=np.int64)
        self.local_start = np.zeros(n, dtype=np.int64)
        self.owner = np.zeros(n, dtype=np.int32)
        g = l = 0
        for b in range(nb):
            parts = partition(self.lengths[groups[b]], self.world)
            mem = []
            for r in range(self.world):
                ids = groups[b][parts[r]]
                ids = ids[np.argsort(-self.lengths[ids], kind="stable")]
                mem.append(ids)
            cap = int(max((int(self.lengths[m].sum()) for m in mem), default=0))
            self.members.append(mem)
            self.cap.append(cap)
            self.goff.append(g)
            self.loff.append(l)
            for r, ids in enumerate(mem):
                o = 0
                for u in ids:
                    self.row_start[u] = g + r * cap + o
                    self.local_start[u] = l + o
                    self.owner[u] = r
                    o += int(self.lengths[u])
            g += self.world * cap
            l += cap
        self.rows_total = g
        self.rows_local = l

    def frames_of_rank(self, rank):
        return int(sum(int(self.lengths[m[rank]].sum()) for m in self.members))


class _DeviceBlock(object):
    """A raw cudaMalloc allocation exposed to torch through __cuda_array_interface__."""

    def __init__(self, ptr, shape, typestr):
        self.ptr = ptr
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 3,
                                         "strides": None}


class PeerUnavailable(RuntimeError):
    """Raised on EVERY rank when the IPC-shared result blocks cannot be set up on some rank."""


class PeerTransport(object):
    """Result buffer of one rank as an IPC-shared cudaMalloc block plus the mapped pointers of every
    peer's block (see module docstring).  Collective constructor: every rank of ``group`` must call it."""

    def __init__(self, rows, cols, dtype, device, group=None):
        import torch
        import torch.distributed as dist

        from . import _lib
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.group, self.device = group, device
        self.row_bytes = cols * (4 if dtype == torch.float32 else 8)
        nbytes = max(1, rows) * self.row_bytes
        # Collective set-up that cannot leave some ranks inside a collective and others in an exception:
        # every step is attempted locally, the outcome is agreed on by an all-reduce, and on any failure
        # (CUDA IPC unavailable in this environment, peer access refused ...) EVERY rank raises PeerUnavailable,
        # which ShardedBatch turns into the NCCL transport.
        self.local_ptr, self.peer_ptr, self.tensor = None, [None] * self.world, None
        with torch.cuda.device(device):
            import os
            err = None
            handle = (ctypes.c_ubyte * 64)()
            try:
                if os.environ.get("NNK_PEER_FORCE_FAIL") == "alloc":
                    raise RuntimeError("forced failure (test)")
                ptr = ctypes.c_void_p()
                _lib.check(_lib.lib.nnk_peer_alloc(ctypes.c_size_t(nbytes), ctypes.byref(ptr)), "nnk_peer_alloc")
                self.local_ptr = ptr.value
                _lib.check(_lib.lib.nnk_peer_export(ctypes.c_void_p(self.local_ptr), handle), "nnk_peer_export")
            except Exception as e:  # noqa: BLE001 -- any local failure is reported to the group below
                err = e
            handles = [None] * self.world
            dist.all_gather_object(handles, None if err is not None else bytes(handle), group=group)
            if err is None and all(h is not None for h in handles):
                try:
                    if os.environ.get("NNK_PEER_FORCE_FAIL") == "open" and self.rank == self.world - 1:
                        raise RuntimeError("forced failure (test)")
                    for r in range(self.world):
                        if r == self.rank:
                            continue
                        buf = (ctypes.c_ubyte * 64).from_buffer_copy(handles[r])
                        out = ctypes.c_void_p()
                        _lib.check(_lib.lib.nnk_peer_open(buf, ctypes.byref(out)), "nnk_peer_open")
                        self.peer_ptr[r] = out.value
                except Exception as e:  # noqa: BLE001
                    err = e
            elif err is None:
                err = RuntimeError("a peer could not export its result block")
            ok = torch.tensor([0 if err is not None else 1], dtype=torch.int32, device=device)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
            if int(ok.item()) == 0:
                self.close()
                raise PeerUnavailable("peer-memory transport unavailable (%s)" % (err if err is not None else "failure on another rank"))
            self.block = _DeviceBlock(self.local_ptr, (max(1, rows), cols), "<f4" if dtype == torch.float32 else "<f8")
            self.tensor = torch.as_tensor(self.block, device=device)
            # ONE push stream, peers visited in the order rank+1, rank+2, ...: at any moment every GPU sends
            # to one peer and receives from one peer (a rotating permutation), so no destination is written by
            # seven sources at once.
            self.n_streams = max(1, min(4, int(os.environ.get("NNK_PEER_STREAMS", "1"))))
            self.streams = [torch.cuda.Stream(device=device) for _ in range(self.n_streams)]
            self.flag = torch.zeros(1, dtype=torch.int32, device=device)
        dist.barrier(group=group)

    def push(self, row0, n_rows, after_event):
        """Copy rows [row0, row0 + n_rows) of the local block into the same rows of every peer's block
        (copy engines, one stream per peer), once ``after_event`` (recorded behind the solve) has fired."""
        from . import _lib
        if n_rows == 0:
            return
        off, nbytes = row0 * self.row_bytes, n_rows * self.row_bytes
        for st in self.streams:
            st.wait_event(after_event)
        for k in range(1, self.world):  # stream i walks the offsets k = i+1, i+1+n, ...: n disjoint rotating permutations
            r = (self.rank + k) % self.world
            st = self.streams[(k - 1) % self.n_streams]
            _lib.check(_lib.lib.nnk_peer_copy(ctypes.c_void_p(self.peer_ptr[r] + off), ctypes.c_void_p(self.local_ptr + off),
                                              ctypes.c_size_t(nbytes), ctypes.c_void_p(st.cuda_stream)), "nnk_peer_copy")

    def finish(self, stream):
        """``stream`` waits for this rank's pushes, then for every other rank's (tiny NCCL all-reduce)."""
        import torch.distributed as dist
        for st in self.streams:
            stream.wait_stream(st)
        dist.all_reduce(self.flag, group=self.group)

    def close(self, collective=True):
        """Unmap the peers' blocks, then (after a barrier: nobody may still map a block that is about to be
        freed) release the own block.  Collective unless ``collective=False``."""
        import torch.distributed as dist

        from . import _lib
        for r, pp in enumerate(self.peer_ptr):
            if pp:
                _lib.lib.nnk_peer_close(ctypes.c_void_p(pp))
        self.peer_ptr = [None] * self.world
        if collective and dist.is_initialized():
            dist.barrier(group=self.group)
        if self.local_ptr:
            self.tensor = None
            _lib.lib.nnk_peer_free(ctypes.c_void_p(self.local_ptr))
            self.local_ptr = None


class ShardedBatch(object):
    """One rank's slice of a sharded batch, resident on its GPU in plan layout: ``means`` /
    ``variances`` ``(rows_local, D)`` (or a global ``(D,)`` variance), per-bucket launch metadata and
    the flat gathered result buffer (``transport``: "peer" = IPC-shared block, see :class:`PeerTransport`)."""

    def __init__(self, plan, rank, device, D_in, D_out, dtype, transport=None, group=None):
        import torch

        self.plan, self.rank, self.device = plan, int(rank), device
        self.D_in, self.D_out, self.dtype = int(D_in), int(D_out), dtype
        self.means = torch.zeros((max(1, plan.rows_local), D_in), dtype=dtype, device=device)
        self.variances = torch.ones((max(1, plan.rows_local), D_in), dtype=dtype, device=device)
        self.peer = None
        if transport == "peer" and plan.world > 1:
            try:
                self.peer = PeerTransport(plan.rows_total, D_out, dtype, device, group)
            except PeerUnavailable as e:  # agreed on by all ranks: everybody takes the NCCL all-gather instead
                if self.rank == 0:
                    import sys
                    sys.stderr.write("nnmnkwii_b200.sharding: %s; falling back to the NCCL all-gather\n" % e)
        if self.peer is not None:
            self.result = self.peer.tensor
        else:
            self.result = torch.zeros((max(1, plan.rows_total), D_out), dtype=dtype, device=device)
        self.meta = []
        for b in range(plan.n_buckets):
            ids = plan.members[b][self.rank]
            lens = plan.lengths[ids]
            self.meta.append({
                "n_utt": len(ids), "max_T": int(lens.max(initial=0)),
                "utt_off": torch.from_numpy(np.ascontiguousarray(plan.local_start[ids])).to(device),
                "out_off": torch.from_numpy(np.ascontiguousarray(plan.row_start[ids])).to(device),
                "utt_len": torch.from_numpy(lens.astype(np.int32)).to(device),
            })

    def load(self, means, variances):
        """Copy this rank's utterances out of full host arrays (contiguous row slices, no fancy indexing)."""
        import torch

        plan = self.plan
        off = np.concatenate([[0], np.cumsum(plan.lengths)])
        var1d = np.asarray(variances).ndim == 1
        if var1d:
            self.variances = torch.from_numpy(np.ascontiguousarray(variances)).to(device=self.device, dtype=self.dtype)
        for b in range(plan.n_buckets):
            for u in plan.members[b][self.rank]:
                a, e, l0 = int(off[u]), int(off[u + 1]), int(plan.local_start[u])
                self.means[l0:l0 + e - a].copy_(torch.from_numpy(means[a:e]), non_blocking=True)
                if not var1d:
                    self.variances[l0:l0 + e - a].copy_(torch.from_numpy(variances[a:e]), non_blocking=True)
        return self


class ShardedResult(object):
    """Gathered trajectories in shard order: utterance ``u`` is ``flat[row_start[u] : row_start[u] + lengths[u]]``."""

    def __init__(self, flat, plan, timings=None):
        self.flat, self.plan, self.timings = flat, plan, timings
        self.row_start, self.lengths = plan.row_start, plan.lengths

    def utterance(self, u):
        a = int(self.row_start[u])
        return self.flat[a:a + int(self.lengths[u])]

    def to_utterance_order(self):
        """``(sum_T, D_out)`` in the caller's utterance order (device segment copy; CPU tensors: slices)."""
        import torch

        lens = self.lengths
        dst = np.concatenate([[0], np.cumsum(lens)])[:-1].astype(np.int64)
        out = torch.empty((int(lens.sum()), self.flat.shape[1]), dtype=self.flat.dtype, device=self.flat.device)
        if not self.flat.is_cuda:
            for u in range(len(lens)):
                out[int(dst[u]):int(dst[u]) + int(lens[u])] = self.utterance(u)
            return out
        from . import _device as dev
        from . import _lib
        dv = self.flat.device
        src_t = torch.from_numpy(np.ascontiguousarray(self.row_start)).to(dv)
        dst_t = torch.from_numpy(dst).to(dv)
        len_t = torch.from_numpy(lens.astype(np.int32)).to(dv)
        step = 65535
        for s0 in range(0, len(lens), step):
            n = min(step, len(lens) - s0)
            _lib.check(_lib.lib.nnk_segment_copy(
                self.flat.data_ptr(), out.data_ptr(), self.flat.element_size(), self.flat.shape[1], self.flat.shape[1],
                out.shape[1], src_t[s0:].data_ptr(), dst_t[s0:].data_ptr(), len_t[s0:].data_ptr(), n,
                int(lens[s0:s0 + n].max(initial=0)), dev.current_stream_ptr(dv)), "nnk_segment_copy")
        return out


def _solve_bucket(batch, b, windows_c, chains, n_chain, status):
    """Enqueue the MLPG solve of bucket ``b`` on the current stream, trajectories written into the
    rank's slot of ``batch.result`` (the single-GPU CUDA path; no collective)."""
    from . import _device as dev

    m = batch.meta[b]
    if m["n_utt"] == 0 or m["max_T"] == 0:
        return
    var1d = batch.variances.dim() == 1
    dev.run_mlpg("fwd", means=batch.means, variances=batch.variances, rhs=None, out=batch.result,
                 offsets=m["utt_off"], lengths=m["utt_len"], order=None, chains=chains, n_chain=n_chain,
                 max_T=m["max_T"], windows_c=windows_c, in_ld=batch.D_in, var_ld=0 if var1d else batch.D_in, go_ld=0,
                 out_ld=batch.D_out, dtype_code=dev.torch_dtype_code(batch.dtype), go_f64=0, n_utt=m["n_utt"],
                 device=batch.device, check=False, out_offsets=m["out_off"], status=status)


def _gather_bucket(result, plan, b, rank, group):
    """All-gather of bucket ``b`` (in place: every rank's block already sits in its slot)."""
    import torch.distributed as dist

    cap, g0, world = plan.cap[b], plan.goff[b], plan.world
    if cap == 0:
        return None
    region = result[g0:g0 + world * cap]
    mine = result[g0 + rank * cap:g0 + (rank + 1) * cap]
    if dist.get_backend(group) == "nccl":
        return dist.all_gather_into_tensor(region.view(-1), mine.view(-1), group=group, async_op=True)
    parts = [region[r * cap:(r + 1) * cap] for r in range(world)]
    tmp = [p.clone() for p in parts]
    dist.all_gather(tmp, mine.clone(), group=group)
    for p, t in zip(parts, tmp):
        p.copy_(t)
    return None


def solve_sharded(batch, windows, layout, group=None, comm_stream=None, status=None):
    """One pass over a resident :class:`ShardedBatch`: per bucket, solve then all-gather, the gather of
    bucket ``b`` overlapping the solve of bucket ``b + 1``.  Returns the event that marks the end of
    the pass on the current stream (after it, ``batch.result`` holds every rank's trajectories)."""
    import torch
    import torch.distributed as dist

    from . import _device as dev
    from . import _lib

    plan, rank = batch.plan, batch.rank
    is_cuda = batch.result.is_cuda
    wc = _lib.make_windows(windows)
    chains = dev.chains_on_device(layout.chains, batch.device) if is_cuda else None
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    assert world == plan.world
    if not is_cuda or world == 1:
        for b in range(plan.n_buckets):
            _solve_bucket(batch, b, wc, chains, layout.n_chain, status)
            if world > 1:
                _gather_bucket(batch.result, plan, b, rank, group)
        return None
    cur = torch.cuda.current_stream(batch.device)
    if batch.peer is not None:  # copy-engine pushes over NVLink, overlapped with the next bucket's solve
        for b in range(plan.n_buckets):
            _solve_bucket(batch, b, wc, chains, layout.n_chain, status)
            done = torch.cuda.Event()
            done.record(cur)
            n_rows = int(plan.lengths[plan.members[b][rank]].sum())
            batch.peer.push(plan.goff[b] + rank * plan.cap[b], n_rows, done)
        batch.peer.finish(cur)
        return None
    if comm_stream is None:
        comm_stream = _comm_stream(batch.device)
    works = []
    for b in range(plan.n_buckets):
        _solve_bucket(batch, b, wc, chains, layout.n_chain, status)
        done = torch.cuda.Event()
        done.record(cur)
        with torch.cuda.stream(comm_stream):
            comm_stream.wait_event(done)
            works.append(_gather_bucket(batch.result, plan, b, rank, group))
    for w in works:  # join: the current stream waits for every gather
        if w is not None:
            w.wait()
    cur.wait_stream(comm_stream)
    return None


_comm_streams = {}


def _comm_stream(device):
    import torch
    key = str(device)
    if key not in _comm_streams:
        _comm_streams[key] = torch.cuda.Stream(device=device)
    return _comm_streams[key]


def default_transport(device):
    """"peer" on CUDA devices unless NNK_SHARD_TRANSPORT=nccl; the collective of the process group otherwise."""
    import os
    import torch
    if torch.device(device).type != "cuda":
        return None
    return "nccl" if os.environ.get("NNK_SHARD_TRANSPORT", "peer") == "nccl" else "peer"


def mlpg_batch_sharded(means, variances, windows, lengths, layout=None, group=None, device=None, n_buckets=4,
                       utterance_order=True, transport=None):
    """MLPG over a flat ``(sum_T, D)`` batch sharded by utterance over the ranks of ``group``.

    Every rank passes the SAME full host inputs (NumPy) and keeps only its own utterances on its GPU;
    every rank gets the full result: a ``(sum_T, D_out)`` tensor in utterance order
    (``utterance_order=True``) or the :class:`ShardedResult` in shard order.  For a batch that is
    already resident build a :class:`ShardedBatch` once and call :func:`solve_sharded` per pass.
    """
    import torch
    import torch.distributed as dist

    from . import paramgen as G

    rank, world = dist.get_rank(group), dist.get_world_size(group)
    lengths = np.asarray(lengths, dtype=np.int64)
    if layout is None:
        layout = G.StreamLayout.single(means.shape[1], len(windows))
    plan = ShardPlan(lengths, world, n_buckets)
    if device is None:
        from . import _device as dev
        dev.require_cuda()
        device = dev.cuda_device()
    dtype = torch.float32 if means.dtype == np.float32 and np.asarray(variances).dtype == np.float32 else torch.float64
    np_dt = np.float32 if dtype == torch.float32 else np.float64
    if transport is None:
        transport = default_transport(device)
    batch = ShardedBatch(plan, rank, device, layout.D_in, layout.D_out, dtype, transport=transport, group=group)
    batch.load(np.ascontiguousarray(means, dtype=np_dt), np.ascontiguousarray(variances, dtype=np_dt))
    status = torch.zeros(1, dtype=torch.int64, device=device) if batch.result.is_cuda else None
    solve_sharded(batch, windows, layout, group, status=status)
    if status is not None:
        from . import _device as dev
        dev.raise_if_failed(status)
    res = ShardedResult(batch.result, plan)
    if batch.peer is not None:  # the shared block is released here: hand back tensors that own their memory
        out = res.to_utterance_order() if utterance_order else ShardedResult(batch.result.clone(), plan)
        torch.cuda.synchronize(device)
        dist.barrier(group=group)  # nobody may still be pushing into a block that is about to be freed
        batch.peer.close()
        batch.result = None
        return out
    return res.to_utterance_order() if utterance_order else res


_ = ctypes
