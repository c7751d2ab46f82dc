"""Data-parallel gradient exchange for the training step: one process per GPU, images sharded by rank, parameter
gradients summed over ranks with an NCCL all-reduce (NVLink 5 / NVSwitch) per bucket while the backward chain is
still running.

Replaces the reference's single-process nn.DataParallel (train.py:65-71: replicate / scatter / gather on GPU 0 and
`reduce_add_coalesced` of the replica gradients).  Semantics match: the averaged gradient of the per-rank losses;
BatchNorm statistics stay per rank (the per-replica statistics of DataParallel); initial parameters and buffers are
rank 0's (DataParallel replicates GPU 0's module every step).

Design (one process per GPU):
  * every parameter gradient lives in ONE persistent fp32 arena (`GradArena`), laid out in the order the backward chain
    produces them (head first: layers3.0 = 47 MB and layers2.6/2.7 = 38 MB each come out at the very start).  The
    weight-gradient / BatchNorm-gradient kernels write their un-scaled results straight into their arena slots
    (`1 / (loss_scale * world)` is folded into that un-scaling), so there is no flatten copy, no copy back, no divide;
  * the arena is cut into buckets; when the last gradient of a bucket has been enqueued, the bucket's in-place
    all-reduce (`yb_allreduce_bucket`, the library's own NCCL communicator) is enqueued on a communication stream
    behind CUDA events recorded on the producing streams -- no host wait anywhere, so the whole step, collectives
    included, is capturable into one CUDA graph; the main stream joins the communication stream before the optimizer;
  * the communicator's rendezvous id travels through torch.distributed's store (plumbing); nothing on the data path
    uses torch.distributed.

CPU tensors (the world_size-2 `gloo` host-logic tests) take the same bucketing code with torch.distributed.all_reduce
as the transport.
"""
import ctypes

import torch
import torch.distributed as dist

from . import lib as _l

_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2, torch.int32: 3}


def _dist_ready():
    return dist.is_available() and dist.is_initialized()


class Communicator(object):
    """The library's NCCL communicator (include/yolo2_b200.h: yb_comm_*) for this process' GPU."""
    _seq = 0

    def __init__(self, device=None, process_group=None):
        if not _dist_ready():
            raise RuntimeError('ddp.Communicator: torch.distributed must be initialised (it carries the rendezvous id)')
        self.rank, self.world = dist.get_rank(process_group), dist.get_world_size(process_group)
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        lib = _l.load()
        ident = (ctypes.c_char * 128)()
        key = 'yb_comm_id_%d' % Communicator._seq
        Communicator._seq += 1
        store = dist.distributed_c10d._get_default_store()
        if self.rank == 0:
            _l.check(lib.yb_comm_unique_id(ident), 'yb_comm_unique_id')
            store.set(key, bytes(ident.raw))
        else:
            raw = store.get(key)
            ctypes.memmove(ident, raw, 128)
        handle = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _l.check(lib.yb_comm_init(ctypes.byref(handle), self.world, ident, self.rank), 'yb_comm_init')
        self.handle = handle
        self.bytes_reduced = 0
        # Every collective of this communicator is issued on ONE dedicated stream; callers on other streams are ordered against it with
        # CUDA events (fork / join).  NCCL then never has to serialise the communicator across streams itself, which is what keeps
        # eager use, CUDA-graph capture and their mixture legal (a captured collective must not depend on uncaptured work elsewhere).
        self.stream = torch.cuda.Stream(device=self.device)

    def _stream(self, stream):
        return ctypes.c_void_p(self.stream.cuda_stream)

    def _fork(self, caller):
        ev = torch.cuda.Event()
        ev.record(caller)
        self.stream.wait_event(ev)

    def _join(self, caller):
        ev = torch.cuda.Event()
        ev.record(self.stream)
        caller.wait_event(ev)

    def all_reduce(self, tensor, stream=None):
        """In-place sum over ranks.  stream=None: ordered after the work already enqueued on torch's current stream, and that stream
        waits for the result (asynchronously).  stream=self.stream: the caller has done the ordering itself (gradient buckets)."""
        if not (tensor.is_cuda and tensor.is_contiguous()):
            raise RuntimeError('Communicator.all_reduce: contiguous CUDA tensor required')
        caller = None
        if stream is not self.stream:
            caller = torch.cuda.current_stream(self.device) if stream is None else stream
            self._fork(caller)
        _l.check(_l.load().yb_allreduce_bucket(self.handle, ctypes.c_void_p(tensor.data_ptr()), tensor.numel(), _DTYPES[tensor.dtype],
                                               self._stream(None)), 'yb_allreduce_bucket')
        if caller is not None:
            tensor.record_stream(self.stream)
            self._join(caller)
        self.bytes_reduced += tensor.numel() * tensor.element_size()
        return tensor

    def broadcast(self, tensor, root=0, stream=None):
        """Rank `root`'s values into `tensor` on every rank; ordered against torch's current stream like all_reduce(stream=None)."""
        if not (tensor.is_cuda and tensor.is_contiguous()):
            raise RuntimeError('Communicator.broadcast: contiguous CUDA tensor required')
        caller = torch.cuda.current_stream(self.device)
        self._fork(caller)
        try:
            return self._broadcast(tensor, root)
        finally:
            self._join(caller)

    def _broadcast(self, tensor, root):
        stream = None
        t = tensor
        if t.dtype not in _DTYPES:                      # e.g. int64 num_batches_tracked: ship the raw words
            t = t.view(torch.int32) if t.element_size() % 4 == 0 and t.dim() > 0 else None
        if t is None:
            tmp = tensor.reshape(1).view(torch.int32)
            _l.check(_l.load().yb_broadcast_buffer(self.handle, ctypes.c_void_p(tmp.data_ptr()), tmp.numel(), 3, root, self._stream(stream)),
                     'yb_broadcast_buffer')
            return tensor
        _l.check(_l.load().yb_broadcast_buffer(self.handle, ctypes.c_void_p(t.data_ptr()), t.numel(), _DTYPES[t.dtype], root, self._stream(stream)),
                 'yb_broadcast_buffer')
        return tensor

    def destroy(self):
        """Call after every CUDA graph that captured a collective of this communicator has been destroyed."""
        if self.handle is not None and self.handle.value:
            torch.cuda.synchronize(self.device)
            _l.check(_l.load().yb_comm_destroy(self.handle), 'yb_comm_destroy')
        self.handle = None


class GradArena(object):
    """One flat fp32 buffer holding every parameter gradient, in backward (production) order, cut into buckets."""

    def __init__(self, named_shapes, device, bucket_bytes=32 << 20):
        self.names = [n for n, _ in named_shapes]
        sizes = [int(torch.Size(s).numel()) for _, s in named_shapes]
        # 256-byte aligned slots: vectorised kernels write them, NCCL reads whole buckets
        offs, off = [], 0
        for n in sizes:
            offs.append(off)
            off += (n + 63) // 64 * 64
        self.flat = torch.zeros(off, dtype=torch.float32, device=device)
        self.views = {name: self.flat[o:o + n].view(shape) for (name, shape), o, n in zip(named_shapes, offs, sizes)}
        self.buckets = []          # (start, end, [names])
        start, names = 0, []
        for i, name in enumerate(self.names):
            names.append(name)
            end = offs[i + 1] if i + 1 < len(offs) else off
            if (end - start) * 4 >= bucket_bytes or i + 1 == len(self.names):
                self.buckets.append((start, end, names))
                start, names = end, []
        self.bucket_of = {name: bi for bi, (_, _, ns) in enumerate(self.buckets) for name in ns}

    def bucket_tensor(self, bi):
        s, e, _ = self.buckets[bi]
        return self.flat[s:e]


class GradientAllReducer(object):
    """Bucketed gradient all-reduce.

    GPU (arena mode): `attach(arena)` once; the backward chain calls `on_grad(name, streams=...)` after enqueueing the
    kernel that writes `arena.views[name]`; a bucket whose gradients are all enqueued is all-reduced on the communication
    stream; `finish()` joins.  Gradients arrive pre-divided by the world size (`grad_divisor`).
    CPU (host-logic tests over gloo): `on_grad(name, tensor)` with arbitrary tensors, flattened per bucket."""

    def __init__(self, bucket_bytes=32 << 20, process_group=None, communicator=None):
        self.bucket_bytes = int(bucket_bytes)
        self.group = process_group
        self.comm = communicator
        self.world = communicator.world if communicator is not None else (dist.get_world_size(process_group) if _dist_ready() else 1)
        self.comm_stream = None
        self.arena = None
        self._left = None
        self._launched = 0
        self._bucket, self._bucket_size, self._pending = [], 0, []
        self.bytes_reduced = 0
        self.steps = 0          # finish() calls executed by Python (CUDA-graph replays do not come through here)

    @property
    def grad_divisor(self):
        """The trainer folds 1 / world into the un-scaling of the gradients it writes into the arena."""
        return float(self.world)

    # ---- arena mode (GPU) ---------------------------------------------------------------------------
    def attach(self, arena):
        if self.comm is None and self.world > 1:
            self.comm = Communicator(arena.flat.device, self.group)
        self.arena = arena
        self.comm_stream = self.comm.stream if self.comm is not None else torch.cuda.Stream(device=arena.flat.device)
        self._reset()

    def _reset(self):
        self._left = [len(names) for _, _, names in self.arena.buckets]
        self._launched = 0

    def on_grad(self, name, grad=None, streams=()):
        """`name`'s gradient has been enqueued.  Arena mode: `streams` = every stream that may carry kernels writing this
        bucket (main + weight-gradient side stream)."""
        if self.world == 1:
            return
        if self.arena is None:
            return self._on_grad_cpu(name, grad)
        bi = self.arena.bucket_of[name]
        self._left[bi] -= 1
        if self._left[bi] == 0:
            self._launch(bi, streams)

    def _launch(self, bi, streams):
        dev = self.arena.flat.device
        streams = [s for s in streams if s is not None] or [torch.cuda.current_stream(dev)]
        what = 'start'
        try:
            for i, st in enumerate(streams):
                what = 'event on producing stream %d of %d (%r)' % (i, len(streams), st)
                ev = torch.cuda.Event()
                ev.record(st)
                self.comm_stream.wait_event(ev)
            buf = self.arena.bucket_tensor(bi)
            what = 'all-reduce'
            self.comm.all_reduce(buf, stream=self.comm_stream)
        except Exception as ex:
            raise RuntimeError('gradient bucket %d: %s failed (capturing: %s): %s' % (bi, what, torch.cuda.is_current_stream_capturing(), ex)) from ex
        self.bytes_reduced += buf.numel() * 4
        self._launched += 1

    def finish(self):
        """All buckets reduced before anything enqueued on the current stream after this call (optimizer, clipping)."""
        if self.world == 1:
            return
        self.steps += 1
        if self.arena is None:
            return self._finish_cpu()
        if self._launched != len(self.arena.buckets):
            missing = [names for left, (_, _, names) in zip(self._left, self.arena.buckets) if left > 0]
            self._reset()
            raise RuntimeError('gradient all-reduce: buckets never completed (missing gradients among %s)' % (missing[:2],))
        torch.cuda.current_stream(self.arena.flat.device).wait_stream(self.comm_stream)
        self._reset()

    def broadcast_module(self, module, root=0):
        """Parameters and buffers of `module` become rank `root`'s (what DataParallel's per-step replicate guarantees)."""
        if self.world == 1:
            return
        if self.comm is None:
            dev = next(module.parameters()).device
            self.comm = Communicator(dev, self.group)
        with torch.no_grad():
            for t in list(module.parameters()) + list(module.buffers()):
                self.comm.broadcast(t.data if t.is_contiguous() else t.data.contiguous(), root)

    def destroy(self):
        if self.comm is not None:
            self.comm.destroy()
            self.comm = None

    # ---- CPU tensors over torch.distributed (gloo): host-logic tests ------------------------------------
    def _on_grad_cpu(self, name, grad):
        if grad.is_cuda:
            raise RuntimeError('GradientAllReducer: CUDA gradients go through the arena (attach()); there is no unfused GPU path')
        self._bucket.append((name, grad))
        self._bucket_size += grad.numel() * grad.element_size()
        if self._bucket_size >= self.bucket_bytes:
            self._flush_cpu()

    def _flush_cpu(self):
        if not self._bucket:
            return
        items, self._bucket, self._bucket_size = self._bucket, [], 0
        flat = torch.cat([g.reshape(-1) for _, g in items])
        work = dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=self.group, async_op=True)
        self.bytes_reduced += flat.numel() * flat.element_size()
        self._pending.append((flat, items, work))

    def _finish_cpu(self):
        self._flush_cpu()
        for flat, items, work in self._pending:
            work.wait()
            off = 0
            for _, g in items:
                n = g.numel()
                g.copy_(flat[off:off + n].view_as(g)).mul_(1.0 / self.world)
                off += n
        self._pending = []


_DEFAULT = None
_LOCAL_ONLY = 0


class local_only(object):
    """Context: this rank steps on its own shard with no collective at all (compute-only timing of a data-parallel step)."""

    def __enter__(self):
        global _LOCAL_ONLY
        _LOCAL_ONLY += 1

    def __exit__(self, *exc):
        global _LOCAL_ONLY
        _LOCAL_ONLY -= 1
        return False


def default_reducer(create=True):
    """Process-wide reducer used by `train.iterate` / `model.loss` when torch.distributed is initialised with world > 1."""
    global _DEFAULT
    if _LOCAL_ONLY:
        return None
    if _DEFAULT is None and create and _dist_ready() and dist.get_world_size() > 1:
        _DEFAULT = GradientAllReducer()
    return _DEFAULT


def set_default_reducer(reducer):
    global _DEFAULT
    _DEFAULT = reducer


def shutdown():
    """Destroy the default reducer's communicator (after the CUDA graphs that captured its collectives are gone)."""
    global _DEFAULT
    if _DEFAULT is not None:
        _DEFAULT.destroy()
        _DEFAULT = None


def global_mean_factor(local_count, process_group=None):
    """Weight that turns a per-rank MEAN over `local_count` items into this rank's share of the mean over the items of
    ALL ranks: local_count / sum_over_ranks(local_count) (one scalar all-reduce).

    Used for the class term of the region loss (`train/cross_entropy = 1`): the reference computes the loss on the
    batch gathered from all replicas (train.py:344-347), where that term is a mean over the positives of the whole
    batch and is then divided by cnt = B_global * cells * A (model/__init__.py:162-166).  With images sharded over
    ranks, (sum_r CE_r / N_r) * f_r / cnt_local averaged over ranks equals (sum CE / N_total) / cnt_global exactly
    when f_r = N_r / N_total, because cnt_global = world * cnt_local.  The sum-type terms need no correction.
    `local_count`: 0-dim tensor.  CUDA tensors use the library communicator of the default reducer (capturable);
    CPU tensors torch.distributed (gloo).  Returns a float32 0-dim tensor."""
    n = local_count.detach().to(torch.float32).reshape(())
    if _LOCAL_ONLY or not _dist_ready() or dist.get_world_size(process_group) == 1:
        return torch.ones_like(n)
    total = n.clone()
    if n.is_cuda:
        red = default_reducer()
        if red.comm is None:
            red.comm = Communicator(n.device, process_group)
        red.comm.all_reduce(total.reshape(1))
    else:
        dist.all_reduce(total, op=dist.ReduceOp.SUM, group=process_group)
    return n / total.clamp(min=1.0)


def shard_range(total, rank, world):
    """Contiguous [start, end) of `total` images owned by `rank` (remainder spread over the first ranks)."""
    base, rem = divmod(total, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)
