"""Data-parallel plumbing: the only distributed step of the path is the gradient all-reduce
(reference: apex DistributedDataParallel(model, delay_allreduce=True) at train_tasks.py:497 — one flattened
all-reduce after backward, averaged over the world size; apex's default delay_allreduce=False at train_concap.py:513 —
bucketed all-reduces overlapped with the backward; batch split per rank at task_utils.py:435-437).

Here the gradients already live in ONE flat fp32 buffer (engine.ParamStore.grad), so the all-reduce runs in place
on contiguous, fixed-address buckets (NCCL over NVLink/NVSwitch on GPUs; gloo in the CPU tests)."""
import torch
import torch.distributed as dist

from .engine import _pad8


def trainable_ranges(ps, frozen):
    """Coalesced [lo, hi) ranges of the flat gradient buffer of ParamStore `ps` owned by parameters not in `frozen` (entry names),
    each entry with its padding: with nothing frozen, the whole buffer."""
    out = []
    for name, (off, shape) in ps.entries.items():
        if name in frozen:
            continue
        n = 1
        for d in shape:
            n *= d
        hi = off + _pad8(n)
        if out and out[-1][1] == off:
            out[-1][1] = hi
        else:
            out.append([off, hi])
    return [tuple(r) for r in out]


def shard_slices(table, world):
    """Per bucket (lo, hi) of a bucket table: its `world` slices [(lo_r, hi_r)] for ranks r = 0 .. world - 1, cut at multiples of
    per = ceil((hi - lo) / world) rounded up to 4 elements (the chunk-table alignment of optim.build_chunks), so the bucket padded to
    world * per elements splits into equal parts; the last slices may be short or empty. A function of the table alone: every rank
    computes the same slices (pure host logic, unit-tested on CPU)."""
    out = []
    for lo, hi in table:
        per = (-(-(hi - lo) // world) + 3) // 4 * 4
        out.append(tuple((min(lo + r * per, hi), min(lo + (r + 1) * per, hi)) for r in range(world)))
    return tuple(out)


class FlatGradAllReducer:
    def __init__(self, flat_grad, n_buckets=8, group=None, align=1024):
        self.flat = flat_grad
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        # a sharded optimizer (optim shard_state=True) turns the exchange into a reduce-scatter: each rank receives the average of
        # its own slice of every bucket (self.slices) only
        self.scatter = False
        self._scattered = set()   # buckets reduce-scattered since the sharded optimizer's last step
        n = flat_grad.numel()
        step = max(align, (n + n_buckets - 1) // n_buckets)
        step = (step + align - 1) // align * align
        self._bounds = [(i, min(i + step, n)) for i in range(0, n, step)]
        self.set_ranges([(0, n)])
        # NCCL has a fused average; gloo only sums
        self.use_avg = dist.is_initialized() and dist.get_backend(group) == "nccl"
        self._comm = None        # communication stream of overlapped_backward

    def set_ranges(self, ranges):
        """Restricts allreduce() to the flat ranges [lo, hi) of `ranges` (the trainable parameters; frozen ones have no gradient
        to exchange): every bucket is cut to its parts inside them. The whole buffer gives the full buckets. self.table: their
        (lo, hi) in ascending order, the same on every rank (Plan.bucket_schedule is keyed on it)."""
        self.table = tuple((max(lo, a), min(hi, b)) for (lo, hi) in self._bounds for (a, b) in ranges if min(hi, b) > max(lo, a))
        self.buckets = [self.flat[lo:hi] for lo, hi in self.table]
        self.slices = shard_slices(self.table, self.world)

    def allreduce(self, stream=None):
        """Averages the flat gradient buffer over all ranks, bucket by bucket (in place). With `scatter` (a sharded optimizer): each
        bucket is reduce-scattered instead, and only this rank's slices hold the average."""
        if self.world == 1:
            return
        if self.scatter:
            for lo, hi in self.table:
                self.reduce_scatter_range(lo, hi, async_op=False)
            return
        for b in self.buckets:
            if self.use_avg:
                dist.all_reduce(b, op=dist.ReduceOp.AVG, group=self.group)
            else:
                dist.all_reduce(b, op=dist.ReduceOp.SUM, group=self.group)
                b.div_(self.world)

    def allreduce_range(self, lo, hi, async_op=True):
        """Averages flat[lo:hi] over all ranks; returns the async work handle (or None for world 1). Used by the
        overlapped step: backward finishes the buffer from its end, ranges are reduced while backward continues."""
        if self.world == 1 or hi <= lo:
            return None
        if self.scatter:
            return self.reduce_scatter_range(lo, hi, async_op)
        t = self.flat[lo:hi]
        if self.use_avg:
            return dist.all_reduce(t, op=dist.ReduceOp.AVG, group=self.group, async_op=async_op)
        w = dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group, async_op=False)
        t.div_(self.world)
        return w

    def _padded(self, t, lo, hi):
        """(the bucket [lo, hi) of the flat tensor t as world equal parts, this rank's part, whether that is a staging copy): the
        bucket itself when it splits evenly, else a zero-padded copy."""
        sl = shard_slices(((lo, hi),), self.world)[0]
        per = sl[0][1] - sl[0][0]
        if per * self.world == hi - lo:
            b = t[lo:hi]
        else:
            b = torch.zeros(per * self.world, dtype=t.dtype, device=t.device)
        return b, b[self.rank * per:(self.rank + 1) * per], b.data_ptr() != t[lo:].data_ptr()

    def reduce_scatter_range(self, lo, hi, async_op=True):
        """Averages this rank's slice (self.slices) of the bucket flat[lo:hi] over all ranks, in place; returns the work handle (None
        for world 1). The rest of the bucket keeps this rank's own gradient. NCCL: reduce_scatter_tensor with its fused average,
        asynchronous. gloo sums only, and its reduce-scatter takes CPU tensors: a CUDA bucket goes through a host copy, and only
        this rank's slice is copied back (synchronously)."""
        if self.world == 1 or hi <= lo:
            return None
        if (lo, hi) in self._scattered:
            raise RuntimeError("shard_state: a second synchronised backward before the optimizer step would average this rank's "
                               "slice again; accumulate micro-batches under model.no_sync() and step once per synchronised backward")
        self._scattered.add((lo, hi))
        if self.use_avg or self.flat.device.type == "cpu":
            return self._reduce_scatter(self.flat, lo, hi, async_op)
        host = self.flat[lo:hi].cpu()
        self._reduce_scatter(host, 0, hi - lo, False)
        a, e = shard_slices(((lo, hi),), self.world)[0][self.rank]
        self.flat[a:e].copy_(host[a - lo:e - lo])
        return None

    def _reduce_scatter(self, t, lo, hi, async_op):
        """reduce_scatter_range on the elements [lo, hi) of t (the flat buffer, or a host copy of one bucket)."""
        b, mine, staged = self._padded(t, lo, hi)
        if staged:
            b[:hi - lo].copy_(t[lo:hi])
        op = dist.ReduceOp.AVG if self.use_avg else dist.ReduceOp.SUM
        w = dist.reduce_scatter_tensor(mine, b, op=op, group=self.group, async_op=async_op and not staged and self.use_avg)
        if not self.use_avg:
            mine.div_(self.world)
        if staged:
            if w is not None:
                w.wait()
            a, e = shard_slices(((lo, hi),), self.world)[0][self.rank]
            t[a:e].copy_(mine[:e - a])
        return w

    def reset_exchange(self):
        """The reduce-scattered gradient was consumed (a sharded step) or discarded (zero_grad): the next backward exchanges again."""
        self._scattered.clear()

    def all_gather_range(self, t, lo, hi, async_op=True):
        """Every rank's slice of the bucket [lo, hi) of the flat tensor t (same layout as the gradient buffer: the weights) to every
        rank, in place; returns the work handle (None for world 1). NCCL: all_gather_into_tensor, asynchronous. gloo: a CUDA bucket
        goes through a host copy (synchronously)."""
        if self.world == 1 or hi <= lo:
            return None
        if self.use_avg or t.device.type == "cpu":
            return self._all_gather(t, lo, hi, async_op)
        host = t[lo:hi].cpu()
        self._all_gather(host, 0, hi - lo, False)
        t[lo:hi].copy_(host)
        return None

    def _all_gather(self, t, lo, hi, async_op):
        """all_gather_range on the elements [lo, hi) of t (a flat buffer, or a host copy of one bucket)."""
        b, mine, staged = self._padded(t, lo, hi)
        if staged:
            a, e = shard_slices(((lo, hi),), self.world)[0][self.rank]
            mine[:e - a].copy_(t[a:e])
        w = dist.all_gather_into_tensor(b, mine, group=self.group, async_op=async_op and not staged and self.use_avg)
        if staged:
            if w is not None:
                w.wait()
            t[lo:hi].copy_(b[:hi - lo])
        return w

    def allreduce_range_sync(self, lo, hi):
        """flat[lo:hi] averaged over all ranks, enqueued on the CURRENT stream (used under CUDA-graph capture)."""
        if self.world == 1 or hi <= lo:
            return
        t = self.flat[lo:hi]
        if self.use_avg:
            dist.all_reduce(t, op=dist.ReduceOp.AVG, group=self.group)
        else:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
            t.div_(self.world)

    def comm_stream(self):
        """The communication stream of the overlapped backward (created on first use)."""
        if self._comm is None:
            self._comm = torch.cuda.Stream(device=self.flat.device)
        return self._comm

    def overlapped_backward(self, plan):
        """Runs the backward of `plan` in the pieces of plan.bucket_schedule(self.table) and averages each bucket (allreduce_range,
        asynchronous) on a communication stream as soon as the piece that finishes it has run, so the exchange overlaps the rest of
        the backward. Returns once the current stream waits for every collective: work queued after it (an optimizer step, a
        gradient-norm clip) sees the averaged buffer."""
        comm = self.comm_stream()
        works = []

        def handover(ranges):
            works.extend(self.allreduce_range(lo, hi) for lo, hi in ranges)
        plan.run_backward_pieces(self.table, handover, comm)
        torch.cuda.current_stream().wait_stream(comm)
        for w in works:
            if w is not None:
                w.wait()

    def broadcast_params(self, flat_params, src=0):
        """Rank-`src` parameters to every rank (what apex DDP does at wrap time)."""
        if self.world > 1:
            dist.broadcast(flat_params, src=src, group=self.group)


class DistributedDataParallel:
    """Drop-in for `apex.parallel.DistributedDataParallel(model, delay_allreduce=...)` as the reference uses it
    (train_tasks.py:490-497, train_concap.py:513): rank 0's parameters are broadcast at wrap time and every `loss.backward()`
    averages the flat fp32 gradient buffer over the world, restricted to the ranges of the trainable parameters. Not an nn.Module
    wrapper with hooks: the engine's backward calls the reducer itself. `.module` is the wrapped model, calls and attributes
    (model.no_sync()) are forwarded.

    delay_allreduce=True (the default here, and train_tasks.py's choice): one all-reduce of the buffer after the backward.
    delay_allreduce=False (apex's default): the buckets of the buffer are averaged in descending offset order while the backward
    still runs, each as soon as no later backward op writes it (Plan.bucket_schedule). Both modes send the same messages, so they
    give bitwise the same parameters. A world of one, and a plan with anomaly checks (whose NaN report must come before any
    collective), take the first path. Backwards under model.no_sync() exchange nothing in either mode."""

    def __init__(self, model, delay_allreduce=True, n_buckets=8, group=None):
        self.module = model
        eng = model.engine
        self.reducer = FlatGradAllReducer(eng.ps.grad, n_buckets=n_buckets, group=group)
        self.reducer.broadcast_params(eng.ps.flat)
        eng.shadow_clean = False
        model._ddp_reducer = self.reducer
        model._ddp_overlap = not delay_allreduce
        # only the ranges of trainable parameters are exchanged; the model updates them when a requires_grad flag changes
        model._ddp_set_ranges = self.reducer.set_ranges
        self.reducer.set_ranges(model._trainable_ranges())

    def __call__(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    def __getattr__(self, name):
        return getattr(self.module, name)


def shard_batch(global_batch, rank, world):
    """Per-rank batch like the reference: batch_size // world_size samples each (task_utils.py:435-437)."""
    per = global_batch // world
    return rank * per, per
