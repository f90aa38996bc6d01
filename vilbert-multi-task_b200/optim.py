"""Fused multi-tensor AdamW and RAdam on the engine's flat parameter / gradient buffers (SURVEY.md §8 f2).

Drop-ins for the two optimizers the reference's training driver offers (train_tasks.py:401-428, `--optim`):

    optimizer = AdamW(optimizer_grouped_parameters, lr=base_lr, correct_bias=False)        # pytorch_transformers 1.0.0
 -> optimizer = FusedAdamW(optimizer_grouped_parameters, lr=base_lr, correct_bias=False, model=model)

    optimizer = RAdam(optimizer_grouped_parameters, lr=base_lr)                             # vilbert/optimization.py
 -> optimizer = FusedRAdam(optimizer_grouped_parameters, lr=base_lr, model=model)

Same constructor arguments and defaults, same `param_groups` list of dicts (one group per tensor with its own lr /
weight_decay in the reference; the warm-up schedulers of train_tasks.py:431-437 mutate group["lr"] exactly as before).
step() is ONE kernel launch over the flat buffers (csrc/vb_optim.cu) that also writes the 16-bit tensor-core operand copy
of the updated weights and zeroes the gradients, so the training step needs no separate weight cast and the
`model.zero_grad()` that follows optimizer.step() in the reference (train_tasks.py:551) finds the buffer already clean.

`max_grad_norm=c` (apex FusedAdam's keyword, passed by the reference's --fp16 optimizer, train_concap.py:452-457) clips the
global L2 norm of the trainable gradients to c as torch.nn.utils.clip_grad_norm_ does, and skips a step whose gradient holds a
NaN or an inf, both decided on the device: one norm launch over the gradient buffer writes a small record that the optimizer
launch reads, so nothing is read back to the host.

`with optimizer.step_in_backward(): loss.backward()` runs the same step while the backward runs: each bucket of the flat
buffers is updated on a side stream as soon as no later backward op touches it (INTEGRATION.md §1k, DESIGN.md §4d).

`shard_state=True` with model=ddp.DistributedDataParallel(...) shards the moments over the data-parallel ranks (ZeRO stage 1,
INTEGRATION.md §1a, DESIGN.md §4c): the backward reduce-scatters each gradient bucket instead of all-reducing it, each rank steps
its own slice against moments it stores for that slice only, and the updated fp32 weights are all-gathered.
"""
import contextlib
import ctypes as C

import numpy as np
import torch

from . import _lib as L

# The step in the backward, chosen by measurement on an H100 (DESIGN.md §4d, tools/step_in_backward_probe.py): the number of
# buckets a single process cuts the trainable ranges into (as ddp.FlatGradAllReducer cuts them), and the CTA cap of each
# bucket's launch (vb_adamw_step_capped / vb_radam_step_capped; 0: the 8 x SMs grid of step()).
STEP_BUCKETS = 4
STEP_MAX_CTAS = 264

_GROUP_DT = np.dtype([("lr", "<f4"), ("beta1", "<f4"), ("beta2", "<f4"), ("eps", "<f4"), ("weight_decay", "<f4"), ("correct_bias", "<i4"),
                      ("one_minus_beta1", "<f4"), ("one_minus_beta2", "<f4")])


def group_row(lr, betas, eps, weight_decay, correct_bias=False):
    """The vb_adamw_group row of one param group. 1 - beta is formed here from the Python floats and rounded to fp32 once, as the
    reference's fp32 torch ops see `1.0 - beta2`: the kernel forming 1 - fp32(beta2) instead would shrink every second-moment
    increment by 1.3e-5 at beta2 = 0.999."""
    return (lr, betas[0], betas[1], eps, weight_decay, 1 if correct_bias else 0, 1.0 - betas[0], 1.0 - betas[1])


def build_chunks(ranges, chunk=32768):
    """ranges: [(flat offset, numel, group index)] -> (start int64[], count int32[], group int32[]): contiguous pieces of at
    most `chunk` elements that never cross a tensor boundary (pure host logic, unit-tested on CPU)."""
    assert chunk % 4 == 0
    st, cn, gr = [], [], []
    for off, n, gi in ranges:
        if off % 4:
            raise ValueError("parameter tensors must start on a 4-element boundary of the flat buffer")
        for s in range(0, n, chunk):
            st.append(off + s); cn.append(min(chunk, n - s)); gr.append(gi)
    return np.asarray(st, np.int64), np.asarray(cn, np.int32), np.asarray(gr, np.int32)


def shard_state_layout(slices, rank):
    """slices: ddp.shard_slices of a bucket table -> (((lo, hi, state offset) of this rank's slice of every bucket), total): the
    layout of the rank's compact moment buffers, its slices back to back (pure host logic, unit-tested on CPU)."""
    out, at = [], 0
    for sl in slices:
        lo, hi = sl[rank]
        out.append((lo, hi, at))
        at += hi - lo
    return tuple(out), at


def shard_chunks(ranges, layout, chunk=32768):
    """ranges: [(flat offset, numel, group index)] of the trainable tensors; layout: shard_state_layout -> per slice (start int64[],
    state start int64[], count int32[], group int32[]): the chunk table (build_chunks) of the parts of the ranges inside the slice,
    and where each chunk's moments start in the compact buffers (pure host logic, unit-tested on CPU)."""
    out = []
    for lo, hi, base in layout:
        st, cn, gr = build_chunks([(max(off, lo), min(off + n, hi) - max(off, lo), gi) for off, n, gi in ranges
                                   if off < hi and off + n > lo], chunk)
        out.append((st, st - lo + base, cn, gr))
    return out


def unshard_state(compacts, layouts, numel):
    """The flat-layout buffer of `numel` elements assembled from every rank's compact buffer (compacts[r] in layouts[r], as
    shard_state_layout gives them); elements outside every slice are 0. The host-side statement of what the sharded
    optimizer's state_dict() gathers on the device."""
    full = torch.zeros(numel, dtype=compacts[0].dtype)
    for buf, layout in zip(compacts, layouts):
        for lo, hi, base in layout:
            full[lo:hi] = buf[base:base + hi - lo]
    return full


def bucket_chunks(ranges, table, chunk=32768):
    """ranges: [(flat offset, numel, group index)] of the trainable tensors (as build_chunks takes them); table: disjoint (lo, hi)
    buckets of the flat buffer in ascending order -> per bucket the chunk table (build_chunks) of the parts of the ranges inside it:
    chunks are split at bucket edges, which changes nothing per element. Every element of the ranges lies in exactly one bucket's
    table; one outside every bucket raises ValueError (pure host logic, unit-tested on CPU)."""
    out = [build_chunks([(max(off, lo), min(off + n, hi) - max(off, lo), gi) for off, n, gi in ranges if off < hi and off + n > lo],
                        chunk) for lo, hi in table]
    if sum(int(cn.sum()) for _, cn, _ in out) != sum(n for _, n, _ in ranges):
        raise ValueError("bucket_chunks: trainable elements lie outside every bucket")
    return out


class _ShardedState:
    """The moments of a fused optimizer built with shard_state=True, sharded over the ranks of the reducer's group (ZeRO stage 1).

    The reducer's exchange becomes a reduce-scatter (ddp.FlatGradAllReducer.scatter): after the synchronised backward, this
    rank's slice of every bucket (ddp.shard_slices) holds the averaged gradient. opt.exp_avg / exp_avg_sq hold the moments of
    those slices back to back (shard_state_layout). A step is one vb_*_step_sharded launch over the slices' chunk tables (which
    writes the slices' 16-bit copies and zeroes their gradient), the rest of each bucket's gradient zeroed, the fp32 weights
    all-gathered bucket by bucket, and the 16-bit copies of the gathered parts re-cast. When the bucket table changes (parameters
    frozen or unfrozen) the moments move to the new slices through one gather of the full moments; the moments of tracked
    parameters outside the table are kept whole on every rank (`parked`) until they are trainable again."""

    def __init__(self, opt, red):
        self.opt, self.red = opt, red
        red.scatter = True
        self.table = self.key = None
        self.parked = {}
        self._launches = {}
        ps = opt.engine.ps
        self.norm_sum = torch.zeros(1, dtype=torch.float64, device=ps.flat.device)
        self._set_layout(None)

    # ------------------------------------------------------------------ layout
    def sync(self):
        """Follows the reducer's bucket table and the optimizer's trainable set (collective when the table changed)."""
        opt = self.opt
        opt._refresh_trainable()
        key = (self.red.table, opt._trainable_key)
        if key == self.key:
            return
        if self.red.table != self.table:
            self._set_layout(self.full_moments())
        self._build_chunks()
        self.key = key

    def _set_layout(self, full):
        """This rank's compact moments under the reducer's current table, taken from the flat-layout pair `full` (None: zeros)."""
        opt, red, ps = self.opt, self.red, self.opt.engine.ps
        self.table = red.table
        self.layout, total = shard_state_layout(red.slices, red.rank)
        m, v = (torch.zeros(max(total, 4), dtype=torch.float32, device=ps.flat.device) for _ in range(2))
        if full is not None:
            for lo, hi, base in self.layout:
                m[base:base + hi - lo].copy_(full[0][lo:hi])
                v[base:base + hi - lo].copy_(full[1][lo:hi])
        self.parked = {}
        for _, off, n, _ in opt._tracked:
            if not any(lo < off + n and off < hi for lo, hi in self.table):
                self.parked[(off, n)] = tuple(f[off:off + n].clone() if full is not None else
                                              torch.zeros(n, dtype=torch.float32, device=ps.flat.device) for f in (full or (None, None)))
        opt.exp_avg, opt.exp_avg_sq = m, v
        self.key = None
        self._launches.clear()

    def _build_chunks(self):
        opt, dev = self.opt, self.opt.engine.ps.flat.device
        self.per_bucket = shard_chunks(opt._trainable_ranges(), self.layout, opt._chunk)
        cols = [np.concatenate([b[i] for b in self.per_bucket]) if self.per_bucket else np.zeros(0, dt)
                for i, dt in enumerate((np.int64, np.int64, np.int32, np.int32))]
        self.start, self.state_start, self.count, self.group = (torch.from_numpy(c).to(dev) for c in cols)
        self.n_chunks = len(cols[0])
        self.partials = torch.zeros(max(self.n_chunks, 1), dtype=torch.float64, device=dev)
        self._launches.clear()

    def full_moments(self):
        """(exp_avg, exp_avg_sq) in the flat layout on every rank: each rank's slices all-gathered, the parked moments added
        (collective)."""
        ps, out = self.opt.engine.ps, []
        for buf in (self.opt.exp_avg, self.opt.exp_avg_sq):
            f = torch.zeros_like(ps.flat)
            for lo, hi, base in self.layout:
                f[lo:hi].copy_(buf[base:base + hi - lo])
            for lo, hi in self.table:
                self.red.all_gather_range(f, lo, hi, async_op=False)
            out.append(f)
        for (off, n), (m, v) in self.parked.items():
            out[0][off:off + n].copy_(m)
            out[1][off:off + n].copy_(v)
        return out

    # ------------------------------------------------------------------ stepping
    def _head(self, start, state_start, count, group, n):
        ps, opt = self.opt.engine.ps, self.opt
        return (ps.flat, ps.grad, opt.exp_avg, opt.exp_avg_sq, *ps.shadows.ptrs(), ps.shadows.fp16, start, state_start, count, group, n,
                opt._groups_dev)

    def step(self, advance):
        """The sharded step on the current stream: clip record (global norm: one all-reduce of this rank's float64 sum of
        squares), one launch over this rank's slices, then finish() every bucket. advance: the launch advances the counter (RAdam
        without max_grad_norm)."""
        opt, lib, ps = self.opt, L.lib(), self.opt.engine.ps
        rec = None
        if opt.max_grad_norm is not None:
            L.call(lib.vb_grad_norm_partial, ps.grad, self.start, self.count, self.n_chunks, self.partials, self.norm_sum)
            torch.distributed.all_reduce(self.norm_sum, group=self.red.group)
            L.call(lib.vb_clip_finish, self.norm_sum, C.c_float(opt.grad_scale), C.c_float(opt.max_grad_norm), opt._clip_record,
                   opt._step_dev)
            rec = opt._clip_record
        fn = opt._sharded_fn()
        L.call(fn, *opt._sharded_args(self._head(self.start, self.state_start, self.count, self.group, self.n_chunks), advance, rec, 0))
        if opt.fused_zero_grad:
            for k in range(len(self.table)):
                self.zero_others(k)
        works = [self.gather(k) for k in range(len(self.table))]
        for k, w in enumerate(works):
            if w is not None:
                w.wait()
            self.recast(k)
        self.red.reset_exchange()

    def _others(self, k):
        """The parts of bucket k outside this rank's slice."""
        (lo, hi), (a, e, _) = self.table[k], self.layout[k]
        return [(x, y) for x, y in ((lo, a), (e, hi)) if y > x]

    def zero_others(self, k):
        ps = self.opt.engine.ps
        for x, y in self._others(k):
            L.call(L.lib().vb_memset_zero, ps.grad[x:y], (y - x) * 4)

    def gather(self, k):
        lo, hi = self.table[k]
        return self.red.all_gather_range(self.opt.engine.ps.flat, lo, hi)

    def recast(self, k):
        ps = self.opt.engine.ps
        for x, y in self._others(k):
            L.call(L.lib().vb_cast_f32_to_bf16, *ps.cast_args(x, y - x))

    def bucket_launches(self):
        """Per bucket: (entry point, C arguments of its first launch of a step, of any later one), capped as step_in_backward's."""
        opt = self.opt
        key = (opt.grad_scale, opt.fused_zero_grad, getattr(opt, "leader_group", 0), STEP_MAX_CTAS)
        hit = self._launches.get(key)
        if hit is None:
            fn, hit, at = opt._sharded_fn(), [], 0
            for st, _, _, _ in self.per_bucket:
                n = len(st)
                head = self._head(self.start[at:], self.state_start[at:], self.count[at:], self.group[at:], n)
                hit.append((fn, L.launch_args(fn, *opt._sharded_args(head, True, None, STEP_MAX_CTAS)),
                            L.launch_args(fn, *opt._sharded_args(head, False, None, STEP_MAX_CTAS))))
                at += n
            self._launches[key] = hit
        return hit


class _FlatBufferOptimizer(torch.optim.Optimizer):
    """What the fused optimizers share: the parameters must be views of the engine's flat fp32 buffer; the moments are two
    flat buffers of the same layout (per-parameter state entries are views of them); the work list is a chunk table over
    the trainable tensors; the hyper-parameters live in a device table (one vb_adamw_group row per param group) that is
    re-uploaded from pinned memory when a scheduler changed it; the step counter is a device int32.

    Parameters frozen (requires_grad=False) when the optimizer is built stay out of it. One frozen later is skipped from the next
    step() on, as torch skips a parameter whose .grad is None: step() rebuilds the chunk table in place when the trainable set
    changed. (A step already placed in a plan with Plan.enable_optimizer keeps its chunk count: enable it again after freezing.)

    shard_state=True (model= a ddp.DistributedDataParallel over more than one rank): the moments are this rank's slices
    (ddp.shard_slices of the reducer's bucket table) only; see _ShardedState."""

    def __init__(self, params, defaults, model, engine, zero_grad, chunk, max_grad_norm, shard_state=False):
        name = type(self).__name__
        from .ddp import DistributedDataParallel
        if shard_state:
            if not isinstance(model, DistributedDataParallel):
                raise ValueError(f"{name}(shard_state=True) shards the state over data-parallel ranks: pass "
                                 "model=vilbert_b200.ddp.DistributedDataParallel(...)")
            if model.reducer.world < 2:
                raise ValueError(f"{name}(shard_state=True) needs a data-parallel world of more than one rank")
        if engine is None:
            if model is None:
                raise ValueError(f"{name} needs model= (a vilbert_b200 model) or engine=")
            engine = model.engine
        if defaults["lr"] < 0.0:
            raise ValueError("Invalid learning rate: {} - should be >= 0.0".format(defaults["lr"]))
        betas = defaults["betas"]
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid beta parameters: {} - should be in [0.0, 1.0[".format(betas))
        if not 0.0 <= defaults["eps"]:
            raise ValueError("Invalid epsilon value: {} - should be >= 0.0".format(defaults["eps"]))
        if max_grad_norm is not None:
            max_grad_norm = float(max_grad_norm)
            if not max_grad_norm > 0.0:      # also false for NaN
                raise ValueError(f"Invalid max_grad_norm: {max_grad_norm} - should be > 0.0 (float('inf'): skip non-finite steps "
                                 "without clipping)")
        super().__init__(params, defaults)
        self.engine = engine
        self.shard_state = bool(shard_state)
        self._model = model.module if isinstance(model, DistributedDataParallel) else model
        self._bucket_tables = {}      # (bucket table, trainable key) -> per-bucket launch arguments (_bucket_launches)
        self._single_tables = {}      # frozen set -> the single-process bucket table
        self._side = None             # the stream of the step in the backward
        self._stepped = False         # inside step_in_backward: the step ran in a backward
        self.fused_zero_grad = bool(zero_grad)
        ps = engine.ps
        dev = ps.flat.device
        self.exp_avg = torch.zeros_like(ps.flat) if not shard_state else None
        self.exp_avg_sq = torch.zeros_like(ps.flat) if not shard_state else None
        base, numel = ps.flat.data_ptr(), ps.numel
        self._chunk = chunk
        self._tracked = []       # (param, flat offset, numel, group index) of every parameter trainable at construction
        ranges, seen = [], set()
        for gi, group in enumerate(self.param_groups):
            for p in group["params"]:
                if id(p) in seen:
                    continue     # the tied decoder / word-embedding Parameter is one tensor
                seen.add(id(p))
                if not p.requires_grad:
                    continue
                off = (p.data_ptr() - base) // 4
                if (p.data_ptr() - base) % 4 or off < 0 or off + p.numel() > numel or not p.is_contiguous() or p.dtype != torch.float32:
                    raise ValueError(f"{name}: every parameter must be a contiguous fp32 view of the engine's flat buffer")
                ranges.append((off, p.numel(), gi))
                self._tracked.append((p, off, p.numel(), gi))
                self.state[p] = dict(step=0) if shard_state else \
                    dict(step=0, exp_avg=self.exp_avg[off:off + p.numel()].view(p.shape),
                         exp_avg_sq=self.exp_avg_sq[off:off + p.numel()].view(p.shape))
        st, cn, gr = build_chunks(ranges, chunk)
        self.n_chunks = len(st)
        self._chunk_start = torch.from_numpy(st).to(dev)
        self._chunk_count = torch.from_numpy(cn).to(dev)
        self._chunk_group = torch.from_numpy(gr).to(dev)
        self._trainable_key = (True,) * len(self._tracked)
        self._groups_host = torch.zeros(len(self.param_groups) * _GROUP_DT.itemsize, dtype=torch.uint8).pin_memory() if dev.type == "cuda" else \
            torch.zeros(len(self.param_groups) * _GROUP_DT.itemsize, dtype=torch.uint8)
        self._groups_np = self._groups_host.numpy().view(_GROUP_DT)
        self._groups_dev = torch.zeros_like(self._groups_host, device=dev)
        self._groups_last = None
        self._step_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        self.step_count = 0
        self.grad_scale = 1.0
        self.max_grad_norm = max_grad_norm
        self.grad_norm = self.skipped_steps = None
        if max_grad_norm is not None:
            # vb_clip_record {norm f32, coef f32, skip i32, skipped i32}; the partials table keeps its size when frozen parameters
            # shrink the chunk table
            self._clip_record = torch.zeros(4, dtype=torch.int32, device=dev)
            self._norm_partials = torch.zeros(max(self.n_chunks, 1), dtype=torch.float64, device=dev)
            self.grad_norm = self._clip_record.view(torch.float32)[0]
            self.skipped_steps = self._clip_record[3]
        self._upload_groups()
        self._shard = None
        if shard_state:
            self._model._frozen()            # the reducer's table follows the requires_grad flags of now
            self._shard = _ShardedState(self, model.reducer)
        if dev.type == "cuda":
            engine.refresh_weights()         # frozen tensors (not in any group) keep this copy; updated ones are rewritten every step
            engine.shadow_trusted = True

    def _refresh_trainable(self):
        """Drops parameters frozen since construction from the chunk table (rewritten in place, so the device pointers stay valid);
        returns whether the table changed."""
        key = tuple(p.requires_grad for p, _, _, _ in self._tracked)
        if key == self._trainable_key:
            return False
        self._trainable_key = key
        st, cn, gr = build_chunks([(off, n, gi) for (p, off, n, gi), rg in zip(self._tracked, key) if rg], self._chunk)
        self.n_chunks = len(st)
        if self.n_chunks:
            self._chunk_start[:self.n_chunks].copy_(torch.from_numpy(st))
            self._chunk_count[:self.n_chunks].copy_(torch.from_numpy(cn))
            self._chunk_group[:self.n_chunks].copy_(torch.from_numpy(gr))
        return True

    # ------------------------------------------------------------------ hyper-parameter table
    def _group_row(self, grp):
        """The vb_adamw_group row of one param group."""
        return group_row(grp["lr"], grp["betas"], grp["eps"], grp["weight_decay"])

    def _upload_groups(self):
        g = self._groups_np
        for i, grp in enumerate(self.param_groups):
            g[i] = self._group_row(grp)
        key = g.tobytes()
        if key != self._groups_last:
            self._groups_dev.copy_(self._groups_host, non_blocking=True)
            self._groups_last = key

    def _buffer_args(self):
        """The leading arguments of vb_adamw_step / vb_radam_step: buffers, 16-bit copies, chunk table and group table."""
        ps = self.engine.ps
        return (ps.flat, ps.grad, self.exp_avg, self.exp_avg_sq, *ps.shadows.ptrs(), ps.shadows.fp16, self._chunk_start,
                self._chunk_count, self._chunk_group, self.n_chunks, self._groups_dev)

    @staticmethod
    def _op(fn, *args):
        """(fn, C arguments) of one launch for an engine op list."""
        return fn, L.launch_args(fn, *args)

    def _norm_op(self, step):
        """(fn, args) of vb_grad_norm over the chunk table; it advances the counter `step` (None: none) unless it skips."""
        return self._op(L.lib().vb_grad_norm, self.engine.ps.grad, self._chunk_start, self._chunk_count, self.n_chunks,
                        C.c_float(self.grad_scale), C.c_float(self.max_grad_norm), self._norm_partials, self._clip_record, step)

    def op(self):
        """(fn, args) of the step launch for an engine op list when max_grad_norm is None (the step is then one operation)."""
        ops = self.ops()
        if len(ops) != 1:
            raise ValueError(f"{type(self).__name__} with max_grad_norm is two operations (gradient norm, step): use ops()")
        return ops[0]

    @staticmethod
    def _run(ops, stream):
        for fn, args in ops:
            L.call(fn, *args, stream=stream)

    def _trainable_ranges(self):
        """(flat offset, numel, group index) of the tracked parameters that are trainable now: the chunk table's ranges."""
        return [(off, n, gi) for (p, off, n, gi), rg in zip(self._tracked, self._trainable_key) if rg]

    # ------------------------------------------------------------------ the step in the backward
    @contextlib.contextmanager
    def step_in_backward(self):
        """`with optimizer.step_in_backward(): loss.backward()` gives the state `loss.backward(); optimizer.step()` gives (weights,
        moments, 16-bit copies, zeroed gradients, the device step counter, step_count and state[p]["step"]), with the step running
        while the backward does: each bucket of the flat buffers is updated on a side stream once no later backward op reads or
        writes its weights, 16-bit copies or gradient (engine Plan.step_schedule), on grid-capped launches of the same kernels. The
        backward returns after the current stream waited for that stream, so the next forward reads the updated weights. Do not
        call step() for this iteration; schedulers step as before.

        Entering does what step() does on the host first (the trainable set, the hyper-parameter table), so an lr a scheduler set
        since the last step applies. Each bucket gets the per-element update step() would give it, so under
        torch.use_deterministic_algorithms(True) the two paths agree bit for bit.

        Which backward steps: the step runs inside the backward of a plan-backed call of the model when that call is the only
        pending plan backward of the model, i.e. no other plan-backed forward of the model whose outputs need a gradient is still
        waiting for its backward (its gradient would not be final when this one's buckets are stepped). Otherwise the step runs
        after the backward, unoverlapped, with the same result: when the backward reaches more than one plan-backed forward of
        the model, when it reaches no plan, for a plan with anomaly checks (and not at all when that backward raised: a body that
        raises steps nothing), and under data parallelism with delay_allreduce=True, where it follows the all-reduce. With
        delay_allreduce=False a bucket is stepped after its collective.

        Gradient accumulation: the micro-batches before the last use plain loss.backward() (under model.no_sync() with data
        parallelism); the last one uses this context. Refused with ValueError: max_grad_norm (clipping needs the global norm before
        any element is updated) and model.no_sync() (a step inside an accumulation micro-batch)."""
        name = type(self).__name__
        model = self._model
        if model is None:
            raise ValueError(f"{name}.step_in_backward needs the optimizer built with model=")
        if self.max_grad_norm is not None:
            raise ValueError(f"{name}.step_in_backward: max_grad_norm clips with the global gradient norm, which is known only after "
                             "the whole backward; use loss.backward(); optimizer.step()")
        if not model._ddp_sync:
            raise ValueError(f"{name}.step_in_backward inside model.no_sync(): an accumulation micro-batch does not step; use plain "
                             "loss.backward() for it and the context for the last micro-batch")
        if model._step_in_backward is not None:
            raise ValueError(f"{name}.step_in_backward: the model is already inside a step_in_backward context")
        self._refresh()
        self._upload_groups()
        self._stepped = False
        model._step_in_backward = self._backward_with_step
        raised = True
        try:
            yield
            raised = False
        finally:
            model._step_in_backward = None
            if self._stepped:
                self._count_step()
                self._after_step()
            elif not raised:
                self.step()

    def _refresh(self):
        """The host work of step() before its launch that depends on the trainable set."""
        self._refresh_trainable()
        if self._shard is not None:
            self._shard.sync()

    def _count_step(self):
        self.step_count += 1
        for st in self.state.values():
            st["step"] = self.step_count

    def _single_table(self):
        """The buckets of a single process: ddp.trainable_ranges cut as ddp.FlatGradAllReducer cuts them (STEP_BUCKETS)."""
        frozen = self._model._frozen()
        table = self._single_tables.get(frozen)
        if table is None:
            from .ddp import FlatGradAllReducer
            red = FlatGradAllReducer(self.engine.ps.grad, n_buckets=STEP_BUCKETS)
            red.set_ranges(self._model._trainable_ranges())
            table = self._single_tables[frozen] = red.table
        return table

    def _bucket_launches(self, table):
        """Per bucket of `table`: (entry point, C arguments of its first launch of a step, C arguments of any later one) over its
        chunk sub-table (bucket_chunks), which lives on the device with the cache entry."""
        if self._shard is not None:
            if table != self._shard.table:
                raise RuntimeError(f"{type(self).__name__}: the sharded state follows another bucket table than the backward's")
            return self._shard.bucket_launches()
        key = (table, self._trainable_key, self.grad_scale, self.fused_zero_grad, getattr(self, "leader_group", 0), STEP_MAX_CTAS)
        hit = self._bucket_tables.get(key)
        if hit is not None:
            return hit[0]
        ps, dev = self.engine.ps, self.exp_avg.device
        subs = bucket_chunks(self._trainable_ranges(), table, self._chunk)
        st, cn, gr = (torch.from_numpy(np.concatenate([s[i] for s in subs])).to(dev) for i in range(3))
        out, at = [], 0
        for s in subs:
            n = len(s[0])
            head = (ps.flat, ps.grad, self.exp_avg, self.exp_avg_sq, *ps.shadows.ptrs(), ps.shadows.fp16, st[at:], cn[at:], gr[at:], n,
                    self._groups_dev)
            fn = self._capped_fn()
            out.append((fn, L.launch_args(fn, *self._capped_args(head, True)), L.launch_args(fn, *self._capped_args(head, False))))
            at += n
        self._bucket_tables[key] = (out, st, cn, gr)
        return out

    def _side_stream(self):
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.exp_avg.device)
        return self._side

    def _backward_with_step(self, plan, red):
        """The backward of `plan` with this step in it (the model's hook while step_in_backward is active): the pieces of
        plan.step_schedule over the reducer's table (red: a data-parallel reducer all-reducing during the backward) or the
        single-process table. After each piece the side stream waits for it and, under data parallelism, for the collectives of
        the buckets it steps; it advances the device step counter once, before the first launch. The current stream waits for
        the side stream (and the collectives) before this returns."""
        if self._stepped:
            raise RuntimeError(f"{type(self).__name__}.step_in_backward: a second backward reached a plan after the step ran; run one "
                               "backward per context")
        if self._shard is not None:
            # the forward inside the context may have frozen parameters (a new bucket table): the moments follow it first, on every
            # rank at the same point (collective only when the table changed)
            self._refresh()
        table = red.table if red is not None else self._single_table()
        launches = self._bucket_launches(table)
        side = self._side_stream()
        if plan.e.auto_graph:
            plan.maybe_capture_pieces(table, step=True, allreduce=red is not None)
        works, gathers, first = {}, [], [True]
        shard = self._shard

        def handover(ranges):
            works.update((r, red.allreduce_range(*r)) for r in ranges)

        def step(ks):
            if red is not None:          # collectives enqueued on the communication stream itself, then the asynchronous ones
                side.wait_stream(comm)
            for k in ks:
                w = works.get(table[k])
                if w is not None:
                    w.wait()
                self._launch_bucket(launches[k], first[0], side)
                first[0] = False
                if shard is not None:    # sharded: the rest of the bucket's gradient zeroed, its weights gathered after the step
                    if self.fused_zero_grad:
                        shard.zero_others(k)
                    with torch.cuda.stream(comm):
                        comm.wait_stream(side)
                        gathers.append(shard.gather(k))
        comm = red.comm_stream() if red is not None else None
        plan.run_backward_pieces(table, handover if red is not None else None, comm, step, side)
        if first[0]:          # no bucket: the counter still moves, as in step()
            with torch.cuda.stream(side):
                self._step_dev.add_(1)
        main = torch.cuda.current_stream()
        if red is not None:
            main.wait_stream(comm)
            for w in list(works.values()) + gathers:
                if w is not None:
                    w.wait()
        main.wait_stream(side)
        if shard is not None:
            for k in range(len(table)):
                shard.recast(k)
            red.reset_exchange()
        self._stepped = True

    def _launch_bucket(self, launch, first, stream):
        fn, args_first, args = launch
        L.check(fn(*(args_first if first else args), stream.cuda_stream), fn.__name__)

    def _after_step(self):
        eng = self.engine
        eng.shadow_clean = True
        if self.fused_zero_grad:
            eng.grad_clean = True

    def zero_grad(self, set_to_none=False):
        """The gradients live in the engine's flat buffer and were zeroed by step(); the views stay attached."""
        self.engine.zero_grad()
        if self._shard is not None:
            self._shard.red.reset_exchange()

    def _expose(self, full):
        """Sharded: state[p] as the unsharded optimizer holds it, views of the flat-layout moments `full`."""
        for p, off, n, _ in self._tracked:
            self.state[p] = dict(step=self.state[p]["step"], exp_avg=full[0][off:off + n].view(p.shape),
                                 exp_avg_sq=full[1][off:off + n].view(p.shape))

    def _hide(self):
        for p, _, _, _ in self._tracked:
            self.state[p] = dict(step=self.state[p]["step"])

    def load_state_dict(self, state_dict):
        """Copies exp_avg / exp_avg_sq INTO the flat state buffers (the default implementation would replace the views). Sharded: the
        state dict is the unsharded layout (every parameter's full moments); each rank keeps its slices. Collective."""
        if self._shard is not None:
            self._shard.sync()
            full = self._shard.full_moments()
            self._expose(full)
        groups = state_dict["param_groups"]
        params = [p for g in self.param_groups for p in g["params"]]
        ids = [i for g in groups for i in g["params"]]
        for pid, p in zip(ids, params):
            s = state_dict["state"].get(pid)
            if s is None or p not in self.state:
                continue
            self.state[p]["exp_avg"].copy_(s["exp_avg"])
            self.state[p]["exp_avg_sq"].copy_(s["exp_avg_sq"])
            self.state[p]["step"] = int(s["step"])
            self.step_count = max(self.step_count, int(s["step"]))
        self._step_dev.fill_(self.step_count)
        for g_new, g_old in zip(groups, self.param_groups):
            for k, v in g_new.items():
                if k != "params":
                    g_old[k] = v
        self._upload_groups()
        if self._shard is not None:
            self._hide()
            self._shard._set_layout(full)
            self._shard.sync()

    def state_dict(self):
        """The per-parameter "step" is the device counter's value: replays of a captured step advance it without the host
        knowing, and with max_grad_norm only the device knows which steps were skipped."""
        self.step_count = int(self._step_dev.item())
        for st in self.state.values():
            st["step"] = self.step_count
        if self._shard is None:
            return super().state_dict()
        self._shard.sync()        # sharded: every rank gathers the full moments (collective)
        self._expose(self._shard.full_moments())
        try:
            return super().state_dict()
        finally:
            self._hide()


class FusedAdamW(_FlatBufferOptimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True, model=None, engine=None,
                 zero_grad=True, chunk=32768, max_grad_norm=None, shard_state=False):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, correct_bias=correct_bias),
                         model, engine, zero_grad, chunk, max_grad_norm, shard_state)

    def _group_row(self, grp):
        return group_row(grp["lr"], grp["betas"], grp["eps"], grp["weight_decay"], grp["correct_bias"])

    # ------------------------------------------------------------------ stepping
    def launch(self, stream=None):
        """The kernel launches alone (capturable in a CUDA graph): use the hyper-parameter table and step counter currently on the
        device. `step()` = advance the counter + refresh the table + launch. With max_grad_norm the gradient norm comes first and
        advances the device counter itself, unless the step is skipped."""
        self._run(self.ops(), stream)

    def ops(self):
        """[(fn, args)] of one step for an engine op list (Plan.epilogue): the step launch, preceded by the gradient norm when
        max_grad_norm is set."""
        args = self._buffer_args() + (self._step_dev, C.c_float(self.grad_scale), 1 if self.fused_zero_grad else 0)
        if self.max_grad_norm is None:
            return [self._op(L.lib().vb_adamw_step, *args)]
        return [self._norm_op(self._step_dev), self._op(L.lib().vb_adamw_step_clipped, *args, self._clip_record)]

    def _capped_fn(self):
        return L.lib().vb_adamw_step_capped

    def _sharded_fn(self):
        return L.lib().vb_adamw_step_sharded

    def _sharded_args(self, head, advance, rec, max_ctas):
        """The counter is advanced by the caller (step(), _launch_bucket) or by vb_clip_finish, as for the unsharded launch."""
        return head + (self._step_dev, C.c_float(self.grad_scale), 1 if self.fused_zero_grad else 0, rec, max_ctas)

    def _capped_args(self, head, first):
        return head + (self._step_dev, C.c_float(self.grad_scale), 1 if self.fused_zero_grad else 0, STEP_MAX_CTAS)

    def _launch_bucket(self, launch, first, stream):
        if first:            # the counter moves once per step, before the first launch reads it (correct_bias)
            with torch.cuda.stream(stream):
                self._step_dev.add_(1)
        super()._launch_bucket(launch, first, stream)

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        self._refresh_trainable()
        if self.max_grad_norm is None:
            self.step_count += 1
            self._step_dev.add_(1)
            for st in self.state.values():
                st["step"] = self.step_count
        self._upload_groups()
        if self._shard is not None:
            self._shard.sync()
            self._shard.step(False)
        elif self.n_chunks or self.max_grad_norm is not None:
            self.launch()
        self._after_step()
        return loss


class FusedRAdam(_FlatBufferOptimizer):
    """The reference's RAdam (vilbert/optimization.py:16-100; `--optim RAdam`, train_tasks.py:427-428) as one launch of
    `radam_kernel` per step. Same defaults (lr 1e-3, betas (0.9, 0.999), eps 1e-8, weight_decay 0) and checkpoint layout
    (per parameter index: {step, exp_avg, exp_avg_sq}), so state dicts move between the two.

    Reference behaviour kept on purpose: the rectification term and step size of a step are computed once, from the lr and
    betas of the first param group holding a trainable tensor (the "leader group"), and used for every tensor; each group's
    own lr only enters its weight decay (and its betas its moments). With the reference's grouping that group is the word
    embeddings' at base_lr, so the vil_* heads' lr of 1e-4 does not reach their RAdam update."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, model=None, engine=None, zero_grad=True,
                 chunk=32768, max_grad_norm=None, shard_state=False):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay), model, engine, zero_grad, chunk,
                         max_grad_norm, shard_state)
        self._set_leader()

    def _set_leader(self):
        """The leader is the first param group holding a trainable tensor."""
        trainable = {id(p) for (p, _, _, _), rg in zip(self._tracked, self._trainable_key) if rg}
        self.leader_group = next((gi for gi, g in enumerate(self.param_groups) if any(id(p) in trainable for p in g["params"])), 0)

    def _refresh(self):
        if self._refresh_trainable():
            self._set_leader()
        if self._shard is not None:
            self._shard.sync()

    def _capped_fn(self):
        return L.lib().vb_radam_step_capped

    def _sharded_fn(self):
        return L.lib().vb_radam_step_sharded

    def _sharded_args(self, head, advance, rec, max_ctas):
        return head + (self.leader_group, self._step_dev, 1 if advance else 0, C.c_float(self.grad_scale), 1 if self.fused_zero_grad else 0,
                       rec, max_ctas)

    def _capped_args(self, head, first):
        """advance_step on the first launch of a step only; the leader-group rule is step()'s."""
        return head + (self.leader_group, self._step_dev, 1 if first else 0, C.c_float(self.grad_scale), 1 if self.fused_zero_grad else 0,
                       STEP_MAX_CTAS)

    def _args(self, advance_step):
        return self._buffer_args() + (self.leader_group, self._step_dev, advance_step, C.c_float(self.grad_scale),
                                      1 if self.fused_zero_grad else 0)

    # ------------------------------------------------------------------ stepping
    def launch(self, stream=None, advance_step=False):
        """The kernel launches alone (capturable in a CUDA graph): use the hyper-parameter table currently on the device, and the
        device step counter, first advanced by one on the same stream when `advance_step` (with max_grad_norm: by the gradient
        norm, unless the step is skipped). `step()` = refresh the table + launch(advance_step=True)."""
        self._run(self.ops(advance_step), stream)

    def ops(self, advance_step=True):
        """[(fn, args)] of one step for an engine op list (Plan.epilogue): the step launch, preceded by the gradient norm when
        max_grad_norm is set. Advancing the step counter is part of the step, so every replay of a captured step moves one step
        along the rectification schedule."""
        if self.max_grad_norm is None:
            return [self._op(L.lib().vb_radam_step, *self._args(1 if advance_step else 0))]
        return [self._norm_op(self._step_dev if advance_step else None),
                self._op(L.lib().vb_radam_step_clipped, *self._args(0), self._clip_record)]

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        if self._refresh_trainable():
            self._set_leader()
        if self.max_grad_norm is None:
            self.step_count += 1
            for st in self.state.values():
                st["step"] = self.step_count
        self._upload_groups()
        if self._shard is not None:
            self._shard.sync()
            self._shard.step(self.max_grad_norm is None)
        elif self.n_chunks or self.max_grad_norm is not None:
            self.launch(advance_step=True)
        else:
            self._step_dev.add_(1)
        self._after_step()
        return loss
