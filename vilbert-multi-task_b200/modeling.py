"""Drop-in module surface: BertModel, VILBertForVLTasks, BertForMultiModalPreTraining with the
reference's constructor / forward signatures, output tuples and state_dict key names
(vilbert/vilbert.py:1288-1406, :1435-1597, :1600-1708; SURVEY.md §8b), executing on the H100 engine
(engine.py -> libvilbert_b200.so). There is no PyTorch / CPU fallback: constructing a model on a
non-CUDA device or without the built extension raises.
"""
import contextlib
import operator
import os
import traceback
import warnings
import weakref

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from . import _lib as L
from .config import BertConfig
from .engine import (BERT_OUT_NAMES, HEAD_NAMES, INPUT_GRAD_NAMES, LOSS_HEADS, PRETRAINING_HEAD_NAMES, Engine, check_pack_config, pack_summary,
                     pretraining_pack_rows, pretraining_pack_rows_from_summary)


# Any torch.optim.Optimizer.step() (pytorch_transformers.AdamW and the reference's RAdam subclass it) may have rewritten
# parameters through p.data: bump a global epoch that every model compares with the epoch its 16-bit weight copy was made at.
_OPT_EPOCH = [0]
_REQUIRES_GRAD = operator.attrgetter("requires_grad")


def _on_optimizer_step(optimizer, args, kwargs):
    _OPT_EPOCH[0] += 1


try:
    torch.optim.optimizer.register_optimizer_step_post_hook(_on_optimizer_step)
except AttributeError:      # very old torch: train-mode forwards refresh unconditionally anyway
    pass


class _Node(nn.Module):
    """Container whose children / parameters are registered under the reference's dotted names."""


class _BertNode(_Node):
    """The `bert` sub-module of a model with heads: owns the encoder parameters (names bert.*) and, when called like
    the reference's `model.bert(...)` (vilbert.py:1652), runs the same engine and returns the BertModel 5-tuple."""

    def forward(self, input_txt, input_imgs, image_loc, token_type_ids=None, attention_mask=None, image_attention_mask=None,
                co_attention_mask=None, task_ids=None, output_all_encoded_layers=False, output_all_attention_masks=False):
        owner = self.__dict__["_owner_ref"]()
        return owner._bert_forward(input_txt, input_imgs, image_loc, token_type_ids, attention_mask, image_attention_mask, task_ids,
                                   output_all_encoded_layers, output_all_attention_masks)


def _register_tree(root, store):
    params = {}
    for name in store.entries:
        view = store.p(name)
        prm = nn.Parameter(view, requires_grad=True)
        prm.grad = store.g(name)
        params[name] = prm
        _attach(root, name, prm)
    # tied decoder: the same Parameter object under its reference name (vilbert.py:1190, 1634-1636)
    _attach(root, "cls.predictions.decoder.weight", params["bert.embeddings.word_embeddings.weight"])
    return params


def _attach(root, dotted, prm):
    import weakref
    parts = dotted.split(".")
    mod = root
    for i, p in enumerate(parts[:-1]):
        if p not in mod._modules:
            if i == 0 and p == "bert":
                node = _BertNode()
                node.__dict__["_owner_ref"] = weakref.ref(root)
            else:
                node = _Node()
            mod.add_module(p, node)
        mod = mod._modules[p]
    mod.register_parameter(parts[-1], prm)


class _PlanCall:
    """One call of the module surface on an engine plan: the model, the plan, its inputs and loss-input targets, and the dropout
    step and forward id its forward() ran at. With `names` the call returns those plan outputs and takes their gradients into
    plan.gout; without, it returns the plan's objective (the task loss as a 0-d tensor, or the three [1] pre-training losses) and
    takes d(total)/d(loss) into plan.loss_grad, 0 for a loss that receives none.

    backward() always runs at its own forward. If the plan no longer holds that forward (the plan ran again, another plan
    overwrote the shared arena, or the backward switched to the plan of another gradient set), the forward is recomputed from the
    same inputs and targets. In train mode, if another forward moved the dropout step since, the step of this forward is set
    around the recomputed forward and the backward, which regenerate their dropout masks from it, and restored afterwards. The
    backward accumulates into the flat gradient buffer (the Parameters' .grad are views of it) and, when a data-parallel reducer
    is attached and the model is not under no_sync(), averages it over the ranks: after the backward (delay_allreduce=True, a
    world of one, a plan with anomaly checks), or bucket by bucket while the backward runs in pieces (delay_allreduce=False,
    ddp.FlatGradAllReducer.overlapped_backward).

    input_names: the float inputs (INPUT_GRAD_NAMES) whose gradient the plan computes (Plan.input_grads). backward() copies them
    out of the plan right after its backward ran, in the shape, dtype and device of the tensors the caller passed
    (self.input_grads_out; None for an input behind a no_grad layer). They are per-rank: the all-reduce never sees them.

    Anomaly mode (torch.autograd.set_detect_anomaly(True), or the detect_anomaly() context, with check_nan): the plans are built with
    NaN checks (Plan(anomaly=True)) and forward() keeps the Python stack of the call. backward() reads the plan's report right after
    its backward ran; when a gradient held a NaN it warns with that stack and raises RuntimeError naming the first op, as torch
    names the backward node — before the input gradients are copied out and before the all-reduce, so the caller's optimizer step is
    never reached. The flat gradient buffer keeps what the backward wrote.

    Inside a fused optimizer's step_in_backward() context (model._step_in_backward), the backward of the model's only pending plan
    call (model._pending_calls: calls whose forward made outputs that need a gradient and whose backward has not run) runs in the
    pieces of Plan.step_schedule with the step in it; every other backward runs as above and the context steps after it."""

    def __init__(self, model, plan, inputs, targets=None, names=None):
        self.model, self.plan, self.inputs, self.targets, self.names = model, plan, inputs, targets or {}, names
        self.input_names = tuple(n for n in INPUT_GRAD_NAMES if n in plan.input_grads)
        self.input_grads_out = (None,) * len(self.input_names)
        self.drop_step = self.fwd_id = None
        self.stack = None

    def _load(self):
        plan = self.plan
        with torch.no_grad():      # the plan's input buffers never join the caller's graph, also when backward() reloads them
            plan.load_inputs(**self.inputs)
            li = plan.loss_inputs
            for k, v in self.targets.items():
                li[k].copy_(v.reshape(li[k].shape), non_blocking=True)

    def forward(self):
        model, plan, eng = self.model, self.plan, self.model.engine
        model._sync_weights()
        if plan.train:
            eng.bump_dropout_step()      # fresh nn.Dropout masks for this forward
        self.drop_step = eng.drop_step_host
        if torch.is_anomaly_enabled() and torch.is_anomaly_check_nan_enabled():
            self.stack = traceback.format_stack()[:-1]
        self._load()
        if eng.auto_graph:
            plan.maybe_capture_passes()
        plan.run_forward()
        self.fwd_id = plan.fwd_id
        model._last_plan = plan

    def differentiable(self):
        """Per output of outputs(): whether a trainable parameter lies upstream of it (Plan.out_rg)."""
        rg = self.plan.out_rg
        if self.names is not None:
            return tuple(rg.get(n, True) for n in self.names)
        if self.plan.loss_kind == "pretraining":
            return tuple(rg.get(n, True) for n in PRETRAINING_HEAD_NAMES)
        return (rg.get(LOSS_HEADS[self.plan.loss_kind][0], True),)

    def outputs(self):
        plan = self.plan
        if self.names is not None:
            return tuple(plan.outputs[n].clone() for n in self.names)
        if plan.loss_kind == "pretraining":
            out = plan.objective_out.detach()
            return out[0:1].clone(), out[1:2].clone(), out[2:3].clone()
        return (plan.loss.detach().reshape(()).clone(),)

    def backward(self, grads, wanted=()):
        """wanted: per entry of input_names, whether its gradient is copied out (autograd's needs_input_grad)."""
        model, eng = self.model, self.model.engine
        if self.names is not None:
            live = tuple(n for n, g in zip(self.names, grads) if g is not None)
            if frozenset(live) != self.plan.grad_outputs:     # the plan's backward reaches other outputs: take the plan of this set
                self.plan = model._outputs_plan(self.names, self.inputs, self.plan.train, live, self.plan.frozen, self.plan.input_grads)
                self.fwd_id = None
        plan = self.plan
        red = model._ddp_reducer if model._ddp_sync else None
        overlap = red is not None and model._ddp_overlap and red.world > 1 and not plan.anomaly
        step = self._step_hook(red, overlap)
        step_here = step is not None
        now = eng.drop_step_host
        moved = plan.train and now != self.drop_step
        if moved:
            eng.set_dropout_step(self.drop_step)
        try:
            if not plan.holds_forward(self.fwd_id):
                self._load()
                plan.run_forward()
                self.fwd_id = plan.fwd_id
            model._attach_grads()
            if eng.auto_graph:
                plan.maybe_capture_passes()
                if overlap and not step_here:
                    plan.maybe_capture_pieces(red.table)
            if self.names is not None:
                for n, g in zip(self.names, grads):
                    if g is not None:
                        plan.gout[n].copy_(g.reshape(plan.gout[n].shape))
            else:
                for i, g in enumerate(grads):
                    if g is None:
                        plan.loss_grad[i:i + 1].zero_()
                    else:
                        plan.loss_grad[i:i + 1].copy_(g.detach().reshape(1))
            if step_here:
                step(plan, red if overlap else None)
            elif overlap:
                red.overlapped_backward(plan)
            else:
                plan.run_backward()
            if plan.anomaly and torch.is_anomaly_enabled() and torch.is_anomaly_check_nan_enabled():
                self._raise_on_nan(plan.anomaly_report())
            self.input_grads_out = tuple(self._input_grad(n) if w else None for n, w in zip(self.input_names, wanted))
        finally:
            if moved:
                eng.set_dropout_step(now)
        if red is not None and not overlap:     # data parallel: average the flat gradient buffer over the ranks (apex DDP, delay_allreduce=True)
            red.allreduce()

    def _step_hook(self, red, overlap):
        """The model's step_in_backward hook when this backward runs with the optimizer step in it, else None. It does when the
        context is active, this call is the model's only pending plan backward, its plan has no anomaly checks and its gradient is
        not all-reduced after the backward (delay_allreduce=True). The call stops being pending here."""
        model = self.model
        pending = model._pending_calls
        alone = len(pending) == 1 and self in pending
        pending.discard(self)
        hook = model._step_in_backward
        if hook is not None and alone and not self.plan.anomaly and (red is None or overlap):
            return hook
        return None

    def _raise_on_nan(self, r):
        """torch's anomaly-mode report for the NanRecord `r` (None: nothing to report)."""
        if r is None:
            return
        fn = f"{r.module}: {r.entry}"
        stack = "".join(self.stack) if self.stack else "(the forward ran with anomaly detection off)\n"
        warnings.warn(f"Error detected in {fn}. Traceback of forward call that caused the error:\n{stack}", UserWarning, stacklevel=2)
        raise RuntimeError(f"Function '{fn}' returned nan values in its {r.output}th output.")

    def _input_grad(self, name):
        """A copy of the gradient of the input `name` the backward just wrote, in the shape, dtype and device of the caller's tensor
        (autograd sums it down to an input that broadcast into the plan's buffer); None when the plan wrote none."""
        g = self.plan.input_grad.get(name)
        if g is None:
            return None
        x = self.inputs[name]
        return g.view(self.plan.Bin, self.plan.Nv, -1).to(device=x.device, dtype=x.dtype, copy=True)


class _PlanFn(torch.autograd.Function):
    """Bridges a _PlanCall into torch.autograd: forward runs the call's forward and returns its outputs, backward hands the
    incoming gradients to the call's backward (nothing runs when none of them is live). An output with no trainable parameter
    or differentiable input upstream (every parameter it depends on has requires_grad=False) does not require grad, as in torch.
    The float inputs of call.input_names follow the call as real autograd inputs and receive the gradients the plan computed;
    the backward is not itself differentiable (double backward raises)."""

    @staticmethod
    def forward(ctx, anchor, call, *float_inputs):
        ctx.call = call
        ctx.set_materialize_grads(False)
        call.forward()
        outs = call.outputs()
        dead = [o for o, live in zip(outs, call.differentiable()) if not live]
        if dead:
            ctx.mark_non_differentiable(*dead)
        if len(dead) < len(outs):
            call.model._pending_calls.add(call)
        return outs

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        call = ctx.call
        if not any(g is not None for g in grads):
            return (None, None) + (None,) * len(call.input_names)
        call.backward(grads, ctx.needs_input_grad[2:])
        return (None, None) + call.input_grads_out


class BertPreTrainedModel(nn.Module):
    """Weight handling of the reference's PreTrainedModel (vilbert/utils.py:703-1032) restricted to local
    files: state_dict with the reference key names, legacy gamma/beta renaming, eval mode after loading."""

    config_class = BertConfig
    _heads = "vl"          # which heads own parameters: "vl" | "pretraining" | "none"

    def __init__(self, config, device=None, precision=None, num_labels=None):
        """precision: "fp16" (default: fp16 forward operands, bf16 gradient operands, fp32 accumulation / residual stream),
        "fp32" (split precision, matches the reference's fp32 outputs to 1e-3) or "bf16"; default from
        $VILBERT_B200_PRECISION. The reference's constructors have no such argument: it selects what `model.half()` /
        default fp32 select there."""
        super().__init__()
        if not isinstance(config, BertConfig):
            raise ValueError("Parameter config should be an instance of class `BertConfig`.")
        self.config = config
        precision = precision or os.environ.get("VILBERT_B200_PRECISION", "fp16")
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
        if dev.type != "cuda" or not torch.cuda.is_available():
            raise L.VBError("vilbert_b200 models run on sm_90a GPUs only; there is no CPU path")
        self.engine = Engine(config, dev, heads=self._heads, precision=precision, num_labels=num_labels)
        self._params = _register_tree(self, self.engine.ps)
        self._pnames, self._plist = tuple(self._params), tuple(self._params.values())
        self._frozen_flags, self._frozen_set = None, frozenset()
        self._grad_hint = {}
        self._anchor = torch.zeros((), device=dev, requires_grad=True)
        self._shadow_version = None
        self._opt_epoch = -1
        self._ddp_reducer = None
        self._ddp_set_ranges = None     # data parallel: restricts the reducer to the trainable ranges (ddp.DistributedDataParallel)
        self._ddp_overlap = False       # ... all-reduces the buckets during the backward (delay_allreduce=False)
        self._ddp_sync = True           # False under no_sync()
        self._step_in_backward = None   # a fused optimizer's step_in_backward(): runs the backward with the step in it
        self._pending_calls = weakref.WeakSet()   # plan calls whose outputs need a gradient and whose backward has not run
        self.init_weights()

    # ---- reference init (vilbert.py:1274-1285): N(0, initializer_range) for Linear/Embedding weights, zero bias, LN 1/0
    def init_weights(self):
        std = self.config.initializer_range
        with torch.no_grad():
            for name, prm in self._params.items():
                if "LayerNorm" in name or ".logit_fc.2." in name:
                    prm.fill_(1.0) if name.endswith("weight") else prm.zero_()
                elif name.endswith(".bias"):
                    prm.zero_()
                else:
                    prm.normal_(mean=0.0, std=std)

    def tie_weights(self):
        pass  # the decoder weight IS the word-embedding Parameter (registered twice)

    def _heads_for(self, names):
        """BertModel-only outputs never need the heads' forward."""
        return "none" if all(n in BERT_OUT_NAMES for n in names) else self._heads

    def _sync_weights(self):
        """Refreshes the 16-bit operand copy of the weights from the fp32 master parameters. Optimizers write parameters
        through `p.data` (pytorch_transformers.AdamW: p.data.addcdiv_, vilbert/optimization.py RAdam: p.data.copy_), which no
        tensor version counter sees, so in train mode the copy is refreshed before EVERY forward (one cast kernel) unless the
        engine's own fused optimizer produced it (engine.shadow_trusted). In eval mode the version counter of the flat buffer,
        load_state_dict() and a global post-hook on every torch.optim.Optimizer.step() mark it stale; after writing parameters
        by hand through .data in eval mode call `model.engine.shadow_clean = False`."""
        eng = self.engine
        v = eng.ps.flat._version
        stale = (not eng.shadow_clean) or v != self._shadow_version
        if not eng.shadow_trusted and (self.training or _OPT_EPOCH[0] != self._opt_epoch):
            stale = True
        if stale:
            eng.refresh_weights()
        self._shadow_version, self._opt_epoch = v, _OPT_EPOCH[0]

    def load_state_dict(self, state_dict, strict=True):
        """strict is honoured (missing / unexpected keys raise like nn.Module). The tied decoder weight is one Parameter
        registered under two names: a checkpoint carrying only one of them is complete."""
        sd = dict(state_dict)
        w, d = "bert.embeddings.word_embeddings.weight", "cls.predictions.decoder.weight"
        if w in sd and d not in sd:
            sd[d] = sd[w]
        elif d in sd and w not in sd:
            sd[w] = sd[d]
        r = super().load_state_dict(sd, strict=strict)
        self.engine.shadow_clean = False
        return r

    def zero_grad(self, set_to_none=False):
        """Zeroes the flat gradient buffer. The trainable Parameters' .grad stay views of it (set_to_none is accepted and ignored:
        the engine accumulates into the flat buffer, dropping the views would only hide the gradients from the optimizer); a
        frozen Parameter's (requires_grad=False) .grad is None."""
        self.engine.zero_grad()
        if getattr(self._ddp_reducer, "scatter", False):      # a sharded optimizer's reduce-scatter is discarded with the gradient
            self._ddp_reducer.reset_exchange()
        self._attach_grads(zero_if_detached=False)

    @contextlib.contextmanager
    def no_sync(self):
        """Gradient-accumulation micro-batches under data parallelism, as torch's DistributedDataParallel.no_sync(): the backwards
        inside the context exchange nothing and accumulate into the flat gradient buffer; the first backward outside it averages
        the accumulated buffer over the ranks. Without a data-parallel wrapper it changes nothing."""
        prev, self._ddp_sync = self._ddp_sync, False
        try:
            yield
        finally:
            self._ddp_sync = prev

    def _frozen(self):
        """ParamStore entry names of the Parameters with requires_grad=False: the set every plan-backed call is specialised on.
        Rebuilt only when a flag changed (one pass over the flags per call). A data-parallel reducer is told the new trainable
        ranges."""
        flags = tuple(map(_REQUIRES_GRAD, self._plist))
        if flags != self._frozen_flags:
            self._frozen_flags = flags
            self._frozen_set = frozenset(n for n, f in zip(self._pnames, flags) if not f)
            if self._ddp_set_ranges is not None:
                self._ddp_set_ranges(self._trainable_ranges())
        return self._frozen_set

    def _trainable_ranges(self):
        from .ddp import trainable_ranges
        return trainable_ranges(self.engine.ps, self._frozen())

    def _attach_grads(self, zero_if_detached=True):
        """torch.optim.Optimizer.zero_grad() defaults to set_to_none=True and detaches every .grad from the flat buffer.
        Before a backward the views of the trainable Parameters are re-attached; if they had been dropped since the last backward
        the flat buffer (which the engine kept accumulating into) is zeroed first, which is what the caller asked for. Frozen
        Parameters get .grad None (their range of the flat buffer is never written)."""
        ps = self.engine.ps
        frozen = self._frozen()
        for name in frozen:
            self._params[name].grad = None
        detached = [name for name, prm in self._params.items() if prm.grad is None and name not in frozen]
        if not detached:
            return
        if zero_if_detached:
            self.engine.zero_grad()
        for name in detached:
            self._params[name].grad = ps.g(name)

    def _apply(self, fn, recurse=True):
        raise L.VBError("vilbert_b200 models own flat CUDA parameter buffers that cannot be moved or re-typed in place "
                        "(construct the model on the target GPU; reduced precision is the `precision=` argument)")

    # The calls the reference's drivers make on a freshly built model (train_tasks.py:486-500: model.to(device), model.cuda(),
    # model.half() under --fp16) are accepted when they ask for what the model already is: fp32 master parameters on its GPU.
    def to(self, *args, **kwargs):
        device, dtype, _, _ = torch._C._nn._parse_to(*args, **kwargs)
        mine = self.engine.device
        if device is not None and (device.type != "cuda" or (device.index is not None and device.index != mine.index)):
            raise L.VBError(f"vilbert_b200 model lives on {mine}; it cannot be moved to {device}")
        if dtype is not None and dtype != torch.float32:
            raise L.VBError("parameters stay fp32 (master weights); the tensor-core operand precision is chosen with precision=")
        return self

    def cuda(self, device=None):
        return self.to(torch.device("cuda", device) if isinstance(device, int) else (device or "cuda"))

    def float(self):
        return self

    def half(self):
        """The reference's --fp16 path (`model.half()` + apex FP16_Optimizer, train_concap.py:504-505): here the default precision
        already runs fp16 forward operands with fp32 master weights and accumulation, so this is a no-op for precision "fp16"."""
        if self.engine.precision != "fp16":
            raise L.VBError('model.half(): construct the model with precision="fp16" (the default)')
        return self

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, *model_args, config=None, state_dict=None, **kwargs):
        """Local files only (no network): a directory containing pytorch_model.bin (+ config.json) or a .bin file.
        Returns an eval-mode model like the reference (vilbert/utils.py:1022)."""
        kwargs.pop("default_gpu", None)
        if config is None:
            cfg_path = os.path.join(pretrained_model_name_or_path, "config.json")
            config = BertConfig.from_json_file(cfg_path)
        model = cls(config, *model_args, **kwargs)
        if state_dict is None:
            path = pretrained_model_name_or_path
            if os.path.isdir(path):
                path = os.path.join(path, "pytorch_model.bin")
            state_dict = torch.load(path, map_location="cpu")
        renamed = {}
        for k, v in state_dict.items():
            nk = k.replace("gamma", "weight") if "gamma" in k else k
            nk = nk.replace("beta", "bias") if "beta" in nk else nk
            if nk.startswith("module."):
                nk = nk[len("module."):]
            renamed[nk] = v
        own = model.state_dict()
        if not any(k.startswith("bert.") for k in renamed) and any(("bert." + k) in own for k in renamed):
            renamed = {"bert." + k: v for k, v in renamed.items()}   # base-model checkpoint into a model with heads
        # like the reference's loader (vilbert/utils.py:960-1012) missing and unexpected keys are tolerated but REPORTED
        missing = sorted(k for k in own if k not in renamed and k != "cls.predictions.decoder.weight")
        unexpected = sorted(k for k in renamed if k not in own)
        model.load_state_dict({k: v for k, v in renamed.items() if k in own}, strict=False)
        model.loading_info = {"missing_keys": missing, "unexpected_keys": unexpected}
        if missing or unexpected:
            import logging
            logging.getLogger(__name__).warning("from_pretrained(%s): %d missing keys (kept at their initial values): %s; %d unexpected keys (ignored): %s",
                                                pretrained_model_name_or_path, len(missing), missing[:8], len(unexpected), unexpected[:8])
        model.eval()
        return model

    def _attention_masks(self, output_all_attention_masks):
        """all_attention_mask of the reference's outputs: empty lists unless asked for; with config.visualization the attn_data
        dicts of every layer, without it one None per layer (BertEncoder appends whatever the layer returned, vilbert.py:974-1061)."""
        if not output_all_attention_masks:
            return ([], [], [])
        plan = self._last_plan
        if plan.viz:
            return plan.attention_export()
        c = self.config
        return ([None] * c.num_hidden_layers, [None] * c.v_num_hidden_layers, [None] * len(c.v_biattention_id))

    def _bert_forward(self, input_txt, input_imgs, image_loc, token_type_ids, attention_mask, image_attention_mask, task_ids,
                      output_all_encoded_layers, output_all_attention_masks=False):
        """BertModel.forward outputs (vilbert.py:1388-1406). With output_all_encoded_layers the encoded-layer entries are lists with
        one tensor per connection layer (:1075-1077); only the last entry is connected to autograd here."""
        o = self._run(BERT_OUT_NAMES, input_txt, input_imgs, image_loc, token_type_ids, attention_mask, image_attention_mask, task_ids)
        seq_t, seq_v = o["sequence_output_t"], o["sequence_output_v"]
        if output_all_encoded_layers:
            plan = self._last_plan
            B = seq_t.shape[0]
            enc_t = [a.f32.view(B, plan.Nt, -1).clone() for a in plan.enc_t]
            enc_v = [a.f32.view(B, plan.Nv, -1).clone() for a in plan.enc_v]
            # Reference quirk (:1098-1101, :1388-1394): in this mode the encoder returns ONLY the per-connection-layer states, and
            # BertModel pools encoded_layers[-1], i.e. the output of the last connection layer, not of the tail layers. This
            # inspection path (not the hot path) reproduces that with two tiny fp32 ops on the pooler parameters.
            pt = F.relu(F.linear(enc_t[-1][:, 0], self._params["bert.t_pooler.dense.weight"], self._params["bert.t_pooler.dense.bias"]))
            pv = F.relu(F.linear(enc_v[-1][:, 0], self._params["bert.v_pooler.dense.weight"], self._params["bert.v_pooler.dense.bias"]))
            return (enc_t, enc_v, pt, pv, self._attention_masks(output_all_attention_masks))
        return (seq_t, seq_v, o["pooled_output_t"], o["pooled_output_v"], self._attention_masks(output_all_attention_masks))

    # ---- shared forward machinery
    def _outputs_plan(self, names, inputs, train, live=None, frozen=None, input_grads=frozenset()):
        """The plan of the outputs `names`. A plan is specialised on the set of outputs that receive a gradient; the set `live` a
        backward found is kept as the hint for the next forward of this shape, so in a steady training loop forward and backward
        share one plan and nothing is recomputed. It is also specialised on the frozen parameters (default: the current
        requires_grad flags) and on the inputs it differentiates (_input_grads). With engine.recycle_forward_only an eval-mode call
        under torch.no_grad() takes the forward-only plan, whose buffers are placed by lifetime (Plan(recycle=True))."""
        if frozen is None:
            frozen = self._frozen()
        Nt = inputs["input_txt"].shape[1]
        B, Nv = inputs["input_imgs"].shape[:2]     # FAST_MODE: the text batch is 1, the image batch sets the plan
        key = (B, Nt, Nv, names, train)
        if live is None and self.engine.recycle_forward_only and not train and not torch.is_grad_enabled():
            live = ()
        elif live is None:
            live = self._grad_hint.get(key, ())
        else:
            self._grad_hint[key] = live
        return self.engine.plan(B, Nt, Nv, grad_outputs=live, heads=self._heads_for(names), train=train, frozen=frozen,
                                input_grads=input_grads)

    @staticmethod
    def _input_grads(inputs):
        """The float inputs of INPUT_GRAD_NAMES a call differentiates: those that require grad while grad mode is on (under
        torch.no_grad() none). A floating-point attention mask that requires grad is refused: its gradient would flow through the
        additive (1 - m) * -10000 mask, which the engine does not differentiate."""
        if not torch.is_grad_enabled():
            return frozenset()
        for k in ("attention_mask", "image_attention_mask"):
            m = inputs.get(k)
            if m is not None and m.requires_grad:
                raise NotImplementedError(f"{k} requires grad: gradients through the attention masks are not supported")
        return frozenset(n for n in INPUT_GRAD_NAMES if inputs[n] is not None and inputs[n].requires_grad)

    def _call(self, plan, inputs, targets=None, names=None):
        """One plan-backed call through the autograd bridge, with the inputs the plan differentiates as its autograd inputs."""
        call = _PlanCall(self, plan, inputs, targets, names)
        return _PlanFn.apply(self._anchor, call, *(inputs[n] for n in call.input_names))

    def _run(self, names, input_txt, input_imgs, image_loc, token_type_ids, attention_mask, image_attention_mask, task_ids):
        inputs = dict(input_txt=input_txt, input_imgs=input_imgs, image_loc=image_loc, token_type_ids=token_type_ids,
                      attention_mask=attention_mask, image_attention_mask=image_attention_mask, task_ids=task_ids)
        names = tuple(names)
        plan = self._outputs_plan(names, inputs, bool(self.training), input_grads=self._input_grads(inputs))
        outs = self._call(plan, inputs, names=names)
        return dict(zip(names, outs))


class BertModel(BertPreTrainedModel):
    """Reference: vilbert/vilbert.py:1288-1406. Parameters live under the bare names (embeddings.*, encoder.*)."""
    _heads = "none"

    def state_dict(self, *a, **k):
        sd = super().state_dict(*a, **k)
        return type(sd)((key[len("bert."):], v) for key, v in sd.items() if key.startswith("bert."))

    def load_state_dict(self, state_dict, strict=True):
        return super().load_state_dict({"bert." + k: v for k, v in state_dict.items()}, strict=strict)

    def forward(self, input_txt, input_imgs, image_loc, token_type_ids=None, attention_mask=None, image_attention_mask=None,
                co_attention_mask=None, task_ids=None, output_all_encoded_layers=False, output_all_attention_masks=False):
        return self._bert_forward(input_txt, input_imgs, image_loc, token_type_ids, attention_mask, image_attention_mask, task_ids,
                                  output_all_encoded_layers, output_all_attention_masks)


class VILBertForVLTasks(BertPreTrainedModel):
    """Reference: vilbert/vilbert.py:1600-1708. forward returns the same 10-tuple in the same order
    (:1697-1708). co_attention_mask is accepted and ignored exactly like the reference (:774-775, 796-797)."""
    _heads = "vl"

    def __init__(self, config, num_labels=1, dropout_prob=0.1, default_gpu=True, device=None, precision=None):
        super().__init__(config, device, precision)
        self.num_labels = num_labels
        self.dropout_prob = dropout_prob
        self.engine.head_dropout_prob = dropout_prob
        self.fusion_method = config.fusion_method

    def forward(self, input_txt, input_imgs, image_loc, token_type_ids=None, attention_mask=None, image_attention_mask=None,
                co_attention_mask=None, task_ids=None, output_all_encoded_layers=False, output_all_attention_masks=False):
        if output_all_encoded_layers:
            raise NotImplementedError("VILBertForVLTasks(output_all_encoded_layers=True) is not supported; use model.bert(..., output_all_encoded_layers=True)")
        if image_attention_mask is None:
            raise TypeError("image_attention_mask is required by VILBertForVLTasks.forward (vilbert.py:1693)")
        o = self._run(HEAD_NAMES, input_txt, input_imgs, image_loc, token_type_ids, attention_mask, image_attention_mask, task_ids)
        return tuple(o[n] for n in HEAD_NAMES) + (self._attention_masks(output_all_attention_masks),)


class BertForMultiModalPreTraining(BertPreTrainedModel):
    """Reference: vilbert/vilbert.py:1435-1597; the masked-region objective follows config.visual_target (0: KL divergence to the
    detector's class distribution, 1: feature regression, 2: noise-contrastive against sampled regions). The encoder
    and the three heads run on the engine; by default the three scalar losses are formed with torch on the head outputs
    exactly as the reference does (:1506-1590) and their gradients re-enter the engine through autograd.

    fused_objective=True: a call with masked_lm_labels, next_sentence_label and image_target runs the three objectives as fused
    kernels at the end of the forward (Plan(loss="pretraining", loss_in_forward=True)); no head output is cloned and the tied
    decoder runs on the labelled token rows only. The losses come back as [1]-shaped CUDA tensors whose backward scales each head
    gradient by its own d(total)/d(loss) on the device. Unlike the torch path, more labelled tokens than engine.lm_capacity of the
    rows make the masked-LM loss NaN.

    With engine.pack_padding set, such a call runs on a packed plan (Plan(packed=...), DESIGN.md §4g): the encoder and the three
    heads see the valid tokens and regions only, and the losses and gradients are those of the padded step up to fp32 summation
    order (_packed_rows says which batches pack)."""
    _heads = "pretraining"

    def __init__(self, config, device=None, precision=None, fused_objective=False):
        super().__init__(config, device, precision)
        self.visual_target = config.visual_target
        self.num_negative = config.num_negative
        self.fused_objective = bool(fused_objective)
        if self.visual_target not in (0, 1, 2):
            raise ValueError("visual_target must be 0, 1 or 2")

    def _nce_negatives(self, B, R, dev):
        """Flat region indices [B, R, n] of the negatives of visual_target == 2: 70 % from other samples, 30 % from other regions of
        the same sample, sampled on the device (`self.nce_sampler`, a callable (B, R, device) -> index, replaces it in tests)."""
        n_across, n_inside = int(self.num_negative * 0.7), int(self.num_negative * 0.3)
        rows = torch.randint(0, max(B - 1, 1), (B, R, n_across), device=dev)
        own = torch.arange(B, device=dev).view(B, 1, 1)
        rows = torch.where((rows == own) & (own < B - 1), torch.full_like(rows, B - 1), rows)     # never the sample itself
        across = rows * R + torch.randint(0, R, (B, R, n_across), device=dev)
        cols = torch.randint(0, max(R - 1, 1), (B, R, n_inside), device=dev)
        reg = torch.arange(R, device=dev).view(1, R, 1)
        cols = torch.where((cols == reg) & (reg < R - 1), torch.full_like(cols, R - 1), cols)     # never the region itself
        return torch.cat((across, own * R + cols), dim=2)

    def _nce_region_loss(self, pred, target, masked):
        """visual_target == 2: for every masked region, CE over [its own target feature, sampled negatives] scored by the dot
        product with the prediction (pinned against the reference with the reference's own sample: tiny_visual_target_2.json)."""
        B, R, _ = pred.shape
        dev = pred.device
        sampler = getattr(self, "nce_sampler", None)
        index = (sampler(B, R, dev) if sampler is not None else self._nce_negatives(B, R, dev))[masked]
        flat = target.reshape(B * R, -1)
        samples = torch.cat((target[masked].unsqueeze(1), flat[index]), dim=1)
        score = torch.bmm(samples, pred[masked].unsqueeze(2)).squeeze(2)
        return F.cross_entropy(score, torch.zeros(score.size(0), dtype=torch.long, device=dev))

    def forward(self, input_ids, image_feat, image_loc, token_type_ids=None, attention_mask=None, image_attention_mask=None,
                masked_lm_labels=None, image_label=None, image_target=None, next_sentence_label=None, output_all_attention_masks=False):
        if self.fused_objective and masked_lm_labels is not None and next_sentence_label is not None and image_target is not None:
            return self._fused_losses(input_ids, image_feat, image_loc, token_type_ids, attention_mask, image_attention_mask, masked_lm_labels,
                                      image_label, image_target, next_sentence_label)
        names = ("linguisic_prediction", "vision_prediction", "seq_relationship_score")
        o = self._run(names, input_ids, image_feat, image_loc, token_type_ids, attention_mask, image_attention_mask, None)
        prediction_scores_t, prediction_scores_v, seq_relationship_score = (o[n] for n in names)
        if masked_lm_labels is not None and next_sentence_label is not None and image_target is not None:
            prediction_scores_v = prediction_scores_v[:, 1:]
            masked = image_label == 1
            if self.visual_target == 0:      # KL to the soft class target (vilbert.py:1515-1521)
                img_loss = F.kl_div(F.log_softmax(prediction_scores_v, dim=2), image_target, reduction="none")
                masked_img_loss = torch.sum(img_loss * masked.unsqueeze(2).float()) / max(torch.sum(masked), 0)
            elif self.visual_target == 1:    # regression of the 2048-d region feature, mean over the masked elements (:1507-1513)
                img_loss = F.mse_loss(prediction_scores_v, image_target, reduction="none")
                masked_img_loss = torch.sum(img_loss * masked.unsqueeze(2).float()) / max(torch.sum(masked.unsqueeze(2).expand_as(img_loss)), 1)
            else:                            # contrastive: the true feature against num_negative sampled regions (:1523-1575)
                masked_img_loss = self._nce_region_loss(prediction_scores_v, image_target, masked)
            masked_lm_loss = F.cross_entropy(prediction_scores_t.view(-1, self.config.vocab_size), masked_lm_labels.view(-1), ignore_index=-1)
            next_sentence_loss = F.cross_entropy(seq_relationship_score.view(-1, 2), next_sentence_label.view(-1), ignore_index=-1)
            return masked_lm_loss.unsqueeze(0), masked_img_loss.unsqueeze(0), next_sentence_loss.unsqueeze(0)
        return prediction_scores_t, prediction_scores_v, seq_relationship_score, self._attention_masks(output_all_attention_masks)

    def _fused_losses(self, input_ids, image_feat, image_loc, token_type_ids, attention_mask, image_attention_mask, masked_lm_labels,
                      image_label, image_target, next_sentence_label):
        inputs = dict(input_txt=input_ids, input_imgs=image_feat, image_loc=image_loc, token_type_ids=token_type_ids,
                      attention_mask=attention_mask, image_attention_mask=image_attention_mask)
        targets = dict(masked_lm_labels=masked_lm_labels, image_label=image_label, image_target=image_target,
                       next_sentence_label=next_sentence_label)
        if self.visual_target == 2:
            B, R = image_feat.shape[0], image_feat.shape[1] - 1
            sampler = getattr(self, "nce_sampler", None)
            targets["neg_index"] = sampler(B, R, image_feat.device) if sampler is not None else self._nce_negatives(B, R, image_feat.device)
        B, Nv, Nt = image_feat.shape[0], image_feat.shape[1], input_ids.shape[1]
        input_grads = self._input_grads(inputs)
        packed = self._packed_rows(attention_mask, image_attention_mask, masked_lm_labels, image_label, B, Nt, Nv, input_grads)
        plan = self.engine.plan(B, Nt, Nv, grad_outputs=LOSS_HEADS["pretraining"] if torch.is_grad_enabled() else (), train=bool(self.training),
                                loss="pretraining", loss_in_forward=True, frozen=self._frozen(), input_grads=input_grads, packed=packed)
        return self._call(plan, inputs, targets)

    def _packed_rows(self, attention_mask, image_attention_mask, masked_lm_labels, image_label, B, Nt, Nv, input_grads):
        """(rows_t, rows_v) of the packed plan of a fused call when engine.pack_padding is set and the batch can be packed, else None;
        a batch that cannot is counted in engine.pack_fallbacks by reason (engine.pretraining_pack_rows). Host masks and labels
        are decided on the host with no device read. When any of them is on the device, one vb_pack_summary launch decides and one
        device-to-host copy reads its result: the host then waits for the work queued so far, once per forward."""
        eng = self.engine
        if not eng.pack_padding:
            return None
        check_pack_config(self.config)
        if not eng.lm_compact:
            raise NotImplementedError("engine.pack_padding packs the compacted masked-LM head only: set engine.lm_compact")
        if input_grads:
            raise NotImplementedError("engine.pack_padding does not compute input gradients (they are padded tensors)")
        ts = (attention_mask, image_attention_mask, masked_lm_labels, image_label)
        if any(t is not None and t.is_cuda for t in ts):
            rows = pretraining_pack_rows_from_summary(pack_summary(*ts, B, Nt, Nv), B, Nt, Nv)
        else:
            rows = pretraining_pack_rows(*ts, B, Nt, Nv)
        if isinstance(rows, str):
            eng.pack_fallbacks[rows] += 1
            return None
        return rows
