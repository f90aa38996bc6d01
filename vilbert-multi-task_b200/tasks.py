"""Drop-in replacements for the reference's per-task training, validation and evaluation steps, ForwardModelsTrain,
ForwardModelsVal (vilbert/task_utils.py:31-376) and EvaluatingModel (:626-859), with the same signatures and return values:

    from vilbert_b200.tasks import EvaluatingModel, ForwardModelsTrain, ForwardModelsVal, LoadLosses

Each call runs ONE plan of the engine in which the task's objective and its batch score are fused kernels at the end of the forward
(Plan(loss_in_forward=True, score=True)): no head outputs are cloned, no torch loss is formed, and no score is read back to the host.
The task table's (type, loss) pairs map to the engine's objective kinds as in TASK_KINDS below.

Reference behaviour that is reproduced, not fixed (INTEGRATION.md):
  * batch_size is taken before the batch is reshaped: questions for `expand`, image pairs for `nlvr`, question rounds for `dialog`;
  * ForwardModelsVal returns the summed batch score, ForwardModelsTrain the score divided by batch_size;
  * the VL-binary-classifier with CrossEntropyLoss (Foil, TASK16) fails as in the reference: with an even batch the CE refuses the
    per-sample int labels of the paired head (ValueError), otherwise compute_score_with_logits raises on the 1-D labels (IndexError,
    task_utils.py:618-623 scatters into a 1-D tensor).
What differs: ForwardModelsTrain returns `score` as a 0-d CUDA tensor (float(score) gives the reference's number) and takes the
next batch with next() (the reference calls the Python 2 `.next()`).
"""
import torch
import torch.nn as nn

from .data import expand_batch
from .engine import LOSS_HEADS, MC_REGION_OFFSET, RESULT_MODES, check_pack_config, pack_capacity, prefix_lengths
from .modeling import _PlanCall, _PlanFn

LossMap = {
    "BCEWithLogitLoss": nn.BCEWithLogitsLoss,
    "CrossEntropyLoss": nn.CrossEntropyLoss,
}

# (task type, loss) of vilbert_tasks.yml -> the engine's objective kind
TASK_KINDS = {
    ("VL-classifier", "BCEWithLogitLoss"): "vqa",
    ("VL-classifier-GQA", "BCEWithLogitLoss"): "gqa",
    ("VL-logit", "CrossEntropyLoss"): "logit_ce",
    ("V-logit", "BCEWithLogitLoss"): "vlogit_bce",
    ("V-logit-mc", "BCEWithLogitLoss"): "vlogit_mc",
    ("VL-binary-classifier", "BCEWithLogitLoss"): "binary_bce",
    ("VL-binary-classifier", "CrossEntropyLoss"): "binary_ce",
    ("VL-tri-classifier", "BCEWithLogitLoss"): "tri_bce",
    ("VL-tri-classifier", "CrossEntropyLoss"): "tri_ce",
}

_NO_SCORE = ("binary_ce", "tri_ce")


def LoadLosses(args, task_cfg, task_ids):
    """The reference's LoadLosses (task_utils.py:379-391): task id -> the loss module its `loss` entry names."""
    return {"TASK" + t: LossMap[task_cfg["TASK" + t]["loss"]](**({"reduction": "mean"} if task_cfg["TASK" + t]["loss"] == "BCEWithLogitLoss" else {}))
            for t in task_ids}


def task_kind(task_cfg, task_id):
    """The engine objective kind of one task of the task table."""
    key = (task_cfg[task_id]["type"], task_cfg[task_id]["loss"])
    if key not in TASK_KINDS:
        raise NotImplementedError(f"{task_id}: task type {key[0]!r} with loss {key[1]!r} has no fused objective")
    return TASK_KINDS[key]


def _check_loss(task_cfg, task_id, task_losses):
    """The fused objectives restate the modules LoadLosses builds (BCEWithLogitsLoss(reduction="mean"), CrossEntropyLoss()); any
    other module would be silently ignored, so it is refused."""
    name = task_cfg[task_id]["loss"]
    fn = task_losses[task_id] if task_losses is not None and task_id in task_losses else None
    want = LossMap.get(name)
    ok = want is not None and type(fn) is want and fn.reduction == "mean" and getattr(fn, "weight", None) is None
    if ok and want is nn.BCEWithLogitsLoss:
        ok = fn.pos_weight is None
    if ok and want is nn.CrossEntropyLoss:
        ok = fn.ignore_index == -100 and fn.label_smoothing == 0.0
    if not ok:
        raise NotImplementedError(f"task_losses[{task_id!r}] must be the {name} module LoadLosses builds, got {fn!r}")


def _unpack(task_id, batch):
    """task_utils.py:189-196: Visual7w (TASK4) and GuessWhatPointing (TASK17) carry multiple_choice_ids."""
    if task_id in ("TASK4", "TASK17"):
        features, spatials, image_mask, question, target, input_mask, segment_ids, mc_ids, co_attention_mask, question_id = batch
    else:
        features, spatials, image_mask, question, target, input_mask, segment_ids, co_attention_mask, question_id = batch
        mc_ids = None
    return features, spatials, image_mask, question, target, input_mask, segment_ids, mc_ids, co_attention_mask


def packed_rows(model, task_cfg, task_id, batch, processes):
    """The (rows_t, rows_v) capacities of a packed plan for this batch when model.engine.pack_padding is set and the batch can be
    packed, else None. Decided from the host tensors before the batch moves, so it forces no sync. The masks are replicated as the
    task's `process` replicates them. A batch can be packed when both masks are prefix-valid with at least one valid entry per row
    ("mask"), no V-logit target is non-zero on a masked region ("target": the padded loss would read that region's logit and send
    it a gradient) and no gathered V-logit-mc choice with a non-zero target sits on a masked region, nor do all of a sample's choices
    (its argmax would then fall among masked logits, which the padded plan leaves at logit - 10000) ("choice"); otherwise it runs
    padded and engine.pack_fallbacks counts the reason ("device": the masks are already on the device). Train mode packs too: the
    packed plan draws the padded plan's dropout masks."""
    eng = model.engine
    if not eng.pack_padding:
        return None
    cfg = eng.cfg
    check_pack_config(cfg)

    def fallback(reason):
        eng.pack_fallbacks[reason] += 1
        return None

    features, spatials, image_mask, question, target, input_mask, segment_ids, mc_ids, _ = _unpack(task_id, batch)
    if any(t is not None and t.is_cuda for t in (image_mask, input_mask, target, mc_ids)):
        return fallback("device")
    process = task_cfg[task_id]["process"]
    if process in processes:     # the masks as expand_batch lays them out (a one-wide stand-in for the features and boxes)
        stand_in = image_mask.unsqueeze(-1)
        _, _, image_mask, _, input_mask, _, _, _, _ = expand_batch(process, stand_in, stand_in, image_mask, question, input_mask, input_mask)
    lt, lv = prefix_lengths(input_mask), prefix_lengths(image_mask)
    if lt is None or lv is None:
        return fallback("mask")
    kind = task_kind(task_cfg, task_id)
    if kind == "vlogit_bce" and target.numel() == image_mask.numel():
        if bool((target.reshape(image_mask.shape).ne(0) & image_mask.eq(0)).any()):
            return fallback("target")
    if mc_ids is not None and kind == "vlogit_mc":
        region = mc_ids.long() + MC_REGION_OFFSET
        masked = region.ge(lv.unsqueeze(1))
        if bool((target.reshape(mc_ids.shape).ne(0) & masked).any()) or bool(masked.all(1).any()):
            return fallback("choice")
    B, Nt, Nv = input_mask.size(0), input_mask.size(1) + (1 if cfg.task_specific_tokens else 0), image_mask.size(1)
    rows_t = int(lt.sum()) + (B if cfg.task_specific_tokens else 0)
    return pack_capacity(rows_t, B * Nt), pack_capacity(int(lv.sum()), B * Nv)


class _Step:
    """One task batch on the device, reshaped for the model, with the plan of its objective and the call that runs it."""

    def __init__(self, task_cfg, task_id, batch, model, train, grad, processes, evaluate=False, packed=None):
        eng = model.engine
        self.kind = kind = task_kind(task_cfg, task_id)
        features, spatials, image_mask, question, target, input_mask, segment_ids, mc_ids, _ = _unpack(task_id, batch)
        process = task_cfg[task_id]["process"]
        batch_size = features.size(0)
        if process in processes:
            features, spatials, image_mask, question, input_mask, segment_ids, _, B, num_options = expand_batch(
                process, features, spatials, image_mask, question, input_mask, segment_ids)
            if process == "dialog":
                target = target.reshape(-1)
                batch_size = B
        else:
            num_options = None     # VL-logit tasks are always expanded (otherwise the engine's default, engine.loss_options)
        self.batch_size = batch_size
        task_tokens = question.new_full((question.size(0), 1), int(task_id[4:]))
        B, Nt = question.shape
        Nv = features.size(1)
        choices = None
        if kind == "logit_ce":
            choices = num_options
        elif kind == "vlogit_mc":
            choices = mc_ids.size(1)
        if evaluate:
            # EvaluatingModel: a forward-only plan of the one head the type reads; VL-classifier / GQA have no loss and no score
            has_loss = kind not in ("vqa", "gqa")
            plan = eng.plan(B, Nt, Nv, train=train, loss=kind if has_loss else None, choices=choices,
                            score=has_loss and kind not in _NO_SCORE, loss_in_forward=has_loss, outputs=LOSS_HEADS[kind],
                            results=kind if kind in RESULT_MODES else None, packed=packed)
        else:
            # a packed plan builds the objective's head only: the step returns nothing else, and a kept head is bitwise the same
            plan = eng.plan(B, Nt, Nv, grad_outputs=LOSS_HEADS[kind] if grad else (), train=train, loss=kind, choices=choices,
                            score=kind not in _NO_SCORE, loss_in_forward=True, frozen=model._frozen(),
                            outputs=None if packed is None else LOSS_HEADS[kind], packed=packed)
        inputs = dict(input_txt=question, input_imgs=features, image_loc=spatials, token_type_ids=segment_ids, attention_mask=input_mask,
                      image_attention_mask=image_mask, task_ids=task_tokens)
        targets = {}
        li = plan.loss_inputs
        if "labels" in li:
            if target.numel() != li["labels"].numel():
                # Foil with an even batch: the binary head pairs consecutive samples (vilbert.py:1686-1689) and CrossEntropyLoss
                # refuses the int labels of every sample, as F.cross_entropy does in the reference
                raise ValueError(f"Expected input batch_size ({li['labels'].numel()}) to match target batch_size ({target.numel()}).")
            targets["labels"] = target.reshape(li["labels"].shape)
        elif "target" in li:
            targets["target"] = target.reshape(li["target"].shape)
        if mc_ids is not None and "multiple_choice_ids" in li:
            targets["multiple_choice_ids"] = mc_ids
        self.plan, self.call = plan, _PlanCall(model, plan, inputs, targets)

    def score_error(self):
        if self.kind in _NO_SCORE:
            raise IndexError(f"{self.kind}: the reference's compute_score_with_logits scatters the argmax into a 1-D one-hot of the int "
                             "labels and raises 'Dimension out of range' (task_utils.py:618-623); there is no score to reproduce")


def _model(model):
    m = getattr(model, "module", model)    # a data-parallel wrapper around the model
    if not hasattr(m, "engine") or m._heads != "vl":
        raise TypeError("ForwardModelsTrain / ForwardModelsVal need a vilbert_b200 VILBertForVLTasks")
    return m


def ForwardModelsTrain(args, task_cfg, device, task_id, task_count, task_iter_train, task_dataloader_train, model, task_losses):
    """task_utils.py:167-376. Returns (loss, score): loss a 0-d CUDA tensor whose backward() runs the fused backward into the model's
    gradients; score a 0-d CUDA tensor, batch_score / batch_size."""
    if task_count[task_id] % len(task_dataloader_train[task_id]) == 0:
        task_iter_train[task_id] = iter(task_dataloader_train[task_id])
    task_count[task_id] += 1
    batch = next(task_iter_train[task_id])
    m = _model(model)
    processes = ("dialog", "expand", "retrieval", "nlvr")
    packed = packed_rows(m, task_cfg, task_id, batch, processes)
    batch = tuple(t.cuda(device=device, non_blocking=True) for t in batch)
    _check_loss(task_cfg, task_id, task_losses)
    step = _Step(task_cfg, task_id, batch, m, bool(m.training), True, processes, packed=packed)
    loss, = _PlanFn.apply(m._anchor, step.call)
    step.score_error()
    score = step.plan.score.reshape(()) / float(step.batch_size)
    return loss, score


def ForwardModelsVal(args, task_cfg, device, task_id, batch, model, task_losses):
    """task_utils.py:31-164: (float(loss), float(batch_score), batch_size) from a forward-only plan in the model's current mode,
    with one device-to-host copy of (loss, score). The reference's validation step has no `dialog` reshape; neither has this one."""
    m = _model(model)
    processes = ("expand", "retrieval", "nlvr")
    packed = packed_rows(m, task_cfg, task_id, batch, processes)
    batch = tuple(t.cuda(device=device, non_blocking=True) for t in batch)
    _check_loss(task_cfg, task_id, task_losses)
    with torch.no_grad():
        step = _Step(task_cfg, task_id, batch, m, bool(m.training), False, processes, packed=packed)
        step.call.forward()
        step.score_error()
        loss, score = step.plan.objective_out.tolist()
    return loss, score, step.batch_size


# the objective kinds EvaluatingModel forms results for (task_utils.py:777-857); binary_ce (Foil) fails like ForwardModelsVal
_EVAL_KINDS = ("vqa", "gqa", "logit_ce", "vlogit_bce", "vlogit_mc", "binary_bce", "tri_bce", "binary_ce")


def EvaluatingModel(args, task_cfg, device, task_id, batch, model, task_dataloader, task_losses, results, others):
    """task_utils.py:626-859: (float(loss), float(batch_score), batch_size, results, others), the result dicts of the task type
    appended to `results`. One forward-only plan in the model's current mode builds only the head the type reads and ends with the
    type's objective, its score and vb_task_results (argmax, option probabilities or the IoU at the argmax); one device-to-host
    copy reads loss, score and every per-row result, and the dicts are built on the host. question_id is read from the batch as
    passed in; a row without an id (VisDial's `dialog` batches carry one id per image for batch_size * rounds rows) raises
    IndexError after the rows before it are appended, as in the reference."""
    kind = task_kind(task_cfg, task_id)
    if kind not in _EVAL_KINDS:
        raise NotImplementedError(f"{task_id}: EvaluatingModel has no result for task type {task_cfg[task_id]['type']!r} with loss "
                                  f"{task_cfg[task_id]['loss']!r}")
    question_id = batch[-1].tolist()
    m = _model(model)
    processes = ("dialog", "expand", "retrieval", "nlvr")
    packed = packed_rows(m, task_cfg, task_id, batch, processes)
    batch = tuple(t.cuda(device=device, non_blocking=True) for t in batch)
    if kind not in ("vqa", "gqa"):            # VL-classifier / GQA do not read task_losses
        _check_loss(task_cfg, task_id, task_losses)
    with torch.no_grad():
        step = _Step(task_cfg, task_id, batch, m, bool(m.training), False, processes, evaluate=True, packed=packed)
        step.score_error()
        step.call.forward()
        plan = step.plan
        if plan.results is None:              # VL-binary / VL-tri: loss and score only
            loss, score = plan.objective_out.tolist()
            return loss, score, step.batch_size, results, others
        loss, score, argmax, values = plan.fetch_results()
    pick = argmax.tolist()
    if kind in ("vqa", "gqa"):
        label2ans = task_dataloader[task_id].dataset.label2ans
        for i, a in enumerate(pick):
            results.append({"question_id": question_id[i], "answer": label2ans[a]} if kind == "vqa" else
                           {"questionId": str(question_id[i]), "prediction": label2ans[a]})
    elif kind == "logit_ce":
        for i, probs in enumerate(values.tolist()):
            results.append({"question_id": question_id[i], "answer": probs})
    elif kind == "vlogit_bce":
        iou = values.view(-1).tolist()
        for i, a in enumerate(pick):
            results.append({"id": question_id[i], "target": a, "IOU": iou[i]})
    else:                                     # vlogit_mc
        for i, a in enumerate(pick):
            results.append({"id": question_id[i], "target": a})
    return loss, score, step.batch_size, results, others


__all__ = ["EvaluatingModel", "ForwardModelsTrain", "ForwardModelsVal", "LoadLosses", "TASK_KINDS", "packed_rows", "task_kind"]
