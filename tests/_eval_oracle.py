"""Restatement of the reference's per-task evaluation step, EvaluatingModel (vilbert/task_utils.py:626-859): the batch reshapes of
each `process`, one forward under no_grad, then the loss, the batch score and the result dicts of the task type, formed from the
head outputs as the reference forms them. What vilbert_b200.tasks.EvaluatingModel is checked against (on the GPU, with the module
surface as the model) and what tests/golden/evaluating_model_reference.json pins (on the CPU, with the head outputs the reference
saw).

`question_id[i].item()` is read per result row, as the reference reads it: a VisDial batch (`dialog`) carries one id per image but
yields batch_size * rounds result rows, so it raises IndexError once the rows outrun the ids (the rows before are appended)."""
import torch
import torch.nn.functional as F

import _task_oracle as T

# the (type, loss) pairs EvaluatingModel forms a result for (task_utils.py:777-857); Foil (VL-binary-classifier with
# CrossEntropyLoss) fails in the loss or the score
EVAL_TYPES = ("VL-classifier", "VL-classifier-GQA", "VL-logit", "V-logit", "V-logit-mc", "VL-binary-classifier", "VL-tri-classifier")


def _loss(name, x, t):
    """The modules of LoadLosses (task_utils.py:25-28): BCEWithLogitsLoss(reduction="mean") or CrossEntropyLoss()."""
    return T.bce(x, t) if name == "BCEWithLogitLoss" else F.cross_entropy(x, t)


def results_of(task_type, loss_name, heads, target, question_id, label2ans, results, mc_ids=None, batch_size=None, num_options=None):
    """(float(loss), float(batch_score)) of one evaluation batch from the ten outputs; result dicts are appended to `results`."""
    vil_prediction, vil_prediction_gqa, vil_logit, vil_binary, vil_tri, _, vision_logit = heads[:7]

    def qid(i):
        return question_id[i].item()
    if task_type in ("VL-classifier", "VL-classifier-GQA"):                      # :777-803, argmax answer, no loss / score
        lg = vil_prediction if task_type == "VL-classifier" else vil_prediction_gqa
        pick = torch.max(lg, 1)[1]
        for i in range(pick.size(0)):
            if task_type == "VL-classifier":
                results.append({"question_id": qid(i), "answer": label2ans[pick[i].item()]})
            else:
                results.append({"questionId": str(qid(i)), "prediction": label2ans[pick[i].item()]})
        return 0.0, 0.0
    if task_type == "VL-logit":                                                   # :805-818, softmax over the options
        lg = vil_logit.view(batch_size, num_options)
        loss = _loss(loss_name, lg, target)
        score = (torch.max(lg, 1)[1] == target).sum()
        probs = torch.softmax(lg, dim=1)
        for i in range(lg.size(0)):
            results.append({"question_id": qid(i), "answer": probs[i].tolist()})
        return float(loss), float(score)
    if task_type == "V-logit":                                                    # :820-834, argmax region and its IoU
        loss = _loss(loss_name, vision_logit, target).mean() * target.size(1)
        pick = torch.max(vision_logit, dim=1)[1]
        iou = target.squeeze(2).gather(1, pick.view(-1, 1))
        score = (iou > 0.5).sum()
        for i in range(pick.size(0)):
            results.append({"id": qid(i), "target": pick[i].item(), "IOU": iou[i].item()})
        return float(loss), float(score)
    if task_type == "V-logit-mc":                                                 # :836-847, argmax over the gathered choices
        lg = vision_logit[:, T.MC_OFFSET:].squeeze(2).gather(1, mc_ids).unsqueeze(2)
        loss = _loss(loss_name, lg, target).mean() * target.size(1)
        pick = torch.max(lg, dim=1)[1]
        score = (pick == torch.max(target, dim=1)[1]).sum()
        for i in range(pick.size(0)):
            results.append({"id": qid(i), "target": pick[i].item()})
        return float(loss), float(score)
    if task_type in ("VL-binary-classifier", "VL-tri-classifier"):                # :849-857, no results
        lg = vil_binary if task_type == "VL-binary-classifier" else vil_tri
        loss = _loss(loss_name, lg, target).mean()
        return float(loss), float(T.score_with_logits(lg, target).sum())
    raise ValueError(task_type)


def task_results_rule(logits, mode, target=None):
    """What vb_task_results computes, row by row: (argmax [rows] with torch.max's rules, values). mode "argmax": no values;
    "softmax": exp(x - max) / sum in float64, rounded to float32 (a NaN maximum or an infinite one gives a NaN row); "gather":
    target[r, argmax]."""
    pick = torch.tensor([T.argmax_torch_rule(r) for r in logits], dtype=torch.int64)
    if mode == "argmax":
        return pick, None
    if mode == "gather":
        return pick, target.gather(1, pick.view(-1, 1)).view(-1)
    x = logits.double()
    mx = x.gather(1, pick.view(-1, 1))
    e = torch.exp(x - mx)
    return pick, (e / e.sum(1, keepdim=True)).float()


def evaluating_step(task_cfg, task_id, batch, model, label2ans, results, others):
    """EvaluatingModel's body on `batch` (tensors on the model's device) with `model` any callable of the reference's forward
    signature returning the ten outputs. Returns (float(loss), float(batch_score), batch_size, results, others)."""
    if task_id in ("TASK4", "TASK17"):
        features, spatials, image_mask, question, target, input_mask, segment_ids, mc_ids, _, question_id = batch
    else:
        features, spatials, image_mask, question, target, input_mask, segment_ids, _, question_id = batch
        mc_ids = None
    cfg = task_cfg[task_id]
    (features, spatials, image_mask, question, input_mask, segment_ids), target, batch_size, num_options = T.reshape_batch(
        cfg["process"], features.size(0), features, spatials, image_mask, question, input_mask, segment_ids, target)
    task_tokens = question.new_full((question.size(0), 1), int(task_id[4:]))
    with torch.no_grad():
        heads = model(question, features, spatials, segment_ids, input_mask, image_mask, None, task_tokens)
    loss, score = results_of(cfg["type"], cfg["loss"], heads, target, question_id, label2ans, results, mc_ids, batch_size, num_options)
    return loss, score, batch_size, results, others
