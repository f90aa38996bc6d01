"""Closed forms of the masked-region objectives of visual_target 1 and 2 (vilbert.py:1507-1513, 1523-1575) as the fused kernels
vb_mse_masked_loss and vb_nce_region_loss compute them: loss and d loss / d scores over the whole [B, Nv, D] prediction, in the
precision of the inputs (the tests use float64). test_pretraining_cpu.py checks them against torch autograd of the reference's
expressions; test_pretraining_gpu.py checks the kernels against them."""
import torch


def mse_closed_form(scores, target, label):
    """scores [B, Nv, D], target [B, Nv-1, D], label [B, Nv-1] -> (loss, d scores); no masked row gives loss 0."""
    B, Nv, D = scores.shape
    m = (label == 1).to(scores.dtype).unsqueeze(2)
    denom = max(float(m.sum()) * D, 1.0)
    e = (scores[:, 1:] - target) * m
    d = torch.zeros_like(scores)
    d[:, 1:] = 2.0 * e / denom
    return (e * e).sum() / denom, d


def nce_closed_form(scores, target, label, neg_index):
    """neg_index [B, Nv-1, n] (flat rows of target viewed as [B * R, D]) -> (loss, d scores). Candidate 0 is the row's own target;
    loss = mean over the masked rows of CE(score, 0); no masked row gives NaN; an index outside [0, B * R) gives NaN and is skipped
    in the gradient."""
    B, Nv, D = scores.shape
    R = Nv - 1
    flat = target.reshape(B * R, D)
    masked = (label == 1).nonzero().tolist()
    d = torch.zeros_like(scores)
    if not masked:
        return torch.tensor(float("nan"), dtype=scores.dtype), d
    n_pos = len(masked)
    total = torch.zeros((), dtype=scores.dtype)
    for b, r in masked:
        rows = [b * R + r] + neg_index[b, r].tolist()
        ok = torch.tensor([0 <= i < B * R for i in rows])
        cand = torch.stack([flat[i] if 0 <= i < B * R else torch.zeros(D, dtype=scores.dtype) for i in rows])
        s = cand @ scores[b, r + 1]
        if not ok.all():
            total = total + float("nan")
            s = s.masked_fill(~ok, float("-inf"))
        p = torch.softmax(s, 0)
        if ok.all():
            total = total + (torch.logsumexp(s, 0) - s[0]) / n_pos
        w = p.clone()
        w[0] -= 1.0
        d[b, r + 1] = (w.unsqueeze(1) * cand).sum(0) / n_pos
    return total, d


def nce_reference(scores, target, label, neg_index):
    """The reference's expression (vilbert.py:1558-1575 as the module surface writes it): gather, bmm, F.cross_entropy."""
    B, Nv, D = scores.shape
    R = Nv - 1
    masked = label == 1
    sv = scores[:, 1:]
    samples = torch.cat((target[masked].unsqueeze(1), target.reshape(B * R, D)[neg_index[masked]]), dim=1)
    score = torch.bmm(samples, sv[masked].unsqueeze(2)).squeeze(2)
    return torch.nn.functional.cross_entropy(score, torch.zeros(score.shape[0], dtype=torch.long))


def mse_reference(scores, target, label):
    """vilbert.py:1507-1513."""
    sv = scores[:, 1:]
    masked = (label == 1).unsqueeze(2)
    img_loss = torch.nn.functional.mse_loss(sv, target, reduction="none")
    return torch.sum(img_loss * masked.to(sv.dtype)) / max(torch.sum(masked.expand_as(img_loss)), 1)


def negative_count(num_negative):
    return int(num_negative * 0.7) + int(num_negative * 0.3)
