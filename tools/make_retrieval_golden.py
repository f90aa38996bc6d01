"""Writes tests/golden/retrieval_reference.json: the five retrieval metrics the reference's UNMODIFIED evaluate()
(evaluation/eval_coco_retrieval.py:336-412) returns on the CPU for a stub model with seeded scores, for both `zero_shot` settings.

    python tools/make_retrieval_golden.py [--reference /path/to/vilbert-multi-task]

The script's imports that only serve data loading and logging (multimodal_bert.*, pytorch_pretrained_bert.*, tensorboardX, tqdm)
are stubbed and torch.Tensor.cuda is the identity. The loader yields the reference's 5,000 x 2 batches (caption c against gallery
half h, five captions per image: caption c's image is c // 5). The stub model returns row c, columns 500 h ... 500 h + 499 of a seeded
tie-free logit matrix (seeded_scores): [5000, 1000] for the fine-tuned path, [5000, 1000, 2] for the zero-shot one (scored as
softmax(logits, 1)[:, 0]). tests/test_retrieval_cpu.py regenerates the scores
from the stored seeds and checks vilbert_b200.retrieval against the metrics; nothing on the GPU reads the reference."""
import argparse
import importlib.util
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "retrieval_reference.json")
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
N_CAPTIONS, N_IMAGES, HALF, PER_IMAGE = 5000, 1000, 500, 5


def seeded_scores(seed, zero_shot):
    """float64 [5000, 1000] scores as the reference stores them, from the stub model's seeded float32 logits. Tie-free by
    construction: each row is a seeded permutation of 1,000 distinct values (the zero-shot path puts them in the first of its two
    logits, the second being 0, so the score is a strictly increasing function of them)."""
    g = torch.Generator().manual_seed(seed)
    perm = torch.argsort(torch.rand(N_CAPTIONS, N_IMAGES, generator=g), dim=1).float()
    x = perm / 100.0 - 5.0
    if zero_shot:
        logits = torch.stack((x, torch.zeros_like(x)), dim=2)
        return torch.softmax(logits, dim=2)[:, :, 0].double().numpy(), logits
    return x.double().numpy(), x


def tie_free(scores):
    s = np.sort(scores, axis=1)
    return not (s[:, 1:] == s[:, :-1]).any()


def load_evaluate(reference):
    for name, attrs in (("multimodal_bert", {}),
                        ("multimodal_bert.datasets", {"COCORetreivalDatasetTrain": object, "COCORetreivalDatasetVal": object}),
                        ("multimodal_bert.datasets._image_features_reader", {"ImageFeaturesH5Reader": object}),
                        ("pytorch_pretrained_bert", {}), ("pytorch_pretrained_bert.tokenization", {"BertTokenizer": object}),
                        ("pytorch_pretrained_bert.optimization", {"BertAdam": object, "WarmupLinearSchedule": object}),
                        ("tensorboardX", {"SummaryWriter": object}), ("tqdm", {"tqdm": lambda it, *a, **k: it})):
        mod = types.ModuleType(name)
        mod.__dict__.update(attrs)
        sys.modules[name] = mod
    torch.Tensor.cuda = lambda self, *a, **k: self
    path = os.path.join(reference, "evaluation", "eval_coco_retrieval.py")
    spec = importlib.util.spec_from_file_location("eval_coco_retrieval", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.evaluate


class StubModel:
    """Returns the seeded logits of (caption, gallery half): the caption id rides in caption[0, 0], the half in features[0, 0, 0]."""

    def __init__(self, logits, zero_shot):
        self.logits, self.zero_shot = logits, zero_shot

    def eval(self):
        return self

    def __call__(self, caption, features, spatials, segment_ids, input_mask, image_mask):
        c, h = int(caption[0, 0]), int(features[0, 0, 0])
        rows = self.logits[c, HALF * h:HALF * (h + 1)]
        if self.zero_shot:
            return None, None, rows, None
        return rows.view(HALF, 1)


def loader():
    """The reference DataLoader's batches (batch_size 1): item 2c + h, with a leading batch dimension."""
    for c in range(N_CAPTIONS):
        for h in range(2):
            target = torch.zeros(1, HALF)
            img = c // PER_IMAGE - HALF * h
            if 0 <= img < HALF:
                target[0, img] = 1
            yield (torch.full((1, HALF, 1, 1), float(h)), torch.zeros(1, HALF, 1, 5), torch.ones(1, HALF, 1, dtype=torch.long),
                   torch.tensor([[c, 0]]), torch.ones(1, 2, dtype=torch.long), torch.zeros(1, 2, dtype=torch.long), target,
                   torch.tensor([c]), torch.tensor([h]))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--reference", default=ref_loader.REFERENCE_ROOT, help="reference checkout (default: as oracle/ref_loader.py finds it)")
    a = ap.parse_args()
    evaluate = load_evaluate(a.reference)
    cases = []
    for zero_shot in (False, True):
        seed = 7 + int(zero_shot)
        scores, logits = seeded_scores(seed, zero_shot)
        if not tie_free(scores):
            raise SystemExit(f"seed {seed}: tied scores")
        metrics = evaluate(types.SimpleNamespace(zero_shot=zero_shot), StubModel(logits, zero_shot), loader())
        cases.append({"zero_shot": zero_shot, "seed": seed, "scores_row0_head": [float(x) for x in scores[0, :4]],
                      "metrics": [float(m) for m in metrics]})
        print(f"zero_shot={zero_shot} seed={seed}: r1 {metrics[0]:.3f} r5 {metrics[1]:.3f} r10 {metrics[2]:.3f} medr {metrics[3]} "
              f"meanr {metrics[4]:.3f}")
    out = {"source": "evaluation/eval_coco_retrieval.py:336-412 evaluate(), unmodified, on the CPU with a stub model",
           "captions": N_CAPTIONS, "images": N_IMAGES, "captions_per_image": PER_IMAGE, "cases": cases}
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
