"""Times the device ranking of both retrieval directions from one score matrix at the sizes of Flickr30k / COCO-1k (5,000 captions x
1,000 images) and COCO-5k (25,000 x 5,000), five captions per image: RetrievalEvaluator.rank (caption-to-image, vb_retrieval_rank)
and RetrievalEvaluator.rank_captions (image-to-text: the transpose, the CSR caption sets and vb_retrieval_rank_sets), k = 20.

    python tools/retrieval_rank_probe.py [--reps 20] [--out retrieval_rank_probe.json]

Random scores quantised to 0.01 (ties occur). Each call is timed with CUDA events after a warm-up; reports the median and min-max
per call and the card's name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from retrieval_probe import card  # noqa: E402


def time_call(fn, reps):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return dict(median_ms=statistics.median(ms), min_ms=min(ms), max_ms=max(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from vilbert_b200.retrieval import RetrievalEvaluator
    res = dict(card=card(), k=20, reps=args.reps, shapes=[])
    for C, G in ((5000, 1000), (25000, 5000)):
        g = torch.Generator(device="cuda").manual_seed(0)
        scores = (torch.randn(C, G, device="cuda", generator=g) * 3).round(decimals=2)
        target = torch.arange(C, device="cuda") // (C // G)
        row = dict(captions=C, images=G,
                   t2i=time_call(lambda: RetrievalEvaluator.rank(scores, target, k=20), args.reps),
                   i2t=time_call(lambda: RetrievalEvaluator.rank_captions(scores, target, k=20), args.reps))
        res["shapes"].append(row)
        print(f"{C} x {G}: t2i {row['t2i']['median_ms']:.3f} ms ({row['t2i']['min_ms']:.3f}-{row['t2i']['max_ms']:.3f}), "
              f"i2t {row['i2t']['median_ms']:.3f} ms ({row['i2t']['min_ms']:.3f}-{row['i2t']['max_ms']:.3f})")
    print(json.dumps(res["card"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
