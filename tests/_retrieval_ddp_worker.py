"""2-rank worker of tests/test_retrieval_ddp_gpu.py (launched with torch.distributed.run): evaluate_retrieval_both sharded over the
ranks (group=dist.group.WORLD) against the single-process call made in the same worker, for the fine-tuned model with task tokens
and the zero-shot pre-training model, padded and packed, with and without torch.use_deterministic_algorithms(True).

    python -m torch.distributed.run --nproc-per-node 2 tests/_retrieval_ddp_worker.py OUT.json nccl    # one GPU per rank
    python -m torch.distributed.run --nproc-per-node 2 tests/_retrieval_ddp_worker.py OUT.json gloo    # both ranks on cuda:0

The gallery has 12 images in chunks of 5 (a short last chunk) with ragged image masks; 7 captions split 3 + 4 over the ranks, and
1 caption leaves rank 0's block empty. Rank 0 writes every rank's results to OUT.json."""
import json
import os
import sys
from datetime import timedelta

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_retrieval_i2t_gpu import _Dataset, _cfgj, _model     # noqa: E402

G, NV, NT, CHUNK, K = 12, 11, 9, 5, 10


def dataset(cfgj, C, seed):
    """C captions (caption c -> image 5c mod 12) of ragged lengths against 12 images with ragged, prefix-valid masks."""
    g = torch.Generator().manual_seed(seed)
    ds = _Dataset(C, G // 2, [[5 * c % G] for c in range(C)], Nv=NV, Nt=NT, F=cfgj["v_feature_size"],
                  lens=torch.randint(1, NT + 1, (C,), generator=g).tolist())
    ds.mask = (torch.arange(NV) < torch.randint(1, NV + 1, (G, 1), generator=g)).long()
    ds.feat = torch.relu(ds.feat) * ds.mask.unsqueeze(-1)
    ds.cap = ds.cap % cfgj["vocab_size"]
    return ds, torch.tensor([5 * c % G for c in range(C)])


def ranks_apart(RT, a, b, target):
    """Captions (caption-to-image) and images (image-to-text) whose rank differs between the score matrices a and b, leaving out
    those whose target score sits within 2 max|a - b| of another score in its row or column (the near ties of
    test_retrieval_packed_gpu.py)."""
    d = (a - b).abs().max().item()
    t = target.cpu()

    def near(v, ts):
        gap = (v.unsqueeze(0) - v[ts].unsqueeze(1)).abs()
        gap[torch.arange(len(ts)), ts] = float("inf")
        return bool(gap.min() <= 2 * d)
    ra, rb = RT.RetrievalEvaluator.rank(a, target, k=1)[0].cpu(), RT.RetrievalEvaluator.rank(b, target, k=1)[0].cpu()
    t2i = [c for c in range(a.shape[0]) if ra[c] != rb[c] and not near(a[c].cpu(), t[c:c + 1])]
    ia, ib = RT.RetrievalEvaluator.rank_captions(a, target, k=1)[0].cpu(), RT.RetrievalEvaluator.rank_captions(b, target, k=1)[0].cpu()
    i2t = [g for g in range(a.shape[1]) if ia[g] != ib[g] and not near(a[:, g].cpu(), (t == g).nonzero().view(-1))]
    return t2i, i2t


def main():
    from vilbert_b200 import retrieval as RT
    out_path, backend = sys.argv[1], sys.argv[2]
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", local if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    if backend == "nccl":
        dist.init_process_group("nccl", device_id=dev, timeout=timedelta(minutes=5))
    else:
        dist.init_process_group("gloo", timeout=timedelta(minutes=5))
    group = dist.group.WORLD

    scored, rows = [], []
    score, score_rows = RT.RetrievalEvaluator.score, RT.RetrievalEvaluator._score_rows
    RT.RetrievalEvaluator.score = lambda self, *a, **kw: scored.append(score(self, *a, **kw)) or scored[-1]
    RT.RetrievalEvaluator._score_rows = lambda self, caps, *a: rows.append(int(caps.shape[0])) or score_rows(self, caps, *a)

    golden = os.path.join(ROOT, "tests", "golden")
    res = {}
    for zero_shot in (False, True):
        cfgj = _cfgj(golden, False)
        model = _model(cfgj, zero_shot)
        task_id = None if zero_shot else "TASK8"
        for det in (True, False):
            torch.use_deterministic_algorithms(det)
            for pack in (False, True):
                for C in (7, 1):
                    name = f"{'zeroshot' if zero_shot else 'finetuned'}_{'det' if det else 'default'}_" \
                           f"{'packed' if pack else 'padded'}_C{C}"
                    ds, target = dataset(cfgj, C, seed=C)
                    scored.clear(); rows.clear()
                    model.engine.release_plans()           # so that "packed" below tells this case's plans
                    single = RT.evaluate_retrieval_both(model, ds, task_id=task_id, chunk=CHUNK, k=K, pack=pack)
                    sharded = RT.evaluate_retrieval_both(model, ds, task_id=task_id, chunk=CHUNK, k=K, pack=pack, group=group)
                    a, b = scored
                    r = dict(rows=list(rows), shape=list(b.shape), packed=any(p.packed for p in model.engine.plans.values()),
                             fallbacks=dict(model.engine.pack_fallbacks), scores_equal=bool(torch.equal(a, b)),
                             rel=(a - b).abs().max().item() / a.abs().max().item(), out_equal=single == sharded,
                             scores_checksum=RT.checksum(b), out=json.dumps(sharded, default=float))
                    r["t2i_apart"], r["i2t_apart"] = ranks_apart(RT, a, b, target.to(a.device))
                    res[name] = r
        # a weight one ulp off on rank 1: both ranks refuse before scoring
        torch.use_deterministic_algorithms(True)
        ds, _ = dataset(cfgj, 7, seed=7)
        flat = model.engine.ps.flat
        saved = flat[3].clone()
        if rank == 1:
            flat[3] = torch.nextafter(saved, torch.tensor(float("inf"), device=saved.device))
        try:
            RT.evaluate_retrieval_both(model, ds, task_id=task_id, chunk=CHUNK, k=K, group=group)
            res[f"perturbed_{zero_shot}"] = "no error"
        except ValueError as ex:
            res[f"perturbed_{zero_shot}"] = str(ex)
        flat[3] = saved
        torch.use_deterministic_algorithms(False)
        del model
    gathered = [None] * world
    dist.all_gather_object(gathered, res)
    if rank == 0:
        json.dump(gathered, open(out_path, "w"))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
