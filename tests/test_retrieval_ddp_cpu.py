"""Retrieval evaluation across ranks without a GPU: the caption shards, the padded row gather and the agreement check over two gloo
processes, score(group=...) end to end through a stand-in for the per-rank scoring loop, and the group=None path making no
torch.distributed call at all."""
import json
import os
import sys
import time

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G, NV, NT = 12, 3, 5


def test_shard_bounds_cover_every_caption_once():
    from vilbert_b200.retrieval import shard_bounds
    for C in range(0, 40):
        for W in range(1, 10):
            b = shard_bounds(C, W)
            assert len(b) == W and b[0][0] == 0 and b[-1][1] == C
            assert all(lo <= hi for lo, hi in b) and all(a[1] == c[0] for a, c in zip(b, b[1:]))     # contiguous, in order
            sizes = [hi - lo for lo, hi in b]
            assert max(sizes) - min(sizes) <= 1
            assert sorted(i for lo, hi in b for i in range(lo, hi)) == list(range(C))
            if C < W:
                assert sizes.count(0) == W - C


def test_checksum_is_the_int32_bit_pattern_sum():
    from vilbert_b200.retrieval import checksum
    x = torch.randn(37, 5)
    assert checksum(x) == int(x.numpy().view(np.int32).astype(np.int64).sum())
    assert checksum(x) == checksum(x.clone()) and checksum(x[:, 1:]) == checksum(x[:, 1:].contiguous())
    y = x.clone()
    y[3, 2] = float(np.nextafter(np.float32(y[3, 2]), np.float32(np.inf)))    # one ulp: the bit pattern moves by one
    assert abs(checksum(y) - checksum(x)) == 1
    assert checksum(torch.tensor([1, 2], dtype=torch.int64)) == 3
    assert checksum(torch.ones(3, dtype=torch.bool)) == 0x010101                 # bytes zero-padded to 4
    assert checksum(torch.arange(20, dtype=torch.uint8)[1:17]) == checksum(torch.arange(1, 17, dtype=torch.uint8))


class _Model:
    """What RetrievalEvaluator reads of a model outside its per-rank scoring loop: an engine built without a GPU."""
    _heads = "vl"
    training = False

    def __init__(self):
        from vilbert_b200.config import BertConfig
        from vilbert_b200.engine import Engine
        cfg = dict(json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_b4.json")))["config"], task_specific_tokens=True)
        self.config = BertConfig.from_dict(cfg)
        self.engine = Engine(self.config, "cpu", _build_only=True)

    def eval(self):
        return self


def _expected(captions):
    """A score that depends on the caption and the image only."""
    return (captions.sum(1, keepdim=True) * 100 + torch.arange(G)).float()


def _fake_rows(self, captions, input_mask, segment_ids, task_id, has_task):
    """Stands in for RetrievalEvaluator._score_rows, recording the first token (the caption's index) of the captions it scored."""
    self.scored = getattr(self, "scored", []) + [captions[:, 0].tolist()]
    return _expected(captions)


def _inputs(C, seed=0):
    g = torch.Generator().manual_seed(seed)
    feats, locs = torch.rand(G, NV, 8, generator=g), torch.rand(G, NV, 5, generator=g)
    imask = torch.ones(G, NV, dtype=torch.long)
    caps = torch.randint(0, 1000, (C, NT), generator=g)
    caps[:, 0] = torch.arange(C)
    return feats, locs, imask, caps, torch.ones_like(caps), torch.zeros_like(caps)


def _evaluator(model, feats, locs, imask):
    from vilbert_b200.retrieval import RetrievalEvaluator
    return RetrievalEvaluator(model, feats, locs, imask, chunk=5)


def test_without_a_group_no_distributed_call_is_made(monkeypatch):
    from vilbert_b200 import retrieval as RT
    from test_retrieval_cpu import _FakeDataset, stable_desc

    def refuse(*a, **kw):
        raise AssertionError("a torch.distributed call on the group=None path")
    for name in ("all_gather_into_tensor", "all_gather", "all_gather_object", "all_reduce", "broadcast", "barrier",
                 "get_world_size", "get_rank", "get_backend", "is_initialized", "new_group"):
        monkeypatch.setattr(dist, name, refuse)
    monkeypatch.setattr(RT.RetrievalEvaluator, "_score_rows", _fake_rows)
    model = _Model()
    feats, locs, imask, caps, amask, seg = _inputs(7)
    ev = _evaluator(model, feats, locs, imask)
    scores = ev.score(caps, amask, seg, task_id=8)
    assert ev.scored == [list(range(7))] and torch.equal(scores, _expected(caps))

    # the public evaluation, with both rankings restated on the host
    def rank(scores, target, k=20):
        order = torch.from_numpy(np.stack([stable_desc(r) for r in scores.numpy()]))
        return (order == torch.as_tensor(target).view(-1, 1)).int().argmax(1).int(), order[:, :k].int()

    def rank_captions(scores, target, k=20):
        order = torch.from_numpy(np.stack([stable_desc(r) for r in scores.t().numpy()]))
        hit = torch.as_tensor(target)[order] == torch.arange(scores.shape[1]).view(-1, 1)
        return torch.where(hit.any(1), hit.int().argmax(1), -1).int(), order[:, :k].int()
    monkeypatch.setattr(RT.RetrievalEvaluator, "rank", staticmethod(rank))
    monkeypatch.setattr(RT.RetrievalEvaluator, "rank_captions", staticmethod(rank_captions))
    ds = _FakeDataset(6, 3, [[c] for c in range(6)], Nv=NV, Nt=NT, F=8)
    out = RT.evaluate_retrieval_both(model, ds, task_id="TASK8", chunk=5, k=4, group=None)
    assert set(out) == {"t2i", "i2t", "rsum", "images_without_caption"} and len(out["t2i"][5]) == 6
    assert RT.evaluate_retrieval(model, ds, task_id="TASK8", chunk=5, k=4) == out["t2i"]


# ------------------------------------------------------------------------------------------ two gloo ranks
def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    sys.path.insert(0, ROOT)
    from datetime import timedelta
    from vilbert_b200 import retrieval as RT
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timedelta(seconds=120))
    res = {}
    # the padded gather: uneven blocks (7 rows over 2 ranks), an empty block (1 row), and equal blocks
    for C in (7, 1, 8):
        full = torch.arange(C * G, dtype=torch.float32).view(C, G) - 5.5
        lo, hi = RT.shard_bounds(C, world)[rank]
        res[f"gather_{C}"] = bool(torch.equal(RT.gather_rows(full[lo:hi].clone(), C, dist.group.WORLD), full))
    # score(group=...) through the stand-in scoring loop: each rank scores its block only, every rank returns the whole matrix
    RT.RetrievalEvaluator._score_rows = _fake_rows
    model = _Model()
    for C in (7, 1):
        feats, locs, imask, caps, amask, seg = _inputs(C)
        ev = _evaluator(model, feats, locs, imask)
        got = ev.score(caps, amask, seg, task_id=8, group=dist.group.WORLD)
        res[f"score_{C}"] = (bool(torch.equal(got, _expected(caps))), getattr(ev, "scored", []))
    # the agreement check: rank 1 with other captions, then with one parameter one ulp off; both ranks must raise
    feats, locs, imask, caps, amask, seg = _inputs(7)
    ev = _evaluator(model, feats, locs, imask)
    for case in ("captions", "parameters", "task"):
        c = caps.clone()
        flat = model.engine.ps.flat
        saved = flat[5].clone()
        task = 8
        if rank == 1 and case == "captions":
            c[3, 2] += 1
        if rank == 1 and case == "parameters":
            flat[5] = float(np.nextafter(np.float32(saved), np.float32(np.inf)))
        if rank == 1 and case == "task":
            task = 7
        try:
            ev.score(c, amask, seg, task_id=task, group=dist.group.WORLD)
            res[f"agree_{case}"] = "no error"
        except ValueError as ex:
            res[f"agree_{case}"] = str(ex)
        flat[5] = saved
    out[rank] = res
    dist.barrier()
    dist.destroy_process_group()


def test_two_gloo_ranks_gather_score_and_check_agreement():
    world = 2
    port = 33500 + (os.getpid() % 2000)
    mgr = mp.Manager()
    out = mgr.dict()
    ctx = mp.spawn(_worker, args=(world, port, out), nprocs=world, join=False)
    deadline = time.monotonic() + 300
    while not ctx.join(timeout=5):
        if time.monotonic() > deadline:
            for p in ctx.processes:
                p.kill()
            pytest.fail("the gloo ranks did not finish within 300 s")
    for rank in range(world):
        res = out[rank]
        assert res["gather_7"] and res["gather_1"] and res["gather_8"], res
        ok7, scored7 = res["score_7"]
        ok1, scored1 = res["score_1"]
        assert ok7 and ok1
        assert scored7 == [[0, 1, 2]] if rank == 0 else scored7 == [[3, 4, 5, 6]]      # only the rank's own block
        assert scored1 == [] if rank == 0 else scored1 == [[0]]                        # an empty block scores nothing
        assert "caption ids" in res["agree_captions"] and "parameters" not in res["agree_captions"], res
        assert "parameters" in res["agree_parameters"] and "caption ids" not in res["agree_parameters"], res
        assert "task [8, 7]" in res["agree_task"], res
