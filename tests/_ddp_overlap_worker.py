"""2-rank worker of tests/test_ddp_overlap_gpu.py (launched with torch.distributed.run, one rank per GPU, NCCL): the module surface
under DistributedDataParallel with delay_allreduce=True and False. The ranks hold different masks: with engine.pack_padding rank 0's
VQA batches pack and rank 1's (a hole in an image mask) run padded, so the two ranks cut their backwards at different places while
issuing the same collectives. Two models from the same parameters, one per mode, run ForwardModelsTrain + clipping FusedAdamW steps
and one fused pre-training step; under torch.use_deterministic_algorithms(True) their gradients and parameters must be bitwise equal
after every step (the messages are the same), and without it equal to the last bits of the split-K atomics. The first step's
gradients are also compared with one GPU on the concatenated batch, and no_sync() on a first micro-batch with the delayed mode's two
exchanges."""
import json
import os
import sys
from datetime import timedelta

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _task_oracle as T                          # noqa: E402
from oracle import vilbert_oracle as O           # noqa: E402

Bl, NV, NT = 4, 100, 36          # per rank: the per-GPU shape of config 2 on the tiny model


def rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def main():
    import vilbert_b200
    from vilbert_b200.ddp import DistributedDataParallel as DDP
    from vilbert_b200.optim import FusedAdamW
    from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
    out_path = sys.argv[1]
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev, timeout=timedelta(minutes=5))
    cfgj = dict(json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_b4.json")))["config"], task_specific_tokens=True,
                max_position_embeddings=300)
    params = O.synth_params(O.make_config(cfgj), seed=3, device=dev)
    losses = LoadLosses(None, T.TASK_CFG, ["1"])

    def global_batch(seed):
        b = list(T.make_batch(cfgj, "TASK1", Bl * world, NV, NT, seed=seed))
        b[2][Bl, 1] = 0              # rank 1's first sample: not a prefix mask, so its batch runs padded
        return b

    def local_batch(seed):
        return tuple(t[rank * Bl:(rank + 1) * Bl] for t in global_batch(seed))

    def model(pack=True):
        m = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
        m.load_state_dict(params, strict=False)
        m.eval()                     # no dropout: one GPU on the concatenated batch computes the same gradient
        m.engine.pack_padding = pack
        return m

    def backward(dp, batch):
        loss, _ = ForwardModelsTrain(None, T.TASK_CFG, dev, "TASK1", {"TASK1": 0}, {}, {"TASK1": [batch]}, dp, losses)
        loss.backward()

    res = {}
    for det in (True, False):
        torch.use_deterministic_algorithms(det)
        tag = "det" if det else "default"
        mA, mB = model(), model()
        dA, dB = DDP(mA, delay_allreduce=True), DDP(mB, delay_allreduce=False)
        lr = 1e-3 if det else 0.0    # outside determinism, keep the parameters: atomics' last bits would drift the two runs apart
        oA = FusedAdamW(list(mA.parameters()), lr=lr, model=mA, max_grad_norm=1.0)
        oB = FusedAdamW(list(mB.parameters()), lr=lr, model=mB, max_grad_norm=1.0)
        grads, params_eq, grad_diff, packed = [], [], [], []
        for s in range(4):
            batch = local_batch(s)
            g = []
            for m, d, o in ((mA, dA, oA), (mB, dB, oB)):
                backward(d, batch)
                g.append(m.engine.ps.grad.clone())
                o.step()
            torch.cuda.synchronize()
            packed.append(mB._last_plan.packed is not None)
            grads.append(g[0])
            grad_diff.append(0.0 if torch.equal(g[0], g[1]) else ((g[0] - g[1]).abs().max() / g[0].abs().max()).item())
            params_eq.append(bool(torch.equal(mA.engine.ps.flat, mB.engine.ps.flat)))
        res[f"{tag}_grad_diff"], res[f"{tag}_params_equal"], res[f"{tag}_packed_rank{rank}"] = grad_diff, params_eq, packed
        flat = mA.engine.ps.flat.clone()
        dist.broadcast(flat, 0)
        res[f"{tag}_ranks_equal"] = bool(torch.equal(flat, mA.engine.ps.flat))
        if rank == 0:                # one GPU, the concatenated batch of step 0, padded
            mC = model(pack=False)
            backward(mC, tuple(global_batch(0)))
            gC, gA = mC.engine.ps.grad, grads[0]
            res[f"{tag}_vs_one_gpu_l2"] = rel(gA, gC)
            worst = 0.0
            for k in mC.engine.ps.entries:
                a, c = mA.engine.ps.g(k), mC.engine.ps.g(k)
                if c.abs().max() > 1e-3 * gC.abs().max():
                    worst = max(worst, rel(a, c))
            res[f"{tag}_vs_one_gpu_worst_tensor_l2"] = worst
            del mC
        dist.barrier()
        # gradient accumulation: no_sync() on micro-batch 1, exchange on micro-batch 2 vs the delayed mode's two exchanges
        mA.zero_grad(); mB.zero_grad()
        backward(dA, local_batch(10)); backward(dA, local_batch(11))
        with dB.no_sync():
            backward(dB, local_batch(10))
        backward(dB, local_batch(11))
        torch.cuda.synchronize()
        res[f"{tag}_no_sync_l2"] = rel(mB.engine.ps.grad, mA.engine.ps.grad)
        del mA, mB, dA, dB, oA, oB
    # one fused pre-training step per mode (deterministic)
    torch.use_deterministic_algorithms(True)
    pj = dict(json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_b4.json")))["config"])
    pcfg = O.make_config(pj)
    pparams = O.synth_params(pcfg, seed=4, device=dev, with_task_heads=False)
    inp = O.synth_inputs(pcfg, Bl * world, 37, NT, seed=9, device=dev)
    g = torch.Generator().manual_seed(9)
    lm = torch.full((Bl * world, NT), -1, dtype=torch.long)
    lm[torch.rand(Bl * world, NT, generator=g) < 0.15] = 5
    lm[:, 1] = 7
    il = torch.full((Bl * world, 36), -1, dtype=torch.long)
    il[:, 0] = 1
    it = torch.softmax(torch.randn(Bl * world, 36, pcfg["v_target_size"], generator=g), -1)
    ns = torch.randint(0, 2, (Bl * world,), generator=g)
    sl = slice(rank * Bl, (rank + 1) * Bl)
    args = [inp[k][sl] for k in ("input_txt", "input_imgs", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")]
    args += [x[sl].to(dev) for x in (lm, il, it, ns)]
    pg = []
    for delay in (True, False):
        m = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(pj), fused_objective=True)
        m.load_state_dict(pparams, strict=False)
        m.eval()
        d = DDP(m, delay_allreduce=delay)
        sum(d(*args)).sum().backward()
        torch.cuda.synchronize()
        pg.append(m.engine.ps.grad.clone())
    res["pretraining_equal"] = bool(torch.equal(pg[0], pg[1]))
    torch.use_deterministic_algorithms(False)
    gathered = [None] * world
    dist.all_gather_object(gathered, res)
    if rank == 0:
        json.dump(gathered, open(out_path, "w"))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
