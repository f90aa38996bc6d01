"""Times data-parallel training steps through the module surface with the two all-reduce schedules of
ddp.DistributedDataParallel, alternating them in the same process:

  delayed     delay_allreduce=True: the backward as one CUDA graph, then one all-reduce of the flat gradient buffer
  overlapped  delay_allreduce=False: the backward in the pieces of Plan.bucket_schedule (one graph each), every bucket all-reduced on
              a communication stream as soon as its piece has run

    python -m torch.distributed.run --nproc-per-node N tools/ddp_module_probe.py [--windows 5] [--steps 10] [--warmup 3] [--out DIR]
    python tools/ddp_module_probe.py ...                                         # N = 1

Step: forward, loss.backward(), FusedAdamW.step() (the optimizer zeroes the gradients), on graphs after the warm-up. Workloads, per
GPU, bert_base_6layer_6conect in train mode with random weights and synthetic batches already on the GPU: "vqa", ForwardModelsTrain
on a VQA batch at config 2's shape (B=64, 100 regions, 36 tokens); "pretraining", BertForMultiModalPreTraining(fused_objective=True)
at config 3's shape (B=64, 36 + 1 regions, 36 tokens). Per arm: `windows` windows of `steps` steps, the arms alternating window by
window; the median ms/step over the windows and their range. Rank 0 then times on its GPU alone: the same steps without a wrapper
(t1, and the weak-scaling efficiency t1 / t_N of each arm), and the cost of the cuts alone (a reducer that exchanges nothing, the
backward in pieces against the whole-backward graph). With N = 1 the data-parallel rows are "not measured": a world of one takes the
delayed path. The card name, GPU count, power limit and max SM clock are read in the same run. Prints one JSON line (rank 0), also
written to DIR/ddp_module_probe.json. Needs a GPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SHAPES = {"vqa": (64, 100, 36), "pretraining": (64, 37, 36)}      # (B, regions, tokens) per GPU


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    lines = q.stdout.strip().splitlines() if q.returncode == 0 else []
    return {"gpus": len(lines), "card": lines[0] if lines else "unknown"}


def workload(name, dev):
    """-> (model, step_loss()): a train-mode model and the call that runs one forward and returns the loss to backpropagate."""
    import torch
    import vilbert_b200
    from oracle import vilbert_oracle as O
    cfgj = json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")))
    B, Nv, Nt = SHAPES[name]
    if name == "vqa":
        import _task_oracle as T
        from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
        cfgj = dict(cfgj, task_specific_tokens=True)
        model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj), device=dev)
        batch = tuple(x.to(dev) for x in T.make_batch(cfgj, "TASK1", B, Nv, Nt, seed=1))
        losses = LoadLosses(None, T.TASK_CFG, ["1"])

        def step_loss():
            return ForwardModelsTrain(None, T.TASK_CFG, dev, "TASK1", {"TASK1": 0}, {}, {"TASK1": [batch]}, model, losses)[0]
    else:
        model = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(cfgj), device=dev, fused_objective=True)
        cfg = O.make_config(cfgj)
        inp = O.synth_inputs(cfg, B, Nv, Nt, seed=1, device=dev)
        g = torch.Generator().manual_seed(1)
        lm = torch.full((B, Nt), -1, dtype=torch.long)
        sel = torch.rand(B, Nt, generator=g) < 0.15
        lm[sel] = torch.randint(0, cfg["vocab_size"], (int(sel.sum()),), generator=g)
        il = torch.full((B, Nv - 1), -1, dtype=torch.long)
        il[torch.rand(B, Nv - 1, generator=g) < 0.15] = 1
        it = torch.softmax(torch.randn(B, Nv - 1, cfg["v_target_size"], generator=g), -1)
        ns = torch.randint(0, 2, (B,), generator=g)
        args = [inp[k] for k in ("input_txt", "input_imgs", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")]
        args += [x.to(dev) for x in (lm, il, it, ns)]

        def step_loss():
            return sum(model(*args)).sum()
    model.train()
    return model, step_loss


def timed_arms(arms, windows, steps, warmup):
    """{arm: (set_up(), step())}: warm-up steps per arm, then `windows` windows of `steps` steps with the arms alternating; -> {arm:
    [ms/step of each window]} (CUDA events around each window, which ends in a synchronise)."""
    import torch
    for set_up, step in arms.values():
        set_up()
        for _ in range(warmup):
            step()
    torch.cuda.synchronize()
    out = {k: [] for k in arms}
    for _ in range(windows):
        for k, (set_up, step) in arms.items():
            set_up()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            out[k].append(e0.elapsed_time(e1) / steps)
    return out


def summary(ms):
    return {"median_ms": round(statistics.median(ms), 3), "range_ms": [round(min(ms), 3), round(max(ms), 3)]}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)   # the module surface captures its CUDA graphs on the 3rd run of a plan
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles"))
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    if not torch.cuda.is_available():
        raise SystemExit("ddp_module_probe: needs a GPU (there is nothing to time on the CPU)")
    from vilbert_b200.ddp import DistributedDataParallel, FlatGradAllReducer
    from vilbert_b200.optim import FusedAdamW
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)

    class Silent(FlatGradAllReducer):
        """A reducer of a world of two that exchanges nothing: the backward is cut as for a real one."""
        def __init__(self, flat_grad):
            super().__init__(flat_grad)
            self.world = 2

        def allreduce(self):
            pass

        def allreduce_range(self, lo, hi, async_op=True):
            return None

    res = dict(card(), world=world, windows=a.windows, steps=a.steps, warmup=a.warmup, shapes=SHAPES, workloads={})
    for name in SHAPES:
        model, step_loss = workload(name, dev)
        opt = FusedAdamW(list(model.parameters()), lr=1e-6, model=model)

        def step():
            step_loss().backward()
            opt.step()

        def mode(reducer, overlap):
            def set_up():
                model._ddp_reducer, model._ddp_overlap = reducer, overlap
                model._ddp_set_ranges = None if reducer is None else reducer.set_ranges
                if reducer is not None:
                    reducer.set_ranges(model._trainable_ranges())
            return set_up
        row = {}
        if world > 1:
            red = DistributedDataParallel(model, delay_allreduce=True).reducer
            t = timed_arms({"delayed": (mode(red, False), step), "overlapped": (mode(red, True), step)}, a.windows, a.steps, a.warmup)
            row["delayed"], row["overlapped"] = summary(t["delayed"]), summary(t["overlapped"])
            n_pieces = len(model._last_plan.bucket_schedule(red.table))
            row["buckets"], row["pieces"] = len(red.table), n_pieces
            dist.barrier()
        else:
            row["delayed"] = row["overlapped"] = "not measured (one GPU)"
        if rank == 0:
            t = timed_arms({"one_gpu": (mode(None, False), step)}, a.windows, a.steps, a.warmup)
            row["one_gpu"] = summary(t["one_gpu"])
            if world > 1:
                for arm in ("delayed", "overlapped"):
                    row[f"weak_scaling_{arm}"] = round(row["one_gpu"]["median_ms"] / row[arm]["median_ms"], 3)
            silent = Silent(model.engine.ps.grad)
            t = timed_arms({"whole_backward": (mode(silent, False), step), "pieces": (mode(silent, True), step)}, a.windows, a.steps, a.warmup)
            row["cuts_no_exchange"] = {k: summary(v) for k, v in t.items()}
            row["cuts_no_exchange"]["pieces_n"] = len(model._last_plan.bucket_schedule(silent.table))
            res["workloads"][name] = row
        if world > 1:
            dist.barrier()
        del model, opt, step_loss
        torch.cuda.empty_cache()
    if world > 1:
        dist.destroy_process_group()
    if rank == 0:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ddp_module_probe.json"), "w") as f:
            json.dump(res, f)
        print(json.dumps(res))


if __name__ == "__main__":
    main()
