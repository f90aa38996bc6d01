"""Times one pre-training step (train_concap.py:542-559) through BertForMultiModalPreTraining with the fused objective off and on,
alternating the two arms in the same process:

  module   fused_objective=False: all-logits plan, the three losses formed with torch on cloned head outputs
  fused    fused_objective=True:  the three losses as kernels at the end of the forward, compacted masked-LM head

    python tools/pretrain_step_probe.py [--steps K] [--warmup W] [--out DIR]

Step: forward, (masked_loss_t + masked_loss_v + next_sentence_loss).backward(), one FusedAdamW step, zero_grad. Model:
bert_base_6layer_6conect with random weights, train mode, at the per-GPU shape of bench.py's config 3 (B=64, 36 + 1 regions,
36 tokens, 15 % of the tokens and regions masked), for visual_target 0 and 2 (num_negative 255, negatives drawn on the device).
Batches are synthetic and already on the GPU. Before timing, one seeded step of each arm (same weights, dropout step and negatives,
no optimizer step) gives the three losses and the relative L2 distance of the flat gradients. Per arm: median and spread of the
step time (CUDA events), torch.cuda.max_memory_allocated over the timed steps and the peak above the memory held at the start of
the step. Prints one JSON line, also written to DIR/pretrain_step_probe.json, with the card name, power limit and SM clocks
read in the same run. Needs a GPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, NV, NT = 64, 37, 36


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def batch(cfgj, vt, seed):
    import torch
    from oracle import vilbert_oracle as O
    cfg = O.make_config(cfgj)
    inp = O.synth_inputs(cfg, B, NV, NT, seed=seed, device="cuda")
    g = torch.Generator().manual_seed(seed)
    lm = torch.full((B, NT), -1, dtype=torch.long)
    sel = torch.rand(B, NT, generator=g) < 0.15
    lm[sel] = torch.randint(0, cfg["vocab_size"], (int(sel.sum()),), generator=g)
    il = torch.full((B, NV - 1), -1, dtype=torch.long)
    il[torch.rand(B, NV - 1, generator=g) < 0.15] = 1
    if vt == 0:
        it = torch.softmax(torch.randn(B, NV - 1, cfg["v_target_size"], generator=g), -1).cuda()
    else:
        it = inp["input_imgs"][:, 1:].clone()          # the region features themselves (train_concap.py's image_target)
    ns = torch.randint(0, 2, (B,), generator=g)
    return (inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"],
            lm.cuda(), il.cuda(), it, ns.cuda())


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)   # the module surface captures its CUDA graphs on the 3rd run of a plan
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles"))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("pretrain_step_probe: needs a GPU (there is nothing to time on the CPU)")
    import vilbert_b200
    from oracle import vilbert_oracle as O
    from vilbert_b200.optim import FusedAdamW
    base = json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")))
    res = {"what": "one pre-training step (fwd + (lt + lv + ln).backward() + FusedAdamW), bert_base_6layer_6conect, train mode",
           "shape": {"B": B, "Nv": NV, "Nt": NT}, "card": card(), "steps": a.steps, "warmup": a.warmup, "arms": {}}
    for vt in (0, 2):
        cfgj = dict(base, visual_target=vt)
        if vt == 2:
            cfgj.update(num_negative=255, v_target_size=cfgj["v_feature_size"])
        model = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(cfgj))
        model.load_state_dict(O.synth_params(O.make_config(cfgj), seed=0, device="cuda", with_task_heads=False), strict=False)
        model.train()
        args = batch(cfgj, vt, seed=11)

        # the same seeded step both ways (no optimizer step): losses and gradients
        if vt == 2:
            neg = O.nce_negative_indices(B, NV - 1, 255).cuda()
            model.nce_sampler = lambda b, r, dev: neg.to(dev)
        same = {}
        for fused in (False, True):
            model.fused_objective = fused
            model.engine.set_dropout_step(100)
            model.zero_grad()
            lt, lv, ln = model(*args)
            (lt + lv + ln).sum().backward()
            same[fused] = ([x.item() for x in (lt, lv, ln)], model.engine.ps.grad.clone())
        g0, g1 = same[False][1], same[True][1]
        check = {"losses_module": same[False][0], "losses_fused": same[True][0],
                 "grad_rel_l2": ((g1 - g0).norm() / g0.norm()).item()}
        del same, g0, g1
        model.nce_sampler = None

        opt = FusedAdamW(list(model.parameters()), lr=1e-4, correct_bias=False, model=model)

        def step(fused):
            model.fused_objective = fused
            lt, lv, ln = model(*args)
            (lt + lv + ln).sum().backward()
            opt.step()
            model.zero_grad()

        times, peak, transient = {False: [], True: []}, {False: 0, True: 0}, {False: 0, True: 0}
        for i in range(a.warmup + a.steps):
            for fused in (False, True):
                torch.cuda.synchronize()
                held = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                step(fused)
                e1.record()
                torch.cuda.synchronize()
                if i >= a.warmup:
                    times[fused].append(e0.elapsed_time(e1))
                    peak[fused] = max(peak[fused], torch.cuda.max_memory_allocated())
                    transient[fused] = max(transient[fused], torch.cuda.max_memory_allocated() - held)
        arms = {}
        for fused, name in ((False, "module"), (True, "fused")):
            t = sorted(times[fused])
            arms[name] = {"ms_median": statistics.median(t), "ms_min": t[0], "ms_max": t[-1],
                          "ms_iqr": t[(3 * len(t)) // 4] - t[len(t) // 4], "max_memory_allocated": peak[fused],
                          "step_peak_above_held": transient[fused], "ms": times[fused]}
        res["arms"][f"visual_target_{vt}"] = dict(arms, same_step=check)
        del model, opt
        torch.cuda.empty_cache()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "pretrain_step_probe.json"), "w") as f:
        json.dump(res, f)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
