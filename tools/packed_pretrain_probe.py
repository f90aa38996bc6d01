"""Padded vs packed pre-training steps (engine.pack_padding with BertForMultiModalPreTraining(fused_objective=True)):

  padded       pack_padding off: every GEMM, LayerNorm and attention runs on the padded rows
  packed_dev   pack_padding on, masks and labels on the device (what train_concap.py passes): one vb_pack_summary launch and one
               device-to-host read per forward decide the capacities
  packed_host  pack_padding on, masks and labels on the host (pinned): decided on the host, no device read

    python tools/packed_pretrain_probe.py [--steps K] [--windows R] [--text-lengths 6,24] [--regions 10,36] [--out DIR]

Step: forward, (masked_loss_t + masked_loss_v + next_sentence_loss).backward(), one FusedAdamW step, zero_grad. Model:
bert_base_6layer_6conect with random weights, train mode (every dropout active), at the per-GPU shape of train_concap.py
(B=64, 36 + 1 regions, 36 tokens), for visual_target 0 and 2 (num_negative 255). Batches are synthetic: caption lengths
U{a..b} tokens (--text-lengths a,b) and 1 + U{c..d} regions (--regions c,d; the global region plus the adaptive boxes), 15 % of
the valid tokens and regions labelled, four seeded batches cycled; and one batch with every token and region valid, the worst
case for packing. Per arm, R windows of K back-to-back steps (no synchronisation between the steps of a window, so the device
arm's read stalls the host as it would in a training loop) alternated arm by arm; the step time of a window is its CUDA-event
time over K. Reports the median and range over the windows, plan builds, fallbacks and peak memory, with the card name and
power limit read in the same run. Prints JSON lines, also written to DIR/packed_pretrain_probe.json. Needs a GPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, NV, NT = 64, 37, 36
ARMS = ("padded", "packed_dev", "packed_host")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def batch(cfgj, vt, seed, text, regions, all_valid=False):
    """(device args, host masks and labels) of one synthetic batch."""
    import torch
    from oracle import vilbert_oracle as O
    cfg = O.make_config(cfgj)
    inp = O.synth_inputs(cfg, B, NV, NT, seed=seed, device="cuda")
    g = torch.Generator().manual_seed(seed)
    if all_valid:
        lt, lv = torch.full((B,), NT), torch.full((B,), NV)
    else:
        lt = torch.randint(text[0], text[1] + 1, (B,), generator=g)
        lv = 1 + torch.randint(regions[0], regions[1] + 1, (B,), generator=g)
    mt = (torch.arange(NT) < lt.unsqueeze(1)).long()
    mv = (torch.arange(NV) < lv.unsqueeze(1)).long()
    lm = torch.full((B, NT), -1, dtype=torch.long)
    sel = (torch.rand(B, NT, generator=g) < 0.15) & mt.bool()
    lm[sel] = torch.randint(0, cfg["vocab_size"], (int(sel.sum()),), generator=g)
    il = torch.full((B, NV - 1), -1, dtype=torch.long)
    il[(torch.rand(B, NV - 1, generator=g) < 0.15) & mv[:, 1:].bool()] = 1
    feats = inp["input_imgs"] * mv.cuda().unsqueeze(-1)
    it = torch.softmax(torch.randn(B, NV - 1, cfg["v_target_size"], generator=g), -1).cuda() if vt == 0 else feats[:, 1:].clone()
    ns = torch.randint(0, 2, (B,), generator=g).cuda()
    host = [t.pin_memory() for t in (mt, mv, lm, il)]
    dev = [t.cuda() for t in (mt, mv, lm, il)]
    head = [inp["input_txt"], feats, inp["image_loc"], inp["token_type_ids"]]
    return dict(dev=head + dev[:2] + dev[2:] + [it, ns], host=head + host[:2] + host[2:] + [it, ns],
                valid_t=int(lt.sum()), valid_v=int(lv.sum()))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=10, help="steps per timed window")
    ap.add_argument("--windows", type=int, default=5, help="timed windows per arm (after one warm-up window)")
    ap.add_argument("--text-lengths", default="6,24", help="caption lengths U{a..b} tokens")
    ap.add_argument("--regions", default="10,36", help="adaptive boxes U{c..d}, plus the global region")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles"))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("packed_pretrain_probe: needs a GPU (there is nothing to time on the CPU)")
    import vilbert_b200
    from oracle import vilbert_oracle as O
    from vilbert_b200.optim import FusedAdamW
    text = tuple(int(x) for x in a.text_lengths.split(","))
    regions = tuple(int(x) for x in a.regions.split(","))
    base = json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")))
    head = {"what": "one pre-training step (fwd + (lt + lv + ln).backward() + FusedAdamW), bert_base_6layer_6conect, train mode",
            "shape": {"B": B, "Nv": NV, "Nt": NT}, "text_lengths": f"U{{{text[0]}..{text[1]}}} tokens",
            "regions": f"1 + U{{{regions[0]}..{regions[1]}}}", "card (name, power limit, sm clock, max sm clock)": card(),
            "steps_per_window": a.steps, "windows": a.windows}
    print(json.dumps(head), flush=True)
    rows = [head]
    for vt in (0, 2):
        cfgj = dict(base, visual_target=vt)
        if vt == 2:
            cfgj.update(num_negative=255, v_target_size=cfgj["v_feature_size"])
        model = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(cfgj), fused_objective=True)
        model.load_state_dict(O.synth_params(O.make_config(cfgj), seed=0, device="cuda", with_task_heads=False), strict=False)
        model.train()
        eng = model.engine
        opt = FusedAdamW(list(model.parameters()), lr=1e-5, correct_bias=False, model=model)
        for name, batches in (("ragged", [batch(cfgj, vt, s, text, regions) for s in range(4)]),
                              ("all_valid", [batch(cfgj, vt, 100, text, regions, all_valid=True)])):
            arms = ARMS if name == "ragged" else ("padded", "packed_host")

            def step(arm, i):
                eng.pack_padding = arm != "padded"
                b = batches[i % len(batches)]
                lt, lv, ln = model(*(b["host"] if arm == "packed_host" else b["dev"]))
                (lt + lv + ln).sum().backward()
                opt.step()
                model.zero_grad()

            times = {arm: [] for arm in arms}
            peak, builds, fallbacks = {}, {}, {}
            for w in range(a.windows + 1):          # window 0 warms every arm up (plan builds, graph capture)
                for arm in arms:
                    eng.plan_builds.clear(); eng.pack_fallbacks.clear()
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for i in range(a.steps):
                        step(arm, i)
                    e1.record()
                    torch.cuda.synchronize()
                    if w:
                        times[arm].append(e0.elapsed_time(e1) / a.steps)
                        peak[arm] = max(peak.get(arm, 0), torch.cuda.max_memory_allocated())
                        builds[arm] = builds.get(arm, 0) + sum(eng.plan_builds.values())
                        fallbacks[arm] = dict(fallbacks.get(arm, {}), **eng.pack_fallbacks)
            row = {"visual_target": vt, "batches": name, "valid_rows_t": [b["valid_t"] for b in batches],
                   "valid_rows_v": [b["valid_v"] for b in batches], "padded_rows": [B * NT, B * NV]}
            for arm in arms:
                t = sorted(times[arm])
                row[arm] = {"ms_median": statistics.median(t), "ms_min": t[0], "ms_max": t[-1], "ms_windows": times[arm],
                            "plan_builds_after_warmup": builds[arm], "fallbacks": fallbacks[arm], "max_memory_allocated_gb": peak[arm] / 2**30}
            for arm in arms[1:]:
                row[f"speedup_{arm}"] = row["padded"]["ms_median"] / row[arm]["ms_median"]
            print(json.dumps(row), flush=True)
            rows.append(row)
        del model, opt
        torch.cuda.empty_cache()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "packed_pretrain_probe.json"), "w") as f:
        json.dump(rows, f)


if __name__ == "__main__":
    main()
