"""Fused AdamW (csrc/vb_optim.cu, optim.FusedAdamW) vs the oracle restatement of pytorch_transformers 1.0.0 AdamW
(oracle/adamw_oracle.py) with the reference's per-tensor param groups (train_tasks.py:401-426)."""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import adamw_oracle as AO
from oracle import vilbert_oracle as O


def test_oracle_adamw_matches_torch_adamw_where_they_coincide():
    """Independent cross-check of the restatement: with correct_bias=True and weight_decay=0 pytorch_transformers' AdamW and
    torch.optim.Adam differ only in where eps enters (sqrt(v) + eps vs sqrt(v)/sqrt(bc2) + eps): with eps -> 0 they coincide."""
    g = torch.Generator().manual_seed(0)
    p0 = torch.randn(257, generator=g, dtype=torch.float64)
    pa = p0.clone(); m = torch.zeros_like(pa); v = torch.zeros_like(pa)
    pb = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([pb], lr=1e-3, betas=(0.9, 0.999), eps=1e-30)
    for t in range(1, 6):
        grad = torch.randn(257, generator=g, dtype=torch.float64)
        AO.adamw_step(pa, grad, m, v, t, 1e-3, eps=1e-30, correct_bias=True)
        pb.grad = grad.clone(); opt.step()
        assert torch.allclose(pa, pb.data, rtol=1e-9, atol=1e-12)


def test_oracle_adamw_decay_is_applied_after_the_update_on_the_new_weights():
    p = torch.tensor([2.0]); m = torch.zeros(1); v = torch.zeros(1)
    AO.adamw_step(p, torch.tensor([0.5]), m, v, 1, lr=0.1, eps=0.0, weight_decay=0.5, correct_bias=False)
    # m = 0.05, v = 0.00025 -> p = 2 - 0.1 * 0.05 / sqrt(0.00025) = 2 - 0.316228 = 1.683772; then p *= (1 - 0.1 * 0.5)
    assert abs(p.item() - 1.683772 * 0.95) < 1e-5


def test_chunk_table_never_crosses_tensors():
    from vilbert_b200.optim import build_chunks
    st, cn, gr = build_chunks([(0, 100, 0), (104, 70000, 1), (70104, 3, 2)], chunk=32768)
    assert st.tolist() == [0, 104, 104 + 32768, 104 + 65536, 70104]
    assert cn.tolist() == [100, 32768, 32768, 70000 - 65536, 3] and gr.tolist() == [0, 1, 1, 1, 2]
    with pytest.raises(ValueError):
        build_chunks([(2, 10, 0)])


@pytest.mark.gpu
@pytest.mark.parametrize("precision,correct_bias", [("fp16", False), ("fp32", True)])
def test_fused_adamw_matches_oracle_over_steps(golden_dir, precision, correct_bias):
    """Three optimizer steps with the reference's grouping (per-tensor lr / weight decay, a scheduler changing the lr between
    steps): parameters, moments, the zeroed gradient buffer and the 16-bit weight copy (hi + lo in split precision)."""
    import vilbert_b200
    from vilbert_b200.optim import FusedAdamW
    cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    cfg = O.make_config(cfgj)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj), num_labels=1, precision=precision)
    P = O.synth_params(cfg, seed=0, device="cuda")
    model.load_state_dict(P, strict=True)
    groups = AO.reference_param_groups(model.named_parameters(), base_lr=4e-5)
    opt = FusedAdamW(groups, lr=4e-5, correct_bias=correct_bias, model=model)
    assert len(opt.param_groups) == len(list(model.named_parameters()))
    ref = {k: v.detach().clone().double() for k, v in model.named_parameters()}
    mom = {k: (torch.zeros_like(v), torch.zeros_like(v)) for k, v in ref.items()}
    hyper = {k: (g["lr"], g["weight_decay"]) for (k, _), g in zip(model.named_parameters(), groups)}
    gen = torch.Generator(device="cuda").manual_seed(1)
    eng = model.engine
    for t in range(1, 4):
        scale = 1.0 - 0.2 * (t - 1)                      # what WarmupLinearSchedule does: mutate group["lr"]
        for g, (k, _) in zip(opt.param_groups, model.named_parameters()):
            g["lr"] = hyper[k][0] * scale
        eng.ps.grad.copy_(torch.randn(eng.ps.numel, device="cuda", generator=gen) * 1e-2)
        grads = {k: v.grad.detach().clone().double() for k, v in model.named_parameters()}
        opt.step()
        torch.cuda.synchronize()
        for k in ref:
            AO.adamw_step(ref[k], grads[k], mom[k][0], mom[k][1], t, hyper[k][0] * scale, weight_decay=hyper[k][1], correct_bias=correct_bias)
        # every parameter's gradient was zeroed by the same launch (padding elements between tensors are not part of any group)
        assert all(v.grad.abs().max().item() == 0 for _, v in model.named_parameters()) and eng.grad_clean
    named = dict(model.named_parameters())
    for k in ref:
        scale_ = max(ref[k].abs().max().item(), 1e-6)
        assert ((named[k].detach().double() - ref[k]).abs().max() / scale_).item() < 2e-6, k
        assert ((opt.state[named[k]]["exp_avg"].double() - mom[k][0]).abs().max() / max(mom[k][0].abs().max().item(), 1e-12)).item() < 1e-5, k
        # fp32 kernel vs float64 restatement: a few roundings per step (1 - fp32(0.999) in place of fp32(1 - 0.999) is 1.3e-5)
        assert ((opt.state[named[k]]["exp_avg_sq"].double() - mom[k][1]).abs().max() / max(mom[k][1].abs().max().item(), 1e-12)).item() < 2e-6, k
    # the 16-bit operand copy was produced by the same launch
    ps = eng.ps
    assert torch.equal(ps.shadow, ps.flat.to(ps.op_dtype)) and torch.equal(ps.shadow_b, ps.flat.to(torch.bfloat16))
    if precision == "fp32":
        assert torch.equal(ps.shadow_lo, (ps.flat - ps.shadow.float()).to(ps.op_dtype))
    assert eng.shadow_clean and eng.shadow_trusted


@pytest.mark.gpu
def test_training_loop_with_torch_and_fused_optimizers(golden_dir):
    """ADVICE r1: optimizers write parameters through p.data (no version bump) and torch's zero_grad() drops .grad. A plain
    torch optimizer and FusedAdamW must both train: the loss of a fixed batch goes down and the GEMM weights really move."""
    import vilbert_b200
    from vilbert_b200.optim import FusedAdamW
    cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    # train mode (where the stale-weights bug lived) with every dropout probability 0: a deterministic loss curve
    cfgj = dict(cfgj, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, v_hidden_dropout_prob=0.0, v_attention_probs_dropout_prob=0.0)
    cfg = O.make_config(cfgj)
    inp = O.synth_inputs(cfg, 4, 11, 9, seed=1234, device="cuda")
    tgt = O.synth_vqa_target(4, 3129, device="cuda")
    for kind in ("torch", "fused"):
        model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj), num_labels=1, dropout_prob=0.0)
        model.load_state_dict(O.synth_params(cfg, seed=0, device="cuda"), strict=True)
        model.train()
        if kind == "torch":
            opt = torch.optim.SGD(model.parameters(), lr=0.01)
        else:
            opt = FusedAdamW(AO.reference_param_groups(model.named_parameters(), base_lr=2e-3), lr=2e-3, correct_bias=False, model=model)
        w0 = model.state_dict()["bert.encoder.layer.0.intermediate.dense.weight"].clone()
        losses = []
        for it in range(4):
            out = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
            loss = O.vqa_loss(out[0], tgt)
            loss.backward()
            if kind == "torch":
                # p.data-style update, like pytorch_transformers.AdamW / the reference's RAdam (vilbert/optimization.py:98)
                with torch.no_grad():
                    for p in model.parameters():
                        p.data.add_(p.grad, alpha=-0.01)
                opt.zero_grad()          # torch default set_to_none=True: detaches every .grad
                assert next(iter(model.parameters())).grad is None
            else:
                opt.step(); model.zero_grad()
            losses.append(loss.item())
        assert losses[-1] < losses[0] * 0.97 and losses[1] < losses[0], (kind, losses)
        assert (model.state_dict()["bert.encoder.layer.0.intermediate.dense.weight"] - w0).abs().max().item() > 0
        # the forward really used the updated GEMM weights: recomputing with a fresh engine copy gives the same loss
        out = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
        l_now = O.vqa_loss(out[0], tgt).item()
        model.engine.refresh_weights()
        out2 = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
        assert abs(O.vqa_loss(out2[0], tgt).item() - l_now) < 1e-6 * abs(l_now) + 1e-7
