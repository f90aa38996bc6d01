"""Single-stream baseline (BaseBertForVLTasks) without a GPU: the oracle against the fixtures recorded from the unmodified
reference, the baseline ParamStore's names and shapes against the reference's state_dict, and the launch lists of build-only
baseline plans."""
import json
import os

import pytest
import torch

from oracle import basebert_oracle as BO
from oracle.vilbert_oracle import DropMasks, make_config


def rel(a, b):
    return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


def _golden(golden_dir):
    meta = json.load(open(os.path.join(golden_dir, "tiny_basebert.json")))
    gold = torch.load(os.path.join(golden_dir, "tiny_basebert.pt"))
    return meta, gold


@pytest.mark.parametrize("mode", ["eval", "train"])
def test_oracle_matches_reference(golden_dir, mode):
    """Outputs and every parameter gradient of the seeded objective (fp32, 1e-5 relative), eval mode and train mode with the site
    masks in place of every nn.Dropout."""
    meta, gold = _golden(golden_dir)
    cfg = make_config(meta["config"])
    P = BO.synth_params(cfg, meta["num_labels"], meta["seeds"]["params"])
    for k, s in meta["param_sums"].items():
        assert abs(float(P[k].double().sum()) - s) <= 1e-6 * max(1.0, abs(s)), k
    inp = BO.synth_inputs(cfg, meta["B"], meta["Nt"], meta["Nv"], meta["seeds"]["inputs"])
    R = BO.probe_weights(meta["B"], meta["Nt"], meta["Nv"], meta["num_labels"], cfg["vocab_size"], meta["seeds"]["probe"])
    drop = DropMasks(meta["train_step"], head_p=meta["head_dropout_prob"]) if mode == "train" else None
    Pl = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    out = BO.base_bert_for_vl_tasks(Pl, cfg, drop=drop, **inp)
    sum((out[k] * R[k]).sum() for k in BO.OUT_NAMES).backward()
    g = gold[mode]
    for k in BO.OUT_NAMES:
        assert max(BO.digest_errors(out[k], g["outputs"][k])) < 1e-5, k
    assert set(g["grads"]) == set(Pl)
    for k, ref in g["grads"].items():
        if ("full" in ref and float(ref["full"].abs().max()) == 0.0) or ref.get("absmax") == 0.0:
            assert float(Pl[k].grad.abs().max()) == 0.0, k
        else:
            assert max(BO.digest_errors(Pl[k].grad, ref)) < 1e-5, k
    for k in ("bert.embeddings.position_embeddings.weight", "bert.embeddings.token_type_embeddings.weight",
              "bert.image_embeddings.token_type_embeddings.weight"):
        assert BO.row0_absmax(g["grads"][k]) == 0.0     # padding_idx=0: row 0 takes no gradient
        assert float(Pl[k].grad[0].abs().max()) == 0.0


def test_fixture_digests_are_sensitive():
    """A digest rejects a tensor that differs from the recorded one only outside its samples (one wrong row of an embedding-sized
    gradient), through its norms and sum."""
    t = torch.randn(64, 2048, generator=torch.Generator().manual_seed(3))
    d = BO.digest(t)
    assert max(BO.digest_errors(t, d)) == 0.0
    u = t.clone()
    off = torch.ones(u.numel(), dtype=torch.bool)
    off[d["idx"].long()] = False
    row = off.view(64, 2048)[5]
    u[5][row] += 0.01
    samp, l2, sm = BO.digest_errors(u, d)
    assert samp == 0.0 and max(l2, sm) > 1e-5


def _engine(meta, heads="base", precision="fp16"):
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    return Engine(BertConfig.from_dict(meta["config"]), "cpu", heads=heads, _build_only=True, precision=precision,
                  num_labels=meta["num_labels"])


def test_param_store_matches_reference_state_dict(golden_dir):
    meta, _ = _golden(golden_dir)
    ps = _engine(meta).ps
    ref = {k: tuple(s) for k, s in meta["state_dict"]}
    mine = {k: shape for k, (_, shape) in ps.entries.items()}
    mine["cls.predictions.decoder.weight"] = mine["bert.embeddings.word_embeddings.weight"]     # tied: one entry, two names
    assert mine == ref
    assert ps.p("vil_prediction.main.0.weight_g").dim() == 0 and ps.p("vil_prediction.main.3.weight_g").dim() == 0
    # execution order: embeddings, layers, pooler, heads (the backward finishes the flat buffer from its end)
    names = list(ps.entries)
    assert names.index("bert.image_embeddings.LayerNorm.bias") < names.index("bert.encoder.layer.0.attention.self.query.weight")
    assert names.index("bert.encoder.layer.1.output.LayerNorm.bias") < names.index("bert.pooler.dense.weight") < names.index("cls.predictions.bias")


@pytest.mark.parametrize("precision", ["fp16", "fp32", "bf16"])
def test_baseline_plans_launch_the_new_kernels(golden_dir, precision):
    meta, _ = _golden(golden_dir)
    from vilbert_b200.engine import BASE_HEAD_NAMES
    eng = _engine(meta, precision=precision)
    plan = eng.plan(3, 9, 11, grad_outputs=BASE_HEAD_NAMES, train=True)
    fwd = [op[0].__name__ for op in plan.fwd if op[0] is not None]
    bwd = [op[0].__name__ for op in plan.bwd if op[0] is not None]
    for k in ("vb_mask_concat_additive", "vb_concat_embed_ln_fwd", "vb_tanh_fwd", "vb_weight_norm_fwd", "vb_gather_rows16"):
        assert k in fwd, k
    for k in ("vb_concat_embed_ln_bwd", "vb_embed_text_bwd_padded", "vb_tanh_bwd", "vb_weight_norm_bwd", "vb_scatter_rows_f32"):
        assert k in bwd, k
    assert fwd.count("vb_weight_norm_fwd") == 2 and bwd.count("vb_weight_norm_bwd") == 2
    # no two-stream launches: no separate image LayerNorm, text embedding backward without padding rows, ReLU poolers or fusion
    for k in ("vb_mask_to_additive", "vb_fuse_pooled_fwd", "vb_embed_text_bwd", "vb_fuse_pooled_bwd"):
        assert k not in fwd + bwd, k
    assert fwd.count("vb_attention_fwd") == meta["config"]["num_hidden_layers"]
    assert tuple(plan.outputs["vision_logit"].shape) == (3, 11, 1) and tuple(plan.outputs["linguisic_prediction"].shape) == (3, 9, 120)
    assert tuple(plan.outputs["vision_prediction"].shape) == (3, 11, 1601) and tuple(plan.outputs["vil_prediction"].shape) == (3, 7)


def test_frozen_baseline_plan_skips_frozen_work(golden_dir):
    """Embeddings and the first layer frozen: nothing writes their gradient ranges and the embedding backward is not emitted."""
    meta, _ = _golden(golden_dir)
    from vilbert_b200.engine import BASE_HEAD_NAMES
    eng = _engine(meta)
    frozen = {n for n in eng.ps.entries if n.startswith(("bert.embeddings.", "bert.image_embeddings.", "bert.encoder.layer.0."))}
    plan = eng.plan(3, 9, 11, grad_outputs=BASE_HEAD_NAMES, frozen=frozen)
    bwd = [op[0].__name__ for op in plan.bwd if op[0] is not None]
    assert "vb_concat_embed_ln_bwd" not in bwd and "vb_embed_text_bwd_padded" not in bwd
    assert bwd.count("vb_attention_bwd") == meta["config"]["num_hidden_layers"] - 1
    lo = min(eng.ps.entries[n][0] for n in eng.ps.entries if n.startswith("bert.encoder.layer.1."))
    assert all(off >= lo for (off, _n) in plan.grad_touch)


def test_baseline_box_projection_gradient_is_recorded_at_its_kernel(golden_dir):
    """grad_touch names the backward op that writes each gradient range last; for the box projection that is vb_loc_proj_bwd, so
    no data-parallel segment hands the range to the all-reduce before that kernel has run."""
    meta, _ = _golden(golden_dir)
    from vilbert_b200.engine import BASE_HEAD_NAMES
    eng = _engine(meta)
    plan = eng.plan(3, 9, 11, grad_outputs=BASE_HEAD_NAMES, train=True)
    for n in ("weight", "bias"):
        i = plan.grad_touch[eng.ps.span(f"bert.image_embeddings.image_location_embeddings.{n}")]
        assert plan.bwd[i][0].__name__ == "vb_loc_proj_bwd"


def test_baseline_plan_options_are_checked(golden_dir):
    meta, _ = _golden(golden_dir)
    eng = _engine(meta)
    with pytest.raises(ValueError):
        eng.plan(3, 9, 11, loss="vqa", grad_outputs=("vil_prediction",))
    with pytest.raises(ValueError):
        eng.plan(3, 9, 11, outputs=("vil_logit",))


def test_new_symbols_are_exported():
    from vilbert_b200 import _lib as L
    lib = L.lib()
    new = ("vb_concat_embed_ln_fwd", "vb_concat_embed_ln_bwd", "vb_embed_text_bwd_padded", "vb_weight_norm_fwd", "vb_weight_norm_bwd",
           "vb_tanh_fwd", "vb_tanh_bwd", "vb_mask_concat_additive")
    declared = L.exported_symbols()
    for s in new:
        assert s in declared and hasattr(lib, s), s
