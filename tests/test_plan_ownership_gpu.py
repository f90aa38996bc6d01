"""Forward ownership of the shared activation arena: every way a plan runs its forward ops counts as a forward there, so another
plan's saved activations are no longer taken as intact (Plan.holds_forward) once they have been overwritten."""
import json
import os

import pytest
import torch

from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu


def _plans(golden_dir):
    """Two plans of different shapes on one activation arena, with inputs loaded."""
    from _gpu_util import build_engine
    cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    cfg = O.make_config(cfgj)
    eng = build_engine(cfgj, O.synth_params(cfg, seed=0, device="cuda"), "cuda")
    eng.enable_activation_arena(64 << 20)
    plans = []
    for i, (B, Nt, Nv) in enumerate(((4, 9, 11), (6, 24, 33))):
        inp = O.synth_inputs(cfg, B, Nv, Nt, seed=10 + i, device="cuda")
        p = eng.plan(B, Nt, Nv, grad_outputs=("vil_prediction",), vqa_loss=True)
        p.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                      inp["image_attention_mask"])
        p.vqa_target.copy_(O.synth_vqa_target(B, 3129, seed=3 + i, device="cuda"))
        plans.append(p)
    return plans


def test_capture_and_overlapped_step_claim_the_arena(golden_dir):
    a, b = _plans(golden_dir)
    # capture(): its warm-up runs b's forward over a's activations
    a.run_forward()
    fid = a.fwd_id
    assert a.holds_forward(fid)
    b.capture()
    torch.cuda.synchronize()
    assert not a.holds_forward(fid)
    # run_step_overlapped (one GPU: an all-reduce that does nothing); capture_segments first, since its warm-up is a forward too
    b.capture_segments(4)
    a.run_forward()
    fid = a.fwd_id
    assert a.holds_forward(fid)
    b.run_step_overlapped(lambda lo, hi: None, torch.cuda.Stream())
    torch.cuda.synchronize()
    assert not a.holds_forward(fid)
