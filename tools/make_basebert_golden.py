"""Writes tests/golden/tiny_basebert.{json,pt} from the UNMODIFIED reference vilbert/basebert.py (BaseBertForVLTasks, the
single-stream baseline), after checking that oracle/basebert_oracle.py reproduces it (fp32, 1e-5 relative).

Recorded: the reference's state_dict key list and shapes; eval-mode outputs and every parameter gradient (up to 512 elements in
full, larger tensors as 128 seeded samples with their norms, sum and row-0 magnitude) of the seeded scalar
objective sum_o <out_o, R_o>; the same in train mode with every nn.Dropout replaced by the stateless site mask of
oracle.vilbert_oracle.DropMasks (the 0.5 one of SimpleClassifier and both calls of BaseBertForVLTasks.dropout included).
Parameters, inputs and R come from seeds (oracle.basebert_oracle.synth_*); ragged text and image masks.

Usage: python tools/make_basebert_golden.py   (needs the reference checkout; see oracle/basebert_ref_loader.py)
"""
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import basebert_oracle as BO  # noqa: E402
from oracle import basebert_ref_loader as ref_loader  # noqa: E402
from oracle.vilbert_oracle import DropMasks, make_config  # noqa: E402

TINY = dict(vocab_size=120, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=128, max_position_embeddings=40,
            type_vocab_size=2, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
B, NT, NV, LABELS, STEP = 3, 9, 11, 7, 5
SEEDS = dict(params=0, inputs=1234, probe=7)


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


class SiteDropout(nn.Module):
    """nn.Dropout replaced by the engine's stateless mask of one site. `sites` names the site of each call in order (the reference
    calls BaseBertForVLTasks.dropout twice); `stream` = (Nt, N, slice) draws the mask over the whole [B, N, H] stream and slices."""

    def __init__(self, drop, sites, p, stream=None):
        super().__init__()
        self.drop, self.sites, self.p, self.stream, self.calls = drop, sites, p, stream, 0

    def forward(self, x):
        site = self.sites[min(self.calls, len(self.sites) - 1)]
        self.calls += 1
        if self.stream is None:
            m = self.drop.mask(site, self.p, tuple(x.shape), x.device)
            return x if m is None else x * m
        nt, n = self.stream
        full = self.drop.mask(site, self.p, (x.shape[0], n, x.shape[2]), x.device)
        m = full[:, nt:] if site == "dropout.seq_v" else full[:, :nt]
        return x * m


def run_reference(model, inp, R):
    model.zero_grad()
    outs = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                 inp["image_attention_mask"])
    outs = dict(zip(BO.OUT_NAMES, outs))
    obj = sum((outs[k] * R[k]).sum() for k in BO.OUT_NAMES)
    obj.backward()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters()}
    return {k: v.detach().clone() for k, v in outs.items()}, grads, float(obj)


def run_oracle(P, cfg, inp, R, drop):
    Pl = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    outs = BO.base_bert_for_vl_tasks(Pl, cfg, drop=drop, **inp)
    obj = sum((outs[k] * R[k]).sum() for k in BO.OUT_NAMES)
    obj.backward()
    return {k: v.detach() for k, v in outs.items()}, {k: v.grad for k, v in Pl.items()}


def main():
    base = ref_loader.load()
    cfg = make_config(TINY)
    torch.manual_seed(0)
    model = base.BaseBertForVLTasks(ref_loader.BertConfig(**cfg), num_labels=LABELS)
    keys = [[k, list(v.shape)] for k, v in model.state_dict().items()]
    P = BO.synth_params(cfg, LABELS, SEEDS["params"])
    sd = dict(P)
    sd["cls.predictions.decoder.weight"] = P["bert.embeddings.word_embeddings.weight"]
    model.load_state_dict(sd, strict=True)
    inp = BO.synth_inputs(cfg, B, NT, NV, SEEDS["inputs"])
    R = BO.probe_weights(B, NT, NV, LABELS, cfg["vocab_size"], SEEDS["probe"])
    record = {}
    for mode in ("eval", "train"):
        if mode == "eval":
            model.eval()
            drop = None
        else:
            model.train()
            drop = DropMasks(STEP, head_p=0.1)
            for name, mod in list(model.named_modules()):
                for cn, ch in list(mod.named_children()):
                    if isinstance(ch, nn.Dropout):
                        full = f"{name}.{cn}" if name else cn
                        if full == "dropout":
                            rep = SiteDropout(drop, ("dropout.seq_v", "dropout.seq_t"), ch.p, stream=(NT, NT + NV))
                        else:
                            rep = SiteDropout(drop, (full,), ch.p)
                        setattr(mod, cn, rep)
        outs, grads, obj = run_reference(model, inp, R)
        o_outs, o_grads = run_oracle(P, cfg, inp, R, drop)
        for k in BO.OUT_NAMES:
            assert rel(o_outs[k], outs[k]) < 1e-5, (mode, k, rel(o_outs[k], outs[k]))
        for k, g in grads.items():
            assert rel(o_grads[k], g) < 1e-5 or float(g.abs().max()) == 0.0, (mode, k, rel(o_grads[k], g))
        record[mode] = dict(outputs=outs, grads=grads, objective=obj)
        print(f"{mode}: oracle == reference on {len(outs)} outputs and {len(grads)} gradients (objective {obj:.6f})")
    # padding_idx=0 rows take no gradient (the word table's row 0 still gets one through the tied masked-LM decoder)
    for n in ("bert.embeddings.position_embeddings.weight", "bert.embeddings.token_type_embeddings.weight",
              "bert.image_embeddings.token_type_embeddings.weight"):
        assert float(record["eval"]["grads"][n][0].abs().max()) == 0.0, n
    gdir = os.path.join(ROOT, "tests", "golden")
    meta = dict(config=TINY, num_labels=LABELS, B=B, Nt=NT, Nv=NV, train_step=STEP, head_dropout_prob=0.1, seeds=SEEDS,
                state_dict=keys, param_sums={k: float(v.double().sum()) for k, v in P.items()},
                objective={m: record[m]["objective"] for m in record})
    with open(os.path.join(gdir, "tiny_basebert.json"), "w") as f:
        json.dump(meta, f, indent=1)
    # compact: small tensors in full, larger ones as seeded samples plus norms (oracle.basebert_oracle.digest)
    torch.save({m: {kind: {k: BO.digest(v, seed=i) for i, (k, v) in enumerate(record[m][kind].items())} for kind in ("outputs", "grads")}
                for m in record}, os.path.join(gdir, "tiny_basebert.pt"))
    print("wrote tests/golden/tiny_basebert.json / .pt")


if __name__ == "__main__":
    main()
