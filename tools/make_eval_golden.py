"""Writes tests/golden/evaluating_model_reference.json: what the reference's UNMODIFIED EvaluatingModel (vilbert/task_utils.py:626-859)
returns for every evaluation type x process, run on the CPU with a stub model whose ten outputs are seeded tensors.

    python tools/make_eval_golden.py [--reference /path/to/vilbert-multi-task]

task_utils.py imports cleanly once three modules it needs only for data loading are stubbed (pytorch_transformers.tokenization_bert,
vilbert.datasets, vilbert.datasets._image_features_reader) on top of oracle/ref_loader.load(), and torch.Tensor.cuda is the identity.
Each case stores the task_cfg entry, the batch (tensors the step reads, the others as shapes of zeros), the head outputs the stub
returned, label2ans, and the reference's (loss, batch_score, batch_size, results) or the error it raised. tests/test_eval_cpu.py
checks tests/_eval_oracle.py against it; nothing on the GPU reads the reference."""
import argparse
import json
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "evaluating_model_reference.json")
HEADS = ("vil_prediction", "vil_prediction_gqa", "vil_logit", "vil_binary_prediction", "vil_tri_prediction", "vision_prediction",
         "vision_logit", "linguisic_prediction", "linguisic_logit")
NAN = float("nan")


def load_task_utils(reference):
    os.environ["VILBERT_REFERENCE_ROOT"] = reference
    sys.path.insert(0, ROOT)
    from oracle import ref_loader
    ref_loader.load()
    for name, attrs in (("pytorch_transformers", {}), ("pytorch_transformers.tokenization_bert", {"BertTokenizer": object}),
                        ("vilbert.datasets", {"DatasetMapTrain": {}, "DatasetMapEval": {}}),
                        ("vilbert.datasets._image_features_reader", {"ImageFeaturesH5Reader": object})):
        if name not in sys.modules:
            mod = types.ModuleType(name)
            mod.__dict__.update(attrs)
            sys.modules[name] = mod
    torch.Tensor.cuda = lambda self, *a, **k: self
    import vilbert.task_utils as tu
    return tu


def case(name, task_id, typ, loss, process, B, Nv=6, Nt=5, options=3, nround=2, C=4, n_ans=7, nan_row=False,
         qid_per_row=False, seed=0):
    """One evaluation batch in the dataset layout of its process, and the head outputs the stub model returns for it."""
    g = torch.Generator().manual_seed(seed)
    lead = {"retrieval": (B, options), "nlvr": (B,)}.get(process, (B,))
    nv = 2 * Nv if process == "nlvr" else Nv
    qlead = {"expand": (B, options), "retrieval": (B, options), "dialog": (B, nround, options)}.get(process, (B,))
    Bm = {"expand": B * options, "retrieval": B * options, "dialog": B * nround * options, "nlvr": 2 * B}.get(process, B)
    batch = {"features": {"shape": [*lead, nv, 2048]}, "spatials": {"shape": [*lead, nv, 5]}, "image_mask": {"shape": [*lead, nv]},
             "question": {"shape": [*qlead, Nt]}, "input_mask": {"shape": [*qlead, Nt]}, "segment_ids": {"shape": [*qlead, Nt]},
             "co_attention_mask": {"shape": [*qlead, nv, Nt]}}
    heads = {}
    rnd = lambda *s: (torch.randn(*s, generator=g) * 2).round(decimals=1)     # rounded: tied maxima are common
    if typ in ("VL-classifier", "VL-classifier-GQA"):
        lg = rnd(Bm, n_ans)
        lg[0, 2] = lg[0, 5] = lg[0].max() + 1.0                                 # a tie at the maximum: the first index wins
        if nan_row:
            lg[1, 3] = NAN
        heads["vil_prediction" if typ == "VL-classifier" else "vil_prediction_gqa"] = lg
        target = torch.zeros(B, n_ans)
    elif typ == "VL-logit":
        heads["vil_logit"] = rnd(Bm, 1)
        if nan_row:
            heads["vil_logit"][1, 0] = NAN
        n_q = Bm // options
        target = torch.randint(0, options, (B, nround) if process == "dialog" else (n_q,), generator=g)
    elif typ == "V-logit":
        lg = rnd(Bm, Nv, 1)
        lg[0, 1, 0] = lg[0, 4, 0] = lg[0].max() + 1.0
        if nan_row:
            lg[1, 2, 0] = NAN
        heads["vision_logit"] = lg
        target = (torch.rand(B, Nv, 1, generator=g) * 10).round() / 10
    elif typ == "V-logit-mc":
        heads["vision_logit"] = rnd(Bm, Nv, 1)
        heads["vision_logit"][:, Nv - 2:] = -10000.0
        mc = torch.randint(0, Nv - 101, (B, C), generator=g)
        mc[:, C - 1] = Nv - 102                                                 # a padded choice on a masked region
        batch["multiple_choice_ids"] = {"data": mc.tolist(), "dtype": "int64"}
        target = (torch.rand(B, C, 1, generator=g) > 0.5).float()
        target[0] = 0.0                                                         # no positive: the target argmax is the first choice
    else:   # VL-binary / VL-tri
        n_cls = 2 if typ == "VL-binary-classifier" else 3
        rows = Bm // 2 if (typ == "VL-binary-classifier" and Bm % 2 == 0) else Bm
        heads["vil_binary_prediction" if n_cls == 2 else "vil_tri_prediction"] = rnd(rows, n_cls)
        if loss == "CrossEntropyLoss":
            target = torch.randint(0, n_cls, (B,), generator=g)
        else:
            target = torch.softmax(torch.randn(rows if process == "nlvr" else B, n_cls, generator=g) * 2, 1)
    batch["target"] = {"data": target.tolist(), "dtype": "int64" if target.dtype == torch.int64 else "float32"}
    n_qid = Bm // options if (process == "dialog" and qid_per_row) else B
    batch["question_id"] = {"data": (torch.arange(n_qid) * 7 + 1000).tolist(), "dtype": "int64"}
    label2ans = [f"ans{i}" for i in range(n_ans)]
    return {"name": name, "task_id": task_id, "task_cfg": {"type": typ, "loss": loss, "process": process}, "batch": batch,
            "batch_order": ["features", "spatials", "image_mask", "question", "target", "input_mask", "segment_ids"] +
                           (["multiple_choice_ids"] if task_id in ("TASK4", "TASK17") else []) + ["co_attention_mask", "question_id"],
            "model_batch": Bm, "Nv": Nv, "Nt": Nt,
            "heads": {k: {"data": v.tolist(), "shape": list(v.shape)} for k, v in heads.items()}, "label2ans": label2ans}


def tensor(spec):
    if "data" in spec:
        return torch.tensor(spec["data"], dtype=torch.int64 if spec["dtype"] == "int64" else torch.float32)
    return torch.zeros(spec["shape"], dtype=torch.float32)


def build_batch(c):
    """The batch tuple of a case, in the order the reference unpacks it."""
    out = []
    for k in c["batch_order"]:
        t = tensor(c["batch"][k])
        out.append(t.long() if k in ("question", "input_mask", "segment_ids", "image_mask") else t)
    return tuple(out)


def stub_outputs(c):
    """The ten outputs the stub model returns: the stored heads, zeros for the heads the type does not read."""
    Bm, Nv, Nt = c["model_batch"], c["Nv"], c["Nt"]
    zero = {"vil_prediction": (Bm, 7), "vil_prediction_gqa": (Bm, 7), "vil_logit": (Bm, 1), "vil_binary_prediction": (Bm, 2),
            "vil_tri_prediction": (Bm, 3), "vision_prediction": (Bm, Nv, 3), "vision_logit": (Bm, Nv, 1),
            "linguisic_prediction": (Bm, Nt, 3), "linguisic_logit": (Bm, Nt, 1)}
    heads = [torch.tensor(c["heads"][n]["data"], dtype=torch.float32) if n in c["heads"] else torch.zeros(zero[n]) for n in HEADS]
    return tuple(heads) + (None,)


def cases():
    return [
        case("vqa", "TASK1", "VL-classifier", "BCEWithLogitLoss", "normal", 5, nan_row=True),
        case("gqa", "TASK15", "VL-classifier-GQA", "BCEWithLogitLoss", "normal", 4, seed=1),
        case("visdial_dialog_qid_per_row", "TASK3", "VL-logit", "CrossEntropyLoss", "dialog", 2, qid_per_row=True, seed=2),
        case("visdial_dialog_qid_per_image", "TASK3", "VL-logit", "CrossEntropyLoss", "dialog", 2, seed=3),
        case("vcr_expand", "TASK5", "VL-logit", "CrossEntropyLoss", "expand", 3, options=4, seed=4),
        case("retrieval", "TASK7", "VL-logit", "CrossEntropyLoss", "retrieval", 2, options=4, seed=5),
        case("retrieval_nan_row", "TASK7", "VL-logit", "CrossEntropyLoss", "retrieval", 3, options=4, nan_row=True, seed=6),
        case("refcoco", "TASK9", "V-logit", "BCEWithLogitLoss", "normal", 4, nan_row=True, seed=7),
        case("visual7w", "TASK4", "V-logit-mc", "BCEWithLogitLoss", "normal", 3, Nv=110, C=5, seed=8),
        case("nlvr2", "TASK12", "VL-binary-classifier", "BCEWithLogitLoss", "nlvr", 3, seed=9),
        case("binary_bce_odd", "TASK12", "VL-binary-classifier", "BCEWithLogitLoss", "normal", 3, seed=10),
        case("nlvr2_b2", "TASK12", "VL-binary-classifier", "BCEWithLogitLoss", "nlvr", 2, seed=11),
        case("snli_ve", "TASK13", "VL-tri-classifier", "BCEWithLogitLoss", "normal", 4, seed=12),
        case("foil_even", "TASK16", "VL-binary-classifier", "CrossEntropyLoss", "normal", 4, seed=13),
        case("foil_odd", "TASK16", "VL-binary-classifier", "CrossEntropyLoss", "normal", 3, seed=14),
    ]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--reference", default=os.environ.get("VILBERT_REFERENCE_ROOT", "/root/reference"))
    ap.add_argument("--out", default=OUT)
    a = ap.parse_args()
    tu = load_task_utils(a.reference)
    out = []
    for c in cases():
        task_cfg = {c["task_id"]: c["task_cfg"]}
        outputs = stub_outputs(c)

        def model(question, *rest):
            assert question.size(0) == c["model_batch"], (question.shape, c["model_batch"])
            return outputs
        loader = {c["task_id"]: types.SimpleNamespace(dataset=types.SimpleNamespace(label2ans=c["label2ans"]))}
        losses = tu.LoadLosses(None, task_cfg, [c["task_id"][4:]])
        results = []
        try:
            loss, score, bs, results, _ = tu.EvaluatingModel(None, task_cfg, None, c["task_id"], build_batch(c), model, loader, losses,
                                                             results, [])
            c["expect"] = {"loss": loss, "score": score, "batch_size": bs, "results": results, "error": None}
        except (ValueError, IndexError) as ex:
            c["expect"] = {"results": results, "error": type(ex).__name__}
        print(f"{c['name']}: {c['expect']['error'] or 'ok'}, {len(results)} results")
        out.append(c)
    with open(a.out, "w") as f:
        json.dump({"source": "vilbert/task_utils.py EvaluatingModel (:626-859), unmodified, CPU, stub model", "cases": out}, f,
                  allow_nan=True)
    print(f"wrote {a.out}")


if __name__ == "__main__":
    main()
