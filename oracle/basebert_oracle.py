"""ORACLE — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

fp32 restatement (plain torch, device-agnostic, autograd-capable) of the reference's single-stream baseline,
BaseBertForVLTasks (vilbert/basebert.py:893-978) on basebert.BertModel (:654-774), keyed on the reference's state_dict names.
Dropout is the stateless site mask of vilbert_oracle.DropMasks: drop=None is eval mode. Pinned against the unmodified reference
by tools/make_basebert_golden.py, which writes tests/golden/tiny_basebert.{json,pt}.
"""
import torch
import torch.nn.functional as F

from .vilbert_oracle import _drop, gelu, layer_norm, linear, text_layer

OUT_NAMES = ("vil_prediction", "vil_logit", "vil_binary_prediction", "vision_prediction", "vision_logit", "linguisic_prediction",
             "linguisic_logit")


def weight_norm(P, pre):
    """torch.nn.utils.weight_norm(..., dim=None): w = v * (g / ||v||_F)."""
    v, g = P[pre + ".weight_v"], P[pre + ".weight_g"]
    return v * (g / v.norm())


def bert_model(P, cfg, input_txt, input_imgs, image_loc, token_type_ids=None, attention_mask=None, image_attention_mask=None,
               drop=None, all_layers=False):
    """basebert.BertModel.forward (:706-774): text embeddings (:305-321; padding_idx=0 on all three tables), image embeddings
    (:340-359; every region has token type 1), both concatenated, num_hidden_layers BERT layers under the concatenated additive mask,
    tanh pooler on row 0 (:507-519)."""
    if attention_mask is None:
        attention_mask = torch.ones_like(input_txt)
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_txt)
    if image_attention_mask is None:
        image_attention_mask = torch.ones(input_imgs.shape[0], input_imgs.shape[1], device=input_txt.device).type_as(input_txt)
    B, Nt = input_txt.shape
    e = "bert.embeddings"
    pos = torch.arange(Nt, device=input_txt.device).unsqueeze(0).expand(B, Nt)
    t = (F.embedding(input_txt, P[e + ".word_embeddings.weight"], padding_idx=0)
         + F.embedding(pos, P[e + ".position_embeddings.weight"], padding_idx=0)
         + F.embedding(token_type_ids, P[e + ".token_type_embeddings.weight"], padding_idx=0))
    t = _drop(layer_norm(t, P[e + ".LayerNorm.weight"], P[e + ".LayerNorm.bias"]), drop, e + ".dropout", cfg["hidden_dropout_prob"])
    ie = "bert.image_embeddings"
    v = (linear(P, ie + ".image_embeddings", input_imgs) + P[ie + ".token_type_embeddings.weight"][1]
         + linear(P, ie + ".image_location_embeddings", image_loc))
    v = _drop(layer_norm(v, P[ie + ".LayerNorm.weight"], P[ie + ".LayerNorm.bias"]), drop, ie + ".dropout", cfg["hidden_dropout_prob"])
    x = torch.cat([t, v], dim=1)
    dt = x.dtype
    mask = torch.cat([(1.0 - attention_mask[:, None, None, :].to(dt)) * -10000.0,
                      (1.0 - image_attention_mask[:, None, None, :].to(dt)) * -10000.0], dim=3)
    layers = []
    for i in range(cfg["num_hidden_layers"]):
        x = text_layer(P, f"bert.encoder.layer.{i}", cfg, x, mask, drop)
        layers.append(x)
    pooled = torch.tanh(linear(P, "bert.pooler.dense", x[:, 0]))
    return (layers if all_layers else x), pooled


def base_bert_for_vl_tasks(P, cfg, input_txt, input_imgs, image_loc, token_type_ids=None, attention_mask=None, image_attention_mask=None,
                           drop=None):
    """BaseBertForVLTasks.forward (:923-962) -> dict of the seven outputs (OUT_NAMES). self.dropout is one module called twice: on
    the image rows (site "dropout.seq_v") and on the text rows ("dropout.seq_t"); each site's mask is drawn over the whole
    [B, Nt+Nv, H] stream and sliced, as the engine applies it. SimpleClassifier's Dropout(0.5) is site "vil_prediction.main.2"."""
    seq, pooled = bert_model(P, cfg, input_txt, input_imgs, image_loc, token_type_ids, attention_mask, image_attention_mask, drop)
    Nt = input_txt.shape[1]
    seq_t, seq_v = seq[:, :Nt], seq[:, Nt:]
    hv = layer_norm(gelu(linear(P, "cls.imagePredictions.transform.dense", seq_v)),
                    P["cls.imagePredictions.transform.LayerNorm.weight"], P["cls.imagePredictions.transform.LayerNorm.bias"])
    ht = layer_norm(gelu(linear(P, "cls.predictions.transform.dense", seq_t)),
                    P["cls.predictions.transform.LayerNorm.weight"], P["cls.predictions.transform.LayerNorm.bias"])
    out = {}
    out["vision_prediction"] = linear(P, "cls.imagePredictions.decoder", hv)
    out["linguisic_prediction"] = F.linear(ht, P["bert.embeddings.word_embeddings.weight"]) + P["cls.predictions.bias"]
    out["vil_binary_prediction"] = linear(P, "cls.seq_relationship", pooled)
    h = torch.relu(F.linear(pooled, weight_norm(P, "vil_prediction.main.0"), P["vil_prediction.main.0.bias"]))
    h = _drop(h, drop, "vil_prediction.main.2", 0.5)
    out["vil_prediction"] = F.linear(h, weight_norm(P, "vil_prediction.main.3"), P["vil_prediction.main.3.bias"])
    out["vil_logit"] = linear(P, "vil_logit", pooled)
    p = drop.head_p if drop is not None else 0.0
    dv = _drop(seq, drop, "dropout.seq_v", p)[:, Nt:]
    dt = _drop(seq, drop, "dropout.seq_t", p)[:, :Nt]
    out["vision_logit"] = linear(P, "vision_logit", dv) + ((1.0 - image_attention_mask) * -10000.0).unsqueeze(2).to(seq.dtype)
    out["linguisic_logit"] = linear(P, "linguisic_logit", dt)
    return out


def param_shapes(cfg, num_labels):
    """state_dict names and shapes of BaseBertForVLTasks(cfg, num_labels) (without the tied cls.predictions.decoder.weight)."""
    H, I, V = cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"]
    s = {}

    def lin(n, o, i):
        s[n + ".weight"] = (o, i); s[n + ".bias"] = (o,)

    def ln(n):
        s[n + ".weight"] = (H,); s[n + ".bias"] = (H,)
    s["bert.embeddings.word_embeddings.weight"] = (V, H)
    s["bert.embeddings.position_embeddings.weight"] = (cfg["max_position_embeddings"], H)
    s["bert.embeddings.token_type_embeddings.weight"] = (cfg["type_vocab_size"], H)
    ln("bert.embeddings.LayerNorm")
    lin("bert.image_embeddings.image_embeddings", H, 2048)
    s["bert.image_embeddings.token_type_embeddings.weight"] = (cfg["type_vocab_size"], H)
    lin("bert.image_embeddings.image_location_embeddings", H, 5)
    ln("bert.image_embeddings.LayerNorm")
    for i in range(cfg["num_hidden_layers"]):
        p = f"bert.encoder.layer.{i}"
        for n in ("query", "key", "value"):
            lin(f"{p}.attention.self.{n}", H, H)
        lin(f"{p}.attention.output.dense", H, H); ln(f"{p}.attention.output.LayerNorm")
        lin(f"{p}.intermediate.dense", I, H); lin(f"{p}.output.dense", H, I); ln(f"{p}.output.LayerNorm")
    lin("bert.pooler.dense", H, H)
    s["cls.predictions.bias"] = (V,)
    lin("cls.predictions.transform.dense", H, H); ln("cls.predictions.transform.LayerNorm")
    lin("cls.seq_relationship", 2, H)
    lin("cls.imagePredictions.transform.dense", H, H); ln("cls.imagePredictions.transform.LayerNorm")
    lin("cls.imagePredictions.decoder", 1601, H)
    for i, (o, k) in ((0, (2 * H, H)), (3, (num_labels, 2 * H))):
        s[f"vil_prediction.main.{i}.weight_g"] = ()
        s[f"vil_prediction.main.{i}.weight_v"] = (o, k)
        s[f"vil_prediction.main.{i}.bias"] = (o,)
    lin("vil_logit", 1, H); lin("vision_logit", 1, H); lin("linguisic_logit", 1, H)
    return s


def synth_params(cfg, num_labels, seed=0, device="cpu", std=0.05):
    """Seeded parameters of every entry: N(0, std) weights and biases (non-zero biases exercise every bias gradient), LayerNorm
    weights around 1, and g = ||v|| * U(0.5, 1.5) for the weight-normed linears. At hidden size 768 use the reference's
    initializer_range (0.02): with wider weights the attention rows of the upper layers become peaked, their true query / key
    gradients become small, and a relative comparison of them measures the rounding of the bf16 gradient operands."""
    gen = torch.Generator().manual_seed(seed)
    P = {}
    for n, shp in param_shapes(cfg, num_labels).items():
        if n.endswith("weight_g"):
            continue
        t = torch.randn(shp, generator=gen) * std
        if "LayerNorm.weight" in n:
            t = 1.0 + t
        P[n] = t
    for i in (0, 3):
        v = P[f"vil_prediction.main.{i}.weight_v"]
        P[f"vil_prediction.main.{i}.weight_g"] = v.norm() * (0.5 + torch.rand((), generator=gen))
    return {k: v.to(device) for k, v in P.items()}


def synth_inputs(cfg, B, Nt, Nv, seed=1234, device="cpu"):
    """Seeded inputs with ragged text and image masks; ids and token types include the padding index 0."""
    gen = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, cfg["vocab_size"], (B, Nt), generator=gen)
    tt = torch.randint(0, cfg["type_vocab_size"], (B, Nt), generator=gen)
    am = torch.ones(B, Nt, dtype=torch.int64)
    im = torch.ones(B, Nv, dtype=torch.int64)
    for b in range(B):
        am[b, Nt - 1 - (b % max(Nt // 2, 1)):] = 0
        im[b, Nv - 1 - (b % max(Nv // 2, 1)):] = 0
    am[:, 0] = 1
    im[:, 0] = 1
    feat = torch.randn(B, Nv, 2048, generator=gen)
    loc = torch.rand(B, Nv, 5, generator=gen)
    d = dict(input_txt=ids, input_imgs=feat, image_loc=loc, token_type_ids=tt, attention_mask=am, image_attention_mask=im)
    return {k: v.to(device) for k, v in d.items()}


def probe_weights(B, Nt, Nv, num_labels, vocab, seed=7, device="cpu"):
    """Fixed random weights R_o of the scalar objective sum_o <out_o, R_o> whose gradient the fixtures record."""
    gen = torch.Generator().manual_seed(seed)
    shapes = {"vil_prediction": (B, num_labels), "vil_logit": (B, 1), "vil_binary_prediction": (B, 2), "vision_prediction": (B, Nv, 1601),
              "vision_logit": (B, Nv, 1), "linguisic_prediction": (B, Nt, vocab), "linguisic_logit": (B, Nt, 1)}
    return {k: torch.randn(s, generator=gen).to(device) for k, s in shapes.items()}


# --------------------------------------------------------------------------- compact fixtures
FULL_LIMIT, SAMPLES = 512, 128


def digest(t, seed=0):
    """What a fixture keeps of a recorded tensor: the tensor itself up to FULL_LIMIT elements; above, SAMPLES entries at seeded flat
    indices plus its sum, L1 and L2 norms, largest magnitude and (2-D tensors) the largest magnitude of row 0."""
    t = t.detach().float().cpu()
    if t.numel() <= FULL_LIMIT:
        return {"full": t.clone()}
    flat = t.reshape(-1)
    g = torch.Generator().manual_seed(seed * 7919 + flat.numel())
    idx = torch.randperm(flat.numel(), generator=g)[:SAMPLES].to(torch.int32)     # a copy: a slice would keep the whole permutation
    f64 = flat.double()
    d = {"shape": list(t.shape), "idx": idx, "vals": flat[idx].clone(), "sum": float(f64.sum()), "l1": float(f64.abs().sum()),
         "l2": float(f64.norm()), "absmax": float(f64.abs().max())}
    if t.dim() == 2:
        d["row0_absmax"] = float(t[0].abs().max())
    return d


def digest_errors(t, d):
    """(largest sampled error relative to the largest magnitude, error of the L2 norm and of the sum relative to the L1 norm) of `t`
    against a digest; a full tensor gives its max error relative to its largest magnitude for all three."""
    t = t.detach().float().cpu()
    if "full" in d:
        ref = d["full"]
        e = float((t - ref).abs().max() / (ref.abs().max() + 1e-30))
        return e, e, e
    assert list(t.shape) == d["shape"]
    flat = t.reshape(-1)
    am = d["absmax"] + 1e-30
    samp = float((flat[d["idx"].long()] - d["vals"]).abs().max()) / am
    f64 = flat.double()
    l2 = abs(float(f64.norm()) - d["l2"]) / (d["l2"] + 1e-30)
    s = abs(float(f64.sum()) - d["sum"]) / (d["l1"] + 1e-30)
    return samp, l2, s


def row0_absmax(d):
    return float(d["full"][0].abs().max()) if "full" in d else d["row0_absmax"]
