"""Drop-in module surface of the single-stream baseline (vilbert/basebert.py): BaseBertForVLTasks, the model `--baseline` selects in
train_tasks.py / eval_tasks.py / eval_retrieval.py, and its BertModel, with the reference's constructor / forward signatures, output
tuples and state_dict key names, executing on the H100 engine (engine.BasePlan). A driver swaps
`from vilbert.basebert import BaseBertForVLTasks` for `from vilbert_b200.basebert import BaseBertForVLTasks`.

Text and image embeddings are LayerNormed into one [B, Nt+Nv, H] stream that num_hidden_layers BERT layers process under the
concatenated mask; the pooler is tanh on row 0 (the text CLS token); vil_prediction is SimpleClassifier with its two weight-normed
(dim=None) linears. As everywhere in this package there is no PyTorch / CPU fallback.
"""
import math

import torch

from .engine import BASE_BERT_OUT_NAMES, BASE_HEAD_NAMES
from .modeling import BertPreTrainedModel, _BertNode


class _BaseBertNode(_BertNode):
    """The `bert` sub-module: owns the bert.* parameters and, called like the reference's `self.bert(...)` (basebert.py:933-941),
    runs basebert.BertModel.forward on them."""

    def forward(self, input_txt, input_imgs, image_loc, token_type_ids=None, attention_mask=None, image_attention_mask=None,
                output_all_encoded_layers=True):
        return self.__dict__["_owner_ref"]()._bert_forward(input_txt, input_imgs, image_loc, token_type_ids, attention_mask,
                                                           image_attention_mask, output_all_encoded_layers)


class _BaseModel(BertPreTrainedModel):
    """Shared forward machinery of the two baseline classes."""

    def __init__(self, config, device=None, precision=None, num_labels=None):
        super().__init__(config, device, precision, num_labels=num_labels)
        self.bert.__class__ = _BaseBertNode

    def _heads_for(self, names):
        return "none" if all(n in BASE_BERT_OUT_NAMES for n in names) else None

    def init_weights(self):
        """init_bert_weights (basebert.py:139-152) applied by BaseBertForVLTasks.__init__: N(0, initializer_range) for Linear and
        Embedding weights, zero biases, LayerNorm 1 / 0. For the weight-normed linears `apply` writes the derived `.weight`, which
        the next forward recomputes: their parameters keep nn.Linear's default v ~ U(-1/sqrt(in), 1/sqrt(in)) with g = ||v||, and
        the bias zeroed."""
        super().init_weights()
        with torch.no_grad():
            for i in (0, 3):
                nm = f"vil_prediction.main.{i}"
                if nm + ".weight_v" not in self._params:
                    continue
                v = self._params[nm + ".weight_v"]
                bound = 1.0 / math.sqrt(v.shape[1])
                v.uniform_(-bound, bound)
                self._params[nm + ".weight_g"].copy_(v.norm())

    def _base_forward(self, names, input_txt, input_imgs, image_loc, token_type_ids, attention_mask, image_attention_mask):
        inputs = dict(input_txt=input_txt, input_imgs=input_imgs, image_loc=image_loc, token_type_ids=token_type_ids,
                      attention_mask=attention_mask, image_attention_mask=image_attention_mask, task_ids=None)
        names = tuple(names)
        plan = self._outputs_plan(names, inputs, bool(self.training), input_grads=self._input_grads(inputs))
        outs = self._call(plan, inputs, names=names)
        return dict(zip(names, outs))

    def _bert_forward(self, input_txt, input_imgs, image_loc, token_type_ids=None, attention_mask=None, image_attention_mask=None,
                      output_all_encoded_layers=True):
        """basebert.BertModel.forward (basebert.py:706-774): (encoded_layers, pooled_output). With output_all_encoded_layers the first
        entry is the list of every layer's output, of which only the last is connected to autograd."""
        o = self._base_forward(BASE_BERT_OUT_NAMES, input_txt, input_imgs, image_loc, token_type_ids, attention_mask, image_attention_mask)
        seq, pooled = o["sequence_output"], o["pooled_output"]
        if output_all_encoded_layers:
            plan = self._last_plan
            layers = [a.f32.view(seq.shape).clone() for a in plan.enc[:-1]]
            return layers + [seq], pooled
        return seq, pooled


class BertModel(_BaseModel):
    """Reference: vilbert/basebert.py:654-774. Parameters live under the bare names (embeddings.*, image_embeddings.*, encoder.*,
    pooler.*)."""
    _heads = "base_none"

    def state_dict(self, *a, **k):
        sd = super().state_dict(*a, **k)
        return type(sd)((key[len("bert."):], v) for key, v in sd.items() if key.startswith("bert."))

    def load_state_dict(self, state_dict, strict=True):
        return super().load_state_dict({"bert." + k: v for k, v in state_dict.items()}, strict=strict)

    def forward(self, input_txt, input_imgs, image_loc, token_type_ids=None, attention_mask=None, image_attention_mask=None,
                output_all_encoded_layers=True):
        return self._bert_forward(input_txt, input_imgs, image_loc, token_type_ids, attention_mask, image_attention_mask,
                                  output_all_encoded_layers)


class BaseBertForVLTasks(_BaseModel):
    """Reference: vilbert/basebert.py:893-962. forward returns the 7-tuple (vil_prediction, vil_logit, vil_binary_prediction,
    vision_prediction, vision_logit, linguisic_prediction, linguisic_logit); co_attention_mask is accepted and ignored like the
    reference's. `model.bert(...)` runs basebert.BertModel.forward on the same parameters."""
    _heads = "base"

    def __init__(self, config, num_labels, dropout_prob=0.1, default_gpu=True, device=None, precision=None):
        super().__init__(config, device, precision, num_labels)
        self.num_labels = num_labels
        self.dropout_prob = dropout_prob
        self.engine.head_dropout_prob = dropout_prob

    def forward(self, input_txt, input_imgs, image_loc, token_type_ids=None, attention_mask=None, image_attention_mask=None,
                co_attention_mask=None, output_all_encoded_layers=False):
        if output_all_encoded_layers:
            raise NotImplementedError("BaseBertForVLTasks(output_all_encoded_layers=True): the reference slices the list of layers as "
                                      "a tensor and fails the same way; use model.bert(..., output_all_encoded_layers=True)")
        if image_attention_mask is None:
            raise TypeError("image_attention_mask is required by BaseBertForVLTasks.forward (basebert.py:949-951)")
        o = self._base_forward(BASE_HEAD_NAMES, input_txt, input_imgs, image_loc, token_type_ids, attention_mask, image_attention_mask)
        return tuple(o[n] for n in BASE_HEAD_NAMES)
