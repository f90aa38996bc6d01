"""BertConfig — same constructor, defaults, JSON handling and post-hoc attribute mutation as the
reference's configuration class (vilbert/vilbert.py:141-294), so that the reference's config/*.json
files and driver-side tweaks (``config.task_specific_tokens = True`` ...) work unchanged."""
import copy
import json


class BertConfig(object):
    def __init__(
        self,
        vocab_size_or_config_json_file,
        hidden_size=768,
        num_hidden_layers=12,
        num_attention_heads=12,
        intermediate_size=3072,
        hidden_act="gelu",
        hidden_dropout_prob=0.1,
        attention_probs_dropout_prob=0.1,
        max_position_embeddings=512,
        type_vocab_size=2,
        initializer_range=0.02,
        v_feature_size=2048,
        v_target_size=1601,
        v_hidden_size=768,
        v_num_hidden_layers=3,
        v_num_attention_heads=12,
        v_intermediate_size=3072,
        bi_hidden_size=1024,
        bi_num_attention_heads=16,
        v_attention_probs_dropout_prob=0.1,
        v_hidden_act="gelu",
        v_hidden_dropout_prob=0.1,
        v_initializer_range=0.2,
        v_biattention_id=[0, 1],
        t_biattention_id=[10, 11],
        visual_target=0,
        fast_mode=False,
        fixed_v_layer=0,
        fixed_t_layer=0,
        in_batch_pairs=False,
        fusion_method="mul",
        dynamic_attention=False,
        with_coattention=True,
        objective=0,
        num_negative=128,
        model="bert",
        task_specific_tokens=False,
        visualization=False,
    ):
        assert len(v_biattention_id) == len(t_biattention_id)
        assert max(v_biattention_id) < v_num_hidden_layers
        assert max(t_biattention_id) < num_hidden_layers
        if isinstance(vocab_size_or_config_json_file, str):
            with open(vocab_size_or_config_json_file, "r", encoding="utf-8") as reader:
                json_config = json.loads(reader.read())
            for key, value in json_config.items():
                self.__dict__[key] = value
        elif isinstance(vocab_size_or_config_json_file, int):
            loc = dict(locals())
            self.vocab_size = vocab_size_or_config_json_file
            for k, v in loc.items():
                if k not in ("self", "vocab_size_or_config_json_file", "loc"):
                    self.__dict__[k] = v
        else:
            raise ValueError("First argument must be either a vocabulary size (int)"
                             "or the path to a pretrained model config file (str)")

    @classmethod
    def from_dict(cls, json_object):
        """Starts from the constructor defaults and overwrites per JSON key (vilbert.py:263-268)."""
        config = BertConfig(vocab_size_or_config_json_file=-1)
        for key, value in json_object.items():
            config.__dict__[key] = value
        return config

    @classmethod
    def from_json_file(cls, json_file):
        with open(json_file, "r", encoding="utf-8") as reader:
            text = reader.read()
        return cls.from_dict(json.loads(text))

    def __repr__(self):
        return str(self.to_json_string())

    def to_dict(self):
        return copy.deepcopy(self.__dict__)

    def to_json_string(self):
        return json.dumps(self.to_dict(), indent=2, sort_keys=True) + "\n"

    # ---- support checks for the H100 engine (features the reference has but the hot path here does not)
    def check_supported(self):
        unsupported = []
        if self.hidden_act != "gelu" or self.v_hidden_act != "gelu":
            unsupported.append("hidden_act != 'gelu'")
        # model="roberta": RobertaEmbeddings' shifted position ids are overwritten by BertEmbeddings.forward (vilbert.py:347-351,
        # 380-393), so its embeddings ARE the BERT ones (pinned: tests/golden/tiny_roberta.json); with task tokens the reference
        # raises a TypeError (task_ids land in position_ids), mirrored here
        if getattr(self, "model", "bert") not in ("bert", "roberta"):
            unsupported.append("model=%r" % (self.model,))
        if getattr(self, "model", "bert") == "roberta" and getattr(self, "task_specific_tokens", False):
            unsupported.append("model='roberta' with task_specific_tokens (the reference cannot run it either: RobertaEmbeddings.forward takes no task_ids)")
        if getattr(self, "dynamic_attention", False) and (getattr(self, "in_batch_pairs", False) or getattr(self, "fast_mode", False)):
            # the reference hands the UNEXPANDED text mask to the gate's pooling after the batch expansion (vilbert.py:1008-1053, 1084)
            unsupported.append("dynamic_attention together with in_batch_pairs / fast_mode")
        if getattr(self, "fixed_t_layer", 0) > min(self.t_biattention_id) or getattr(self, "fixed_v_layer", 0) > min(self.v_biattention_id):
            unsupported.append("fixed_t_layer / fixed_v_layer beyond the first connection layer (the reference asserts the same, vilbert.py:965-966)")
        if getattr(self, "in_batch_pairs", False) and getattr(self, "fast_mode", False):
            unsupported.append("in_batch_pairs together with fast_mode")
        if unsupported:
            raise NotImplementedError("vilbert_b200: unsupported config options: " + ", ".join(unsupported))
