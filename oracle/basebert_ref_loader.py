"""ORACLE — TEST INFRASTRUCTURE. Imports the UNMODIFIED reference single-stream baseline (vilbert/basebert.py) with the stubs of
oracle/ref_loader.py plus one more: pytorch_transformers.modeling_bert.BertConfig, which basebert.py imports but only uses as an
attribute bag. Used only by tools/make_basebert_golden.py (the reference does not exist on the GPU box)."""
import sys
import types

from . import ref_loader


class BertConfig:
    """Stand-in for pytorch_transformers.modeling_bert.BertConfig: an attribute bag (basebert.py reads config.<field>)."""

    def __init__(self, **fields):
        self.__dict__.update(fields)


def load():
    ref_loader.load()
    if "pytorch_transformers.modeling_bert" not in sys.modules:
        pt = types.ModuleType("pytorch_transformers")
        mb = types.ModuleType("pytorch_transformers.modeling_bert")
        mb.BertConfig = BertConfig
        pt.modeling_bert = mb
        sys.modules["pytorch_transformers"] = pt
        sys.modules["pytorch_transformers.modeling_bert"] = mb
    import vilbert.basebert as base  # noqa: E402
    return base
