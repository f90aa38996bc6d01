"""vilbert-multi-task_b200 — Hopper-native ViLBERT two-stream co-attentional encoder.

Python surface mirrors the reference (vilbert/vilbert.py: BertConfig, BertModel, VILBertForVLTasks,
BertForMultiModalPreTraining); the arithmetic runs in libvilbert_b200.so (hand-written sm_90a CUDA,
C ABI in include/vilbert_b200.h). Import as ``vilbert_b200``.
"""
__version__ = "0.1.0"

from .config import BertConfig  # noqa: E402,F401


def __getattr__(name):
    # modeling / engine import torch and bind the shared library: load them lazily
    if name in ("BertModel", "VILBertForVLTasks", "BertForMultiModalPreTraining", "BertPreTrainedModel"):
        from . import modeling
        return getattr(modeling, name)
    if name in ("ForwardModelsTrain", "ForwardModelsVal", "LoadLosses"):
        from . import tasks
        return getattr(tasks, name)
    if name in ("RetrievalEvaluator", "evaluate_retrieval", "evaluate_retrieval_both", "retrieval_metrics", "i2t_metrics"):
        from . import retrieval
        return getattr(retrieval, name)
    if name in ("Engine", "Plan", "ParamStore"):
        from . import engine
        return getattr(engine, name)
    raise AttributeError(name)
