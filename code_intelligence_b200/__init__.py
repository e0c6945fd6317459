"""H100-native implementation of the kubeflow/Code-Intelligence Issue_Embeddings encoder hot path
(token ids -> 2400-d [mean | max | last]) and the Label_Microservice MLP head.

Python surface mirrors the reference (``InferenceWrapper``, ``MLPWrapper``); the arithmetic is hand-written
sm_90a CUDA behind the C ABI declared in ``include/issue_emb_b200.h``.  No CPU fallback exists.
"""
from ._lib import IE_MAX_BATCH, LIB_PATH, build, load  # noqa: F401
from .encoder import IssueEncoder  # noqa: F401

__all__ = ["IssueEncoder", "IE_MAX_BATCH", "LIB_PATH", "build", "load"]
