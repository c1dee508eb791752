"""selftoktokenizer_b200 — H100-native (sm_90a) implementation of the SelftokTokenizer encode / decode hot path.

Public surface mirrors mimogpt/infer/SelftokPipeline.py: `SelftokPipeline`, `NormalizeToTensor`,
`parse_args_from_yaml`.  All arithmetic on the path runs in hand-written CUDA behind the C-ABI declared
in include/selftok_b200.h (built to selftoktokenizer_b200/csrc/libselftok_b200.so); there is no CPU or
PyTorch fallback — importing the engine without the built library raises.
"""
from .config import AttrDict, SelftokDims, parse_args_from_yaml, FULL, TINY  # noqa: F401

__all__ = ["SelftokPipeline", "NormalizeToTensor", "parse_args_from_yaml", "SelftokDims"]


def __getattr__(name):
    if name in ("SelftokPipeline", "NormalizeToTensor", "norm_ip", "DeviceVAE"):
        from . import pipeline
        return getattr(pipeline, name)
    raise AttributeError(name)
