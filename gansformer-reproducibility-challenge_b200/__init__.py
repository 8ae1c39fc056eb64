"""GANsformer bipartite-attention hot path for the H100 (sm_90a CUDA behind a C ABI) + the generator host code.

The directory name carries the reference repo's name and is not a Python identifier; import it as
``import gansformer_b200`` (alias package at the repo root) or via ``importlib.import_module``.
"""
from ._build import build_extension, LIB_PATH  # noqa: F401
from . import _lib  # noqa: F401
from .attention import BipartiteAttention, transformer_layer, bipartite_attention_forward  # noqa: F401
from .networks import Generator, MappingNetwork, SynthesisNetwork, SynthesisLayer, ToRGB, nf  # noqa: F401
from .training import Discriminator, TrainConfig, Trainer  # noqa: F401

__all__ = ["build_extension", "BipartiteAttention", "transformer_layer", "bipartite_attention_forward",
           "Generator", "MappingNetwork", "SynthesisNetwork", "SynthesisLayer", "ToRGB", "nf",
           "Discriminator", "TrainConfig", "Trainer"]
