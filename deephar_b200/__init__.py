"""deephar_b200 -- H100-native (sm_90a) forward hot path of dluvizon/deephar.

Host side mirrors the reference's Python surface (reception.build, spnet.build(ModelConfig),
layers.*, keras.Model protocol); all arithmetic runs in libdeephar_b200.so (hand-written CUDA,
C ABI in include/deephar_b200.h).  No CPU fallback.
"""
from . import layers  # noqa: F401
from . import reception  # noqa: F401
from .model import Model  # noqa: F401

__version__ = '0.1.0'
