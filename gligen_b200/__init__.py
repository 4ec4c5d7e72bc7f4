"""gligen_b200: Hopper-native (sm_90a) GLIGEN denoising engine.

Host code is Python/PyTorch (plumbing); every hot op is a hand-written CUDA kernel reached
through the C-ABI library `libgligen_b200.so` (see include/gligen_b200.h).
"""
from .spec import UNetConfig, NAMED_CONFIGS  # noqa: F401

__version__ = "0.1.0"
