"""cmgan_b200: H100-native (sm_90a) hot path of CMGAN behind the reference's nn.Module interface.

    from cmgan_b200 import TSCNet, Discriminator, power_compress, power_uncompress

The compute is libcmgan_b200.so (hand-written CUDA, C ABI in include/cmgan_b200.h); there is no CPU or
PyTorch-op fallback: importing works anywhere, running requires the built library and a CUDA device.
"""
from .generator import TSCNet  # noqa: F401
from .discriminator import Discriminator  # noqa: F401
from .utils import power_compress, power_uncompress  # noqa: F401
from . import signal  # noqa: F401

__all__ = ["TSCNet", "Discriminator", "power_compress", "power_uncompress", "signal"]
