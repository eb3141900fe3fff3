"""H100-native SeedVR2 DiT + video-VAE hot path (see DESIGN.md).

Host code is thin Python; all compute goes through the C-ABI library
``csrc/libsvr2.so`` (``include/svr2.h``).  There is no CPU fallback: importing
``engine`` without the built library raises.
"""
from . import weights  # noqa: F401
