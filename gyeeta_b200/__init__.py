"""gyeeta_b200 — H100-native streaming-sketch aggregation for Gyeeta's madhava ingest path.

The product is gyeeta_b200/libgysketch.so (hand-written sm_90a CUDA kernels + C++ runtime) behind the C ABI of
include/gysketch.h. This package only holds the build recipe, a thin ctypes binding used by tests / bench, the
seeded synthetic event generators and the torch.distributed plumbing of the multi-GPU merge.
There is no CPU fallback: creating an Engine without the built library or without an sm_90 (H100) GPU raises.
"""
from .engine import Engine, GyskError, EVENT_DTYPE, load_library, LIB_PATH  # noqa: F401
