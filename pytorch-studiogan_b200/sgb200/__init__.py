"""sgb200 — H100-native hot path of StudioGAN (BigGAN / BigGAN-Deep G+D step and the FID/IS/PRDC evaluation).

Python here is host glue: module / step API mirroring the reference (``models``, ``utils.ops``, ``utils.losses``,
``worker``), device memory and streams from PyTorch, and ctypes calls into ``lib/libsgb200.so`` (hand-written sm_90a
CUDA behind the C ABI in ``include/sgb200.h``).  There is no CPU or PyTorch fallback for the kernels.
"""
__version__ = "0.1.0"
