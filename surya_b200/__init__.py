"""surya_b200 — Hopper-native (sm_90a) engine for surya's batched model forward passes.

Host side mirrors the reference's predictor/model call surface; every forward op is a hand-written CUDA
kernel in libsurya_b200.so reached through the C ABI in include/surya_b200.h.  There is no CPU or
PyTorch-eager fallback: importing is cheap, but any compute call raises without the library and a GPU.
"""
__version__ = "0.1.0"
