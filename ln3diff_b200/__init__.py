"""ln3diff_b200 -- H100-native (sm_90a) implementation of the LN3Diff generation hot path.

Host side mirrors the reference's Python interface for the path (DiT_models, samplers, Triplane /
ImportanceRenderer); the device work is hand-written CUDA in libln3b200.so behind a C ABI
(include/ln3b200.h) bound with ctypes in `_lib.py`.
"""
__version__ = "0.1.0"
