"""sniffles_b200 — H100-native lead -> cluster -> consensus hot path of Sniffles2.

Only what the path needs: csrc/ (CUDA kernels + C ABI), the ctypes binding, the host-side
mirror of the reference's Task interface and the synthetic input generator."""
__version__ = "0.1.0"
