"""H100-native (sm_90a) Stable Diffusion v1.4 sampling hot path behind the reference's interface.

Product code lives in csrc/ (CUDA kernels + C ABI, built into libsdb200.so); this package is the
thin Python host side mirroring the reference's Rust signatures (pipeline.py). The CPU oracle
under /oracle is test infrastructure and is never imported from here.
"""
from . import synth, topology  # noqa: F401

__all__ = ["synth", "topology"]
