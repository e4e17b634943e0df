"""Minimal stand-in for tinygrad 0.9.2 (TEST INFRASTRUCTURE, see ../README.md): only what the reference's python/ directory uses."""
from .tensor import Tensor  # noqa: F401


class dtypes:  # `from tinygrad import dtypes` (python/dump.py:17) — imported there, never used
    float32 = "float32"
    int32 = "int32"
