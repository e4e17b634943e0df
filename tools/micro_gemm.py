"""Fixed-cost probe of gemm_tc. With SDB_GEMM_DBG=1 every launch prints the clock64 stamps of its first CTA, in cycles since
entry: prologue done / first TMA issued / first operands landed / last MMA issued / accumulator ready / epilogue done / exit,
then the raw clock64 counter value at entry."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from stable_diffusion_burn_b200 import _lib
c = _lib.Context(0)
rng = np.random.default_rng(0)
SHAPES = [(8192, 64, 320, 3), (8192, 320, 320, 3), (8192, 2880, 320, 3), (8192, 320, 320, 1), (2048, 640, 640, 3),
          (512, 1280, 1280, 1), (128, 1280, 1280, 1), (512, 5120, 1280, 1)]
for (M, K, N, passes) in SHAPES:
    a = rng.standard_normal((M, K)).astype(np.float32); w = (rng.standard_normal((K, N)) * K ** -0.5).astype(np.float32)
    for _ in range(3):
        out = c.test_linear(a, w, np.zeros(N, np.float32), passes=passes)
print("ok")
