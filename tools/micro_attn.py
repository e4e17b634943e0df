"""Timeline probe of the fused attention kernel. With SDB_ATTN_DBG=1 every launch prints clock64 stamps of CTA (0,0,0) for key
tiles 8..11, taken by the first softmax warpgroup: S = QK^T issued, S ready, softmax done, PV issued, PV done (the P V product
of a tile is issued after the next tile's QK^T).
   SDB_ATTN_DBG=1 python tools/micro_attn.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from stable_diffusion_burn_b200 import _lib
c = _lib.Context(0)
rng = np.random.default_rng(0)
for (n, Nq, Nk, C, heads) in [(1, 4096, 4096, 320, 8)]:
    q, k, v = (rng.standard_normal((n, N, C)).astype(np.float32) for N in (Nq, Nk, Nk))
    for _ in range(2):
        c.test_attention(q, k, v, heads)
print("ok")
