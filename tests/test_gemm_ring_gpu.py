"""The GEMM's shared-memory stage ring across its wrap-around points, exactly.

Each instantiation sizes its ring to the shared memory it can use: 3 stages for the 3-pass 128 x 160 tile, up to 8 for 1-pass
tiles. A slot handed back one phase early or late shows only at some k-chunk counts, so every count from 1 to past the second
wrap of each ring is run. Small-integer operands are exact in fp16 (their lo halves are zero) and every partial sum is an
integer below 2^24, so each pass count and each split-K fold must reproduce the product bit for bit.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def ints(shape, seed):
    return np.random.default_rng(seed).integers(-4, 5, shape).astype(np.float32)


@pytest.mark.parametrize("passes", [1, 2, 3])
@pytest.mark.parametrize("N", [320, 384])  # 128 x 160 tiles (3/4/6 stages) and 128 x 128 tiles (3/4/7 stages)
@pytest.mark.parametrize("chunks", [1, 2, 3, 4, 5, 6, 7, 8, 9, 13, 15])
def test_ring_wraps_exact(ctx, passes, N, chunks):
    K = 64 * chunks
    a = ints((200, K), chunks)  # two M tiles, the second one masked
    w = ints((K, N), 100 + chunks)
    out = ctx.test_linear(a, w, None, passes=passes)
    assert np.array_equal(out, a @ w)


@pytest.mark.parametrize("passes", [1, 3])
def test_ring_split_k_exact(ctx, passes):
    """45 k-chunks (the level-0 conv's depth) over 4 CTAs: split-K 5 ways, 9 chunks per split, so each split wraps its ring."""
    K = 64 * 45
    a = ints((256, K), 7)
    w = ints((K, 320), 8)
    out = ctx.test_linear(a, w, None, passes=passes)
    assert np.array_equal(out, a @ w)
