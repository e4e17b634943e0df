"""The GEMM's shared-memory stage ring across its wrap-around points, exactly, for all 12 (tile width, pass count) instances.

Each instantiation sizes its ring to the shared memory it can use: 2 stages for the 3-pass 128 x 256 tile, up to 8 for the 1-pass
128 x 64 tile. A slot handed back one phase early or late shows only at some k-chunk counts, so every count from 1 to past the
second wrap of each ring (2 * stages + 1) is run, with a masked second M tile. The operands are lo-visible (gemm_ref.py): their
fp16 lo halves are non-zero and every partial sum is exact in fp32, so a lo tile read from the wrong stage changes the result,
and each pass count must reproduce the exact sum of the terms it forms bit for bit. The launch trace must show the tile width,
stage count and split = 1 each case is meant to reach.
"""
import numpy as np
import pytest

import gemm_ref as G

pytestmark = pytest.mark.gpu

# N -> the tile width it selects: 96 = two 64-wide column tiles, the second half masked; 1024 takes 256-wide tiles when the M
# tiles fill the machine (rows from the device's SM count)
WIDTHS = {96: 64, 384: 128, 320: 160, 1024: 256}
OLD_CHUNKS = (1, 2, 3, 4, 5, 6, 7, 8, 9, 13, 15)
CASES = sorted({(chunks, N, passes)
                for N, bn in WIDTHS.items() for passes in (1, 2, 3)
                for chunks in set(range(1, 2 * G.pick_stages(bn, passes) + 2)) | (set(OLD_CHUNKS) if bn in (128, 160) else set())},
               key=lambda c: (c[1], c[2], c[0]))


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("chunks,N,passes", CASES)
def test_ring_wraps_exact(ctx, sms, chunks, N, passes):
    bn = WIDTHS[N]
    K = 64 * chunks
    M = G.bn256_rows(sms) if bn == 256 else 200  # the last M tile masked
    a = G.lo_visible((M, K), chunks)
    w = G.lo_visible((K, N), 100 + chunks)
    out, tr = ctx.test_linear(a, w, None, passes=passes, trace=True)
    assert [(g["BN"], g["stages"], g["split"], g["passes"]) for g in tr] == [(bn, G.pick_stages(bn, passes), 1, passes)]
    assert np.array_equal(out.astype(np.float64), G.pass_product(a, w, passes))


@pytest.mark.parametrize("passes", [1, 3])
def test_ring_split_k_exact(ctx, sms, passes):
    """45 k-chunks (the level-0 conv's depth) over 4 CTAs: split-K (5 ways on 132 SMs, 9 chunks per split), so each split wraps
    its ring."""
    K = 64 * 45
    a = np.random.default_rng(7).integers(-4, 5, (256, K)).astype(np.float32)
    w = np.random.default_rng(8).integers(-4, 5, (K, 320)).astype(np.float32)
    out, tr = ctx.test_linear(a, w, None, passes=passes, trace=True)
    assert [(g["BN"], g["split"]) for g in tr] == [(160, G.pick_split(2, 2, 45, sms))] and tr[0]["split"] > 1
    assert np.array_equal(out, a @ w)
