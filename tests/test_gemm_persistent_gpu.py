"""The persistent tile loop and the register epilogue of gemm_tc (LNC, GEGLU, GEGLU_LNC).

Those instances launch at most one CTA per SM; each CTA runs tiles c, c + G, c + 2G, ... and carries the operand ring's slot and
phase from one tile to the next. The shapes here have more tiles than SMs, a tile count that is not a multiple of the grid, a
masked last M tile, and a K that wraps the ring at least twice per tile, at 1, 2 and 3 passes.

* The same rows launched 128 at a time (a single-tile grid per launch) give the same bits, and the result meets the fp64 bars of
  test_gemm_instances_gpu.py.
* A launch repeated around another shape gives an identical result.
"""
import math

import numpy as np
import pytest
import torch

import gemm_ref as G

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def gelu_erf(x):
    return 0.5 * x * (1.0 + np.vectorize(math.erf)(x / math.sqrt(2.0)))


def rows_for(sms, n_tiles):
    """Rows whose 128-row tiles times n_tiles exceed the SM count by a few tiles and are not a multiple of it; last tile masked."""
    m_tiles = sms // n_tiles + 3
    assert (m_tiles * n_tiles) > sms and (m_tiles * n_tiles) % sms != 0
    return m_tiles * 128 - 40


def assert_tile_loop(g, bn, passes, epi):
    assert (g["BN"], g["stages"], g["passes"], g["split"], G.epi_of(g["epi"])) == (bn, G.pick_stages(bn, passes), passes, 1, epi)


# ------------------------------------------------------------------ LNC / GEGLU_LNC / GEGLU: tile loop == single-tile grids
LN_CASES = {"LNC128": (384, False, 128, "LNC"), "LNC160": (320, False, 160, "LNC"), "GEGLU_LNC": (512, True, 128, "GEGLU_LNC")}
C_LN = 1280  # 20 k-chunks: at least twice the deepest ring (7 stages of a 1-pass 128-wide tile)


def ln_operands(M, N, seed):
    rng = np.random.default_rng(seed)
    K0 = 320
    a = rng.standard_normal((M, K0)).astype(np.float32)
    w0 = (rng.standard_normal((K0, C_LN)) / math.sqrt(K0)).astype(np.float32)
    b0 = (rng.standard_normal(C_LN) * 0.5 + 1.5).astype(np.float32)
    g = (1 + 0.1 * rng.standard_normal(C_LN)).astype(np.float32); be = (0.1 * rng.standard_normal(C_LN)).astype(np.float32)
    w1 = (rng.standard_normal((C_LN, N)) / math.sqrt(C_LN)).astype(np.float32)
    b1 = rng.standard_normal(N).astype(np.float32) * 0.3
    return a, w0, b0, g, be, w1, b1


@pytest.mark.parametrize("passes", (1, 2, 3))
@pytest.mark.parametrize("case", sorted(LN_CASES))
def test_ln_consumer_tile_loop(ctx, sms, case, passes):
    N, geglu, bn, epi = LN_CASES[case]
    assert C_LN // 64 >= 2 * G.pick_stages(bn, passes)
    M = rows_for(sms, N // bn)
    a, w0, b0, g, be, w1, b1 = ln_operands(M, N, N + passes)
    ctx.set_option("precision", passes)
    try:
        out, tr = ctx.test_ln_fold(a, w0, b0, g, be, w1, b1, passes=passes, geglu=geglu, trace=True)
        parts = [ctx.test_ln_fold(a[i:i + 128], w0, b0, g, be, w1, b1, passes=passes, geglu=geglu) for i in range(0, M, 128)]
    finally:
        ctx.set_option("precision", 0)
    assert len(tr) == 2
    assert_tile_loop(tr[1], bn, passes, epi)
    assert np.array_equal(out, np.concatenate(parts))
    ar, w0r = G.rounded_operands(a, w0, passes)
    y = ar.astype(np.float64) @ w0r.astype(np.float64) + b0
    mu = y.mean(-1, keepdims=True); var = ((y - mu) ** 2).mean(-1, keepdims=True)
    pre = ((y - mu) / np.sqrt(var + 1e-5) * g + be) @ w1.astype(np.float64) + b1
    ref = pre[:, :N // 2] * gelu_erf(pre[:, N // 2:]) if geglu else pre
    assert rel(out, ref) < (4e-5 if passes == 3 else 1.5e-3)


@pytest.mark.parametrize("passes", (1, 2, 3))
def test_geglu_tile_loop(ctx, sms, passes):
    K, N = C_LN, 512
    M = rows_for(sms, N // 128)
    rng = np.random.default_rng(K + N + passes)
    a = rng.standard_normal((M, K)).astype(np.float32)
    w = (rng.standard_normal((K, N)) / math.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32) * 0.1
    out, tr = ctx.test_gemm_ex(a, w, bias=b, passes=passes, geglu=True, trace=True)
    assert_tile_loop(tr[0], 128, passes, "GEGLU")
    parts = [ctx.test_gemm_ex(a[i:i + 128], w, bias=b, passes=passes, geglu=True) for i in range(0, M, 128)]
    assert np.array_equal(out, np.concatenate(parts))
    ar, wr = G.rounded_operands(a, w, passes)
    p = ar.astype(np.float64) @ wr.astype(np.float64) + b
    ref = p[:, :N // 2] * gelu_erf(p[:, N // 2:])
    assert rel(out, ref) < (5e-5 if passes == 3 else 2e-4)


def test_tile_loop_repeats_around_another_shape(ctx, sms):
    """Ring slot and phase start afresh in every launch: a shape, another shape with a different tile count, the first again."""
    rng = np.random.default_rng(5)
    M = rows_for(sms, 4)
    a = rng.standard_normal((M, C_LN)).astype(np.float32); w = (rng.standard_normal((C_LN, 512)) / 32).astype(np.float32)
    a2 = rng.standard_normal((M + 300, 640)).astype(np.float32); w2 = (rng.standard_normal((640, 768)) / 32).astype(np.float32)
    b, b2 = np.zeros(512, np.float32), np.zeros(768, np.float32)
    first = ctx.test_gemm_ex(a, w, bias=b, passes=3, geglu=True)
    between = ctx.test_gemm_ex(a2, w2, bias=b2, passes=1, geglu=True)
    again = ctx.test_gemm_ex(a, w, bias=b, passes=3, geglu=True)
    assert np.array_equal(first, again)
    parts = [ctx.test_gemm_ex(a2[i:i + 128], w2, bias=b2, passes=1, geglu=True) for i in range(0, M + 300, 128)]
    assert np.array_equal(between, np.concatenate(parts))
