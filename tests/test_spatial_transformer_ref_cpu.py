"""The fp64 SpatialTransformer reference of tests/test_spatial_transformer_gpu.py (tests/st_oracle.py) against the oracle's
spatial_transformer, the op definitions the whole-model goldens are made with: exact without rounding, with per-sample context
lengths equal to running each sample on its own context, and with every operand rounded equal to the oracle's fp16 emulation."""
import numpy as np
import pytest
import torch

import st_oracle as S
from oracle import sd_oracle as O

NAME = "b"


def small_block(rng, c, unit_ln=False):
    t = f"{NAME}/transformer"
    a = {f"{NAME}/norm/weight": 1 + 0.2 * rng.standard_normal(c), f"{NAME}/norm/bias": 0.2 * rng.standard_normal(c),
         f"{NAME}/proj_in/weight": rng.standard_normal((c, c, 1, 1)) / np.sqrt(c), f"{NAME}/proj_in/bias": rng.standard_normal(c),
         f"{NAME}/proj_out/weight": rng.standard_normal((c, c, 1, 1)) / np.sqrt(c), f"{NAME}/proj_out/bias": 0.1 * rng.standard_normal(c),
         f"{t}/mlp/geglu/proj/weight": rng.standard_normal((c, 8 * c)) / np.sqrt(c), f"{t}/mlp/geglu/proj/bias": 0.1 * rng.standard_normal(8 * c),
         f"{t}/mlp/lin/weight": rng.standard_normal((4 * c, c)) / np.sqrt(4 * c), f"{t}/mlp/lin/bias": 0.1 * rng.standard_normal(c)}
    for i in (1, 2, 3):
        a[f"{t}/norm{i}/weight"] = np.ones(c) if unit_ln else 1 + 0.3 * rng.standard_normal(c)
        a[f"{t}/norm{i}/bias"] = np.zeros(c) if unit_ln else 0.3 * rng.standard_normal(c)
    for at, cin in (("attn1", c), ("attn2", 768)):
        for k in ("query", "key", "value"):
            a[f"{t}/{at}/{k}/weight"] = 1.5 * rng.standard_normal((c if k == "query" else cin, c)) / np.sqrt(c if k == "query" else cin)
        a[f"{t}/{at}/out/weight"] = rng.standard_normal((c, c)) / np.sqrt(c)
        a[f"{t}/{at}/out/bias"] = 0.1 * rng.standard_normal(c)
    return a


def run_both(a, x, ctx, lens, r):
    W = S.block_weights(lambda k, s: a[k], NAME, x.shape[1])
    P = O.Params(a, dtype=torch.float64)
    with torch.no_grad():
        ref, ys = S.spatial_transformer(W, NAME, x, ctx, lens, r)
        ora = torch.cat([O.spatial_transformer(P, NAME, x[s:s + 1], ctx[s:s + 1, :L]) for s, L in enumerate(lens)])
    return ref.numpy(), ys, ora.numpy()


def inputs(rng, n, c, h, w, L):
    x = torch.from_numpy(rng.standard_normal((n, c, h, w)) + 0.5 * rng.standard_normal((1, c, 1, 1)))
    return x, torch.from_numpy(rng.standard_normal((n, L, 768)))


@pytest.mark.parametrize("c,h,w,lens", [(64, 4, 4, (7, 7)), (128, 4, 6, (9, 2)), (64, 2, 4, (1, 5, 3))])
def test_reference_equals_oracle_spatial_transformer(c, h, w, lens):
    """exact block; sample s attends to its first lens[s] context tokens (the rows past them hold values, not padding)"""
    rng = np.random.default_rng(c + h + len(lens))
    a = small_block(rng, c)
    x, ctx = inputs(rng, len(lens), c, h, w, max(lens))
    ref, ys, ora = run_both(a, x, ctx, lens, S.EXACT)
    assert np.abs(ref - ora).max() <= 1e-12 * np.abs(ora).max()
    assert [tuple(y.shape) for y in ys] == [(len(lens) * h * w, c)] * 4


def test_reference_rounding_matches_oracle_emulation():
    """every GEMM single-pass and the attention on fp16 q / k / P / V: the reference rounds exactly where the oracle's fp16
    emulation does, with the oracle's _round. The oracle rounds the LayerNorm input x (its folded-LayerNorm study) and W where the
    reference rounds gamma W, and applies d^-1/4 to q and k before rounding: unit LayerNorm affines and d = 16 (scale 1/2) make
    these the same values. The context K / V of a 3-pass product stay exact on both sides."""
    rng = np.random.default_rng(11)
    c = 128
    a = small_block(rng, c, unit_ln=True)
    x, ctx = inputs(rng, 2, c, 4, 4, 6)
    saved = dict(O._EMU)
    try:
        O.set_emulation("fp16", "awAWq")
        O.set_emulation_fn(lambda blk, name, role: None if name and "/attn2/key" in name or name and "/attn2/value" in name else "fp16")
        O._EMU["ln_fused"] = True
        ref, _, ora = run_both(a, x, ctx, (6, 6), S.Rounding.of(1, False))
    finally:
        O._EMU.clear()
        O._EMU.update(saved)
    exact, _, _ = run_both(a, x, ctx, (6, 6), S.EXACT)
    assert np.abs(ref - ora).max() <= 1e-12 * np.abs(ora).max()
    # and the rounding is not vacuous: it moves the block by fp16-class amounts
    e = np.linalg.norm(ref - exact) / np.linalg.norm(exact)
    assert 1e-5 < e < 1e-2, e
