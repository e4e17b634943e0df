"""fp64 reference of one UNet SpatialTransformer (unet/mod.rs:461-481, 521-527, 551-592, 641-653) in the form the CUDA path
computes it, for tests/test_spatial_transformer_gpu.py.

The block is restated from torch primitives: the three LayerNorms as the consuming GEMMs apply them (the raw residual y times
gamma-folded weights, then rstd * (acc - mean * colsum) + beta^T W), per-sample context lengths, the residual stream y exposed
after each stage. `Rounding` names which operands are rounded to fp16 (the oracle's `_round`) the way the kernels consume them:
  * a 1-pass GEMM reads fp16 values of both operands: its activation (including the fp16 y the folded consumers read, whose
    statistics come from the unrounded y) and its weights (gamma W rounded after the fold);
  * a 3-pass GEMM reads hi + lo pairs of both (22 bits each): exact here;
  * the attention always reads V and the probabilities P as fp16, and q / k as fp16 unless it forms the logits as the 3-term
    split product of their hi + lo pairs. (The kernel rounds P before dividing by the row sum, against a running maximum: the
    same relative rounding, not the same bits. Rounding the normalised P keeps the reference the oracle's emulation.)
`Rounding()` (all off) is the exact block: tests/test_spatial_transformer_ref_cpu.py shows it equals the oracle's
spatial_transformer."""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch
import torch.nn.functional as F

from oracle.sd_oracle import _round, gelu_erf

HEADS = 8


@dataclass(frozen=True)
class Rounding:
    passes: int = 3      # passes of the block's GEMMs (all but the context K / V)
    qk_split: bool = True  # attention logits from hi + lo q / k (else fp16 q / k)
    attention: bool = False  # fp16 P and V (and q / k unless qk_split)

    @staticmethod
    def of(passes, qk_split):
        return Rounding(passes, qk_split, True)


EXACT = Rounding()


def block_weights(get, name, c):
    """the block's tensors under their dump-dir names (prefix `name`), fp64; get(name, shape) -> array"""
    t = f"{name}/transformer"
    shapes = {f"{name}/norm/weight": (c,), f"{name}/norm/bias": (c,), f"{name}/proj_in/weight": (c, c, 1, 1),
              f"{name}/proj_in/bias": (c,), f"{name}/proj_out/weight": (c, c, 1, 1), f"{name}/proj_out/bias": (c,),
              f"{t}/mlp/geglu/proj/weight": (c, 8 * c), f"{t}/mlp/geglu/proj/bias": (8 * c,), f"{t}/mlp/lin/weight": (4 * c, c),
              f"{t}/mlp/lin/bias": (c,)}
    for i in (1, 2, 3):
        shapes[f"{t}/norm{i}/weight"] = shapes[f"{t}/norm{i}/bias"] = (c,)
    for a, cin in (("attn1", c), ("attn2", 768)):
        shapes[f"{t}/{a}/query/weight"] = (c, c)
        shapes[f"{t}/{a}/key/weight"] = shapes[f"{t}/{a}/value/weight"] = (cin, c)
        shapes[f"{t}/{a}/out/weight"] = (c, c)
        shapes[f"{t}/{a}/out/bias"] = (c,)
    return {k: torch.from_numpy(np.asarray(get(k, s), np.float64)) for k, s in shapes.items()}


def _attention(q, k, v, lens, rnd, qk_split):
    """q [n, Nq, C], k / v [n, Nk, C]; sample s sees its first lens[s] keys. softmax(q k^T / sqrt(d)) v per head."""
    r16 = lambda a: _round(a, "fp16")
    if rnd:
        v = r16(v)
        if not qk_split:
            q, k = r16(q), r16(k)
    n, _, c = q.shape
    d = c // HEADS
    out = torch.empty_like(q)
    for s in range(n):
        L = lens[s]
        for h in range(HEADS):  # one head at a time: the 4096^2 score matrices of level 0 stay small
            cols = slice(h * d, (h + 1) * d)
            sc = q[s, :, cols] @ k[s, :L, cols].T / math.sqrt(d)
            p = (sc - sc.amax(-1, keepdim=True)).exp()
            p = p / p.sum(-1, keepdim=True)
            out[s, :, cols] = (r16(p) if rnd else p) @ v[s, :L, cols]
    return out


def spatial_transformer(W, name, x, context, lens, r: Rounding = EXACT, eps=1e-5):
    """x [n, C, H, W] (the values the block reads), context [n, Lmax, 768], lens [n]. -> (out [n, C, H, W], [y0, y1, y2, y3]):
    the residual stream [n*H*W, C] after proj_in, attn1, attn2 and the MLP."""
    t = f"{name}/transformer"
    n, c, h, w = x.shape
    act = lambda a, p: _round(a, "fp16") if p == 1 else a
    wgt = lambda a, p: _round(a, "fp16") if p <= 2 else a
    P = r.passes

    def ln_fold(y, ln, wmat, bias, p):
        """LayerNorm(y) @ wmat + bias with gamma folded into the weights and the normalisation applied after the product"""
        mu = y.mean(-1, keepdim=True)
        rs = 1.0 / (((y - mu) ** 2).mean(-1, keepdim=True) + eps).sqrt()
        out = rs * ((act(y, p) - mu) @ wgt(W[f"{t}/{ln}/weight"][:, None] * wmat, p)) + W[f"{t}/{ln}/bias"] @ wmat
        return out if bias is None else out + bias

    def lin(a, wname, p, residual):
        return residual + act(a, p) @ wgt(W[f"{wname}/weight"], p) + W[f"{wname}/bias"]

    g = F.group_norm(x, 32, W[f"{name}/norm/weight"], W[f"{name}/norm/bias"], eps)
    g = g.permute(0, 2, 3, 1).reshape(n * h * w, c)
    y0 = act(g, P) @ wgt(W[f"{name}/proj_in/weight"].reshape(c, c), P).T + W[f"{name}/proj_in/bias"]
    # self attention
    wqkv = torch.cat([W[f"{t}/attn1/{k}/weight"] for k in ("query", "key", "value")], 1)
    q, k, v = ln_fold(y0, "norm1", wqkv, None, P).reshape(n, h * w, 3, c).unbind(2)
    o = _attention(q, k, v, [h * w] * n, r.attention, r.qk_split).reshape(n * h * w, c)
    y1 = lin(o, f"{t}/attn1/out", P, y0)
    # cross attention: context K / V from a 3-pass product
    q = ln_fold(y1, "norm2", W[f"{t}/attn2/query/weight"], None, P).reshape(n, h * w, c)
    k, v = (context @ W[f"{t}/attn2/{kk}/weight"] for kk in ("key", "value"))
    o = _attention(q, k, v, lens, r.attention, r.qk_split).reshape(n * h * w, c)
    y2 = lin(o, f"{t}/attn2/out", P, y1)
    # GEGLU MLP
    hg = ln_fold(y2, "norm3", W[f"{t}/mlp/geglu/proj/weight"], W[f"{t}/mlp/geglu/proj/bias"], P)
    y3 = lin(hg[:, :4 * c] * gelu_erf(hg[:, 4 * c:]), f"{t}/mlp/lin", P, y2)
    # proj_out + the block input
    po = act(y3, P) @ wgt(W[f"{name}/proj_out/weight"].reshape(c, c), P).T + W[f"{name}/proj_out/bias"]
    out = x + po.reshape(n, h, w, c).permute(0, 3, 1, 2)
    return out, [y0, y1, y2, y3]
