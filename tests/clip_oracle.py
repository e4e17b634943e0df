"""fp64 reference of one CLIP text-encoder block (clip/mod.rs:109-115, attention :158-180 with the causal mask of
src/backend.rs:130-139, MLP with QuickGELU :204-227) in the form the CUDA path computes it, for tests/test_clip_blocks_gpu.py.

The block is restated from torch primitives with its intermediate values exposed: LN1, q, k, V, the attention output, x after
the attention, LN2, h = QuickGELU(fc1) and the block output. The value bias can be folded into the out-projection bias as
finalize_weights packs it (b_out' = b_out + b_v W_out, exact because every row of P sums to one) or added to V as the oracle does.

`Rounding` names which operands are rounded to fp16 (the oracle's `_round`) the way the kernels consume them:
  * the q | k GEMM and the V^T GEMM write single fp16 values: q, k and V are always rounded;
  * the attention reads P as fp16 (the kernel rounds P before dividing by the row sum, against a running maximum: the same
    relative rounding, not the same bits);
  * a 1-pass GEMM reads fp16 values of both operands (activation and weight); a 3-pass GEMM reads hi + lo pairs of both
    (22 bits each): exact here.
`EXACT` (all off) is the plain fp64 block: tests/test_clip_ref_cpu.py shows that it chains to the oracle's clip_forward."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from oracle.sd_oracle import _round

D, HEADS, LAYERS = 768, 12, 12


@dataclass(frozen=True)
class Rounding:
    passes: int = 3          # passes of the block's GEMMs
    kernel: bool = False     # fp16 q, k, V and P, as the kernels hold them

    @staticmethod
    def of(passes):
        return Rounding(passes, True)


EXACT = Rounding()


def block_names(i):
    b = f"clip/blocks/{i}"
    shapes = {}
    for ln in ("attn_ln", "mlp_ln"):
        shapes[f"{b}/{ln}/weight"] = shapes[f"{b}/{ln}/bias"] = (D,)
    for lin, (fi, fo) in {"attn/query": (D, D), "attn/key": (D, D), "attn/value": (D, D), "attn/out": (D, D),
                          "mlp/fc1": (D, 4 * D), "mlp/fc2": (4 * D, D)}.items():
        shapes[f"{b}/{lin}/weight"] = (fi, fo)  # dump-dir Linear: [in, out]
        shapes[f"{b}/{lin}/bias"] = (fo,)
    return shapes


def encoder_names():
    """every CLIP tensor except the two embedding tables"""
    shapes = {"clip/layer_norm/weight": (D,), "clip/layer_norm/bias": (D,)}
    for i in range(LAYERS):
        shapes.update(block_names(i))
    return shapes


def weights(get, shapes):
    """fp64 tensors; get(name, shape) -> array"""
    return {k: torch.from_numpy(np.asarray(get(k, s), np.float64)) for k, s in shapes.items()}


def layer_norm(x, g, b, eps=1e-5):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / (var + eps).sqrt() * g + b


def quick_gelu(h):
    return h * torch.sigmoid(1.702 * h)


def block(W, i, x, rnd=EXACT, fold_value_bias=True):
    """x [n, L, 768] fp64 -> dict of the block's intermediate values (names of _lib.Context.CLIP_TAPS) and `out`"""
    b = f"clip/blocks/{i}"
    n, L, _ = x.shape
    g16 = (lambda t: _round(t, "fp16")) if rnd.passes == 1 else (lambda t: t)  # a GEMM operand
    k16 = (lambda t: _round(t, "fp16")) if rnd.kernel else (lambda t: t)       # a kernel's fp16 intermediate
    lin = lambda a, name, bias=True: g16(a) @ g16(W[f"{b}/{name}/weight"]) + (W[f"{b}/{name}/bias"] if bias else 0)
    t = {}
    t["ln1"] = layer_norm(x, W[f"{b}/attn_ln/weight"], W[f"{b}/attn_ln/bias"])
    t["q"] = k16(lin(t["ln1"], "attn/query"))
    t["k"] = k16(lin(t["ln1"], "attn/key"))
    t["v"] = k16(lin(t["ln1"], "attn/value", bias=not fold_value_bias))
    hd = D // HEADS
    split = lambda a: a.reshape(n, L, HEADS, hd).transpose(1, 2)
    s = split(t["q"]) @ split(t["k"]).transpose(-1, -2) / np.sqrt(hd)
    s = s + torch.full((L, L), float("-inf"), dtype=s.dtype).triu(1)
    p = torch.softmax(s, dim=-1)
    t["o"] = (k16(p) @ split(t["v"])).transpose(1, 2).reshape(n, L, D)
    bias_out = W[f"{b}/attn/out/bias"] + (W[f"{b}/attn/value/bias"] @ W[f"{b}/attn/out/weight"] if fold_value_bias else 0)
    t["x_attn"] = x + g16(t["o"]) @ g16(W[f"{b}/attn/out/weight"]) + bias_out
    t["ln2"] = layer_norm(t["x_attn"], W[f"{b}/mlp_ln/weight"], W[f"{b}/mlp_ln/bias"])
    t["h"] = quick_gelu(lin(t["ln2"], "mlp/fc1"))
    t["out"] = t["x_attn"] + lin(t["h"], "mlp/fc2")
    return t


def final_layer_norm(W, x):
    return layer_norm(x, W["clip/layer_norm/weight"], W["clip/layer_norm/bias"])


def embed(tok_emb, pos_emb, tokens):
    """tokens int64 [n, L] -> x [n, L, 768] (clip/mod.rs:62-68)"""
    return tok_emb[tokens] + pos_emb[: tokens.shape[1]].unsqueeze(0)
