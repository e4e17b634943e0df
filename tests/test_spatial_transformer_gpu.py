"""The UNet's SpatialTransformer against an fp64 reference of the same block, stage by stage.

Each case runs one of the model's own 16 SpatialTransformers through sdb_test_spatial_transformer: the weights finalize_weights
packed (the folded LayerNorms, head-padded q|k|v, cross-attention q, tile-interleaved GEGLU), the context K / V preparation of
the sampling entries with per-sample lengths, and the block's launch sequence unchanged. The entry hands back the residual
stream y after each stage and the LayerNorm row statistics the producers left, so a failure names the stage that broke, and a
trace of what ran, which every case checks against the paths it claims to reach.

The reference (tests/st_oracle.py) is fp64 on the weights read back from the context. It rounds to fp16 what the kernels read
as fp16: both operands of a 1-pass GEMM, P and V in the attention, q and k unless the attention takes their hi + lo pairs.

The weights of the blocks under test get trained-checkpoint-like statistics on top of the synthetic stream: LayerNorm and
GroupNorm gamma in [0.4, 1.6] and beta in [-0.4, 0.4], query / key weights x 1.7 (peaked softmax). The r sweep shifts the
proj_in bias so that every token row entering a LayerNorm has |mean| / std of about r: the folded LayerNorm forms the variance
as E[y^2] - mean^2 in fp32 and subtracts mean * colsum(W) from an fp32 accumulator, and both lose precision as r grows."""
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import st_oracle as S
from stable_diffusion_burn_b200 import synth

pytestmark = pytest.mark.gpu

# execution-order index -> (dump-dir name, width, pass count of its level)
BLOCKS = {0: ("unet/input_blocks/rt1/transformer", 320, 3), 2: ("unet/input_blocks/rt3/transformer", 640, 3),
          4: ("unet/input_blocks/rt5/transformer", 1280, 1), 6: ("unet/middle_block/transformer", 1280, 1)}
DPAD = {320: 48, 640: 80, 1280: 160}

# name: block index, H, W, n, context lengths, output with an fp16 copy (RT blocks) or without (the middle block)
CASES = {
    "l0": (0, 64, 64, 2, (77, 5), True),          # dpad 48, split q / k, 32 GroupNorm slots per image
    "l0_96x64": (0, 96, 64, 1, (77,), True),      # 768 px non-square
    "l1": (2, 32, 32, 2, (77, 1), True),          # dpad 80, split q / k
    "l1_48x48": (2, 48, 48, 2, (77, 13), True),   # 768 px: 18 slots
    "l2": (4, 16, 16, 2, (77, 13), True),
    "l2_24x24": (4, 24, 24, 2, (77, 13), True),   # 768 px: proj_out leaves no partials, the consumer's GroupNorm is fused
    "mid_n1": (6, 8, 8, 1, (77,), False),         # 64 rows: less than one tile
    "mid_n3": (6, 8, 8, 3, (77, 2, 40), False),   # two images per proj_out tile, the last tile half masked
    "mid_12x12": (6, 12, 12, 2, (77, 13), False),  # 144 rows: a partly masked second query tile; partials off
}
L01 = [k for k, v in CASES.items() if v[0] in (0, 2)]
L2MID = [k for k, v in CASES.items() if v[0] in (4, 6)]

# bars per (passes of the block's GEMMs, variant): 3x the worst value measured on an H100 SXM (80 GB, 700 W), rounded down.
#   y    relative L2 of the residual stream after proj_in, attn1, attn2, the MLP
#   add  relative L2 of what attn1, attn2, the MLP and proj_out add (y1 - y0, y2 - y1, y3 - y2, out - x): a row offset inflates
#        |y| and would dilute the y measure, not this one
#   out  relative L2 and max |out - ref| / max |ref| of the block output
# r = 4 keeps the bars of the default statistics (or its own where tighter); r = 16 has its own (DESIGN.md §2).
TOL = {
    (3, "default"): dict(y=(7.1e-6, 2.4e-4, 3.8e-4, 4.2e-4), add=(4.8e-4, 7.0e-4, 5.3e-4, 4.2e-4), out=(3.3e-4, 5.1e-4)),
    (3, "gn_epilogue=0"): dict(y=(7.1e-6, 2.4e-4, 3.8e-4, 4.3e-4), add=(4.8e-4, 7.0e-4, 5.3e-4, 4.3e-4), out=(3.3e-4, 5.1e-4)),
    (3, "attn_split=0"): dict(y=(7.1e-6, 2.7e-4, 5.3e-4, 5.9e-4), add=(5.2e-4, 1.0e-3, 7.4e-4, 5.9e-4), out=(4.6e-4, 8.0e-4)),
    (3, "precision=3"): dict(y=(1.4e-5, 3.6e-4, 6.8e-4, 7.4e-4), add=(6.5e-4, 1.4e-3, 9.5e-4, 7.4e-4), out=(6.1e-4, 1.0e-3)),
    (3, "r=4"): dict(y=(8.8e-7, 5.7e-5, 1.1e-4, 1.4e-4), add=(4.1e-4, 6.7e-4, 5.2e-4, 1.4e-4), out=(1.4e-4, 2.6e-4)),
    (3, "r=16"): dict(y=(2.8e-7, 1.7e-5, 3.3e-5, 4.2e-5), add=(5.0e-4, 7.0e-4, 5.7e-4, 4.3e-5), out=(4.2e-5, 9.3e-5)),
    (1, "default"): dict(y=(1.7e-5, 6.8e-4, 1.1e-3, 1.4e-3), add=(1.1e-3, 2.4e-3, 2.2e-3, 1.6e-3), out=(1.4e-3, 1.5e-3)),
    (1, "gn_epilogue=0"): dict(y=(1.8e-5, 6.9e-4, 1.1e-3, 1.4e-3), add=(1.1e-3, 2.4e-3, 2.2e-3, 1.6e-3), out=(1.3e-3, 1.4e-3)),
    (1, "precision=1"): dict(y=(1.5e-5, 3.8e-4, 1.1e-3, 1.4e-3), add=(7.7e-4, 2.3e-3, 2.1e-3, 1.6e-3), out=(1.3e-3, 1.5e-3)),
    (1, "r=4"): dict(y=(3.1e-6, 1.9e-4, 5.2e-4, 8.6e-4), add=(1.1e-3, 2.4e-3, 2.2e-3, 1.1e-3), out=(1.1e-3, 1.3e-3)),
    (1, "r=16"): dict(y=(8.2e-7, 6.6e-5, 2.8e-4, 6.2e-4), add=(1.5e-3, 7.5e-3, 1.2e-2, 1.0e-3), out=(1.0e-3, 1.6e-3)),
}
TOL_LN = 7e-7  # LayerNorm row sums against fp64 sums of the y they describe
OPTION_DEFAULTS = {"precision": 0, "attn_split": 1, "gn_epilogue": 1}


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def split22(x):
    hi = x.astype(np.float16).astype(np.float32)
    return hi.astype(np.float64) + (x - hi).astype(np.float16).astype(np.float64)


@pytest.fixture(scope="module")
def blocks(ctx):
    """synthetic weights with controlled statistics on the blocks under test; fp64 copies of them as the context holds them"""
    ctx.init_synthetic(0)
    shapes = dict(ctx.tensor_list())
    get = lambda name: ctx.get_tensor(name, shapes[name])
    rng = np.random.default_rng(2024)
    for idx, (name, c, _) in BLOCKS.items():
        t = f"{name}/transformer"
        for norm in (f"{name}/norm", f"{t}/norm1", f"{t}/norm2", f"{t}/norm3"):
            ctx.set_tensor(f"{norm}/weight", rng.uniform(0.4, 1.6, c).astype(np.float32))
            ctx.set_tensor(f"{norm}/bias", rng.uniform(-0.4, 0.4, c).astype(np.float32))
        for a in ("attn1", "attn2"):
            for k in ("query", "key"):
                ctx.set_tensor(f"{t}/{a}/{k}/weight", 1.7 * get(f"{t}/{a}/{k}/weight"))
    ctx.finalize_weights()
    weights = {idx: S.block_weights(ctx.get_tensor, name, c) for idx, (name, c, _) in BLOCKS.items()}
    yield weights
    for k, v in OPTION_DEFAULTS.items():
        ctx.set_option(k, v)
    ctx.init_synthetic(0)
    ctx.finalize_weights()


def case_inputs(name):
    idx, h, w, n, lens, _ = CASES[name]
    c = BLOCKS[idx][1]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    # every image its own scale, every channel its own offset: GroupNorm statistics leaking between images of a tile show
    img_s = 1.0 + 0.3 * np.arange(n)
    x = (rng.standard_normal((n, c, h, w)) + 0.5 * rng.standard_normal((1, c, 1, 1))) * img_s[:, None, None, None]
    ctxt = synth.make_context(n, max(lens), seed=zlib.crc32(name.encode()) & 0xFFFF)  # rows past a length hold values
    return x.astype(np.float32), ctxt, lens


def effective(idx, opts):
    """(passes of the block GEMMs, split q / k) the options select on block `idx`"""
    level_p = BLOCKS[idx][2]
    prec = opts.get("precision", 0)
    P = prec or level_p
    qk = (level_p >= 2 or prec >= 2) and opts.get("attn_split", 1) == 1 and DPAD[BLOCKS[idx][1]] in (48, 80)
    return P, qk


_REF = {}


def reference(W, name, r_key, x, ctxt, lens, rnd):
    key = (name, r_key, rnd)
    if key not in _REF:
        idx = CASES[name][0]
        with torch.no_grad():
            out, ys = S.spatial_transformer(W, BLOCKS[idx][0], torch.from_numpy(split22(x)), torch.from_numpy(ctxt.astype(np.float64)),
                                            lens, rnd)
        _REF[key] = (out.numpy(), [y.numpy() for y in ys])
    return _REF[key]


def expect_trace(name, tr, opts):
    idx, h, w, n, lens, _ = CASES[name]
    c = BLOCKS[idx][1]
    hw, dpad = h * w, DPAD[c]
    P, qk = effective(idx, opts)
    gn_epi = opts.get("gn_epilogue", 1)
    # proj_out's GroupNorm partials over flattened token rows: whole 128-row tiles of one image, or 2 / 4 images per tile
    slots = (hw // 128 if hw % 128 == 0 else (1 if 128 % hw == 0 and hw >= 32 else 0)) if gn_epi else 0
    g = tr["gemms"]
    assert len(g) == 8, g
    roles = [{"lns"}, {"lnc"}, {"res16", "lns"}, {"lnc"}, {"res16", "lns"}, {"lnc", "geglu"}, {"res16"},
             {"res32"} | ({"gn"} if slots else set())]
    assert [x["epi"] for x in g] == roles, [x["epi"] for x in g]
    assert [x["passes"] for x in g] == [P] * 8
    assert [x["N"] for x in g] == [c, 3 * 8 * dpad, c, 8 * dpad, c, 8 * c, c, c]
    assert g[7]["gn_slots"] == slots, (g[7]["gn_slots"], slots)
    lpad = -(-max(lens) // 32) * 32
    assert tr["attn"] == [dict(dpad=dpad, Nq=hw, Nk=hw, qk3=int(qk), kvlen=0),
                          dict(dpad=dpad, Nq=hw, Nk=lpad, qk3=int(qk), kvlen=1)], tr["attn"]
    assert tr["gn"] == ["apply" if gn_epi else "fused", "apply" if slots else "fused"], tr["gn"]


class Options:
    def __init__(self, ctx, **kw):
        self.ctx, self.kw = ctx, kw

    def __enter__(self):
        for k, v in self.kw.items():
            self.ctx.set_option(k, v)

    def __exit__(self, *exc):
        for k in self.kw:
            self.ctx.set_option(k, OPTION_DEFAULTS[k])


def check(ctx, W, name, variant, r_key=0, **opts):
    idx, h, w, n, lens, act16 = CASES[name]
    c = BLOCKS[idx][1]
    P, qk = effective(idx, opts)
    x, ctxt, lens = case_inputs(name)
    with Options(ctx, **opts):
        res = ctx.test_spatial_transformer(idx, x, ctxt, lens, act16=act16)
    ref, ys = reference(W, name, r_key, x, ctxt, lens, S.Rounding.of(P, qk))
    out = res["out"]
    e = rel(out, ref)
    emax = float(np.abs(out - ref).max() / np.abs(ref).max())
    ey = [rel(res["y"][i], ys[i]) for i in range(4)]
    xs = split22(x)
    ed = [rel(res["y"][i] - res["y"][i - 1], ys[i] - ys[i - 1]) for i in (1, 2, 3)] + [rel(out - xs, ref - xs)]
    # LayerNorm statistics against fp64 row sums of the y tap they describe (norm1: after proj_in, norm2: attn1, norm3: attn2)
    eln = []
    for i in range(3):
        y = res["y"][i].astype(np.float64)
        s1, s2 = y.sum(1), (y * y).sum(1)
        k1, k2 = res["ln"][i, :, 0].astype(np.float64), res["ln"][i, :, 1].astype(np.float64)
        eln.append(max(float(np.max(np.abs(k1 - s1) / np.sqrt(c * s2))), float(np.max(np.abs(k2 - s2) / s2))))
    # |mean| / std of the rows entering the LayerNorms (median over rows, worst LayerNorm)
    mus = max(float(np.median(np.abs(y.mean(1)) / y.std(1))) for y in ys[:3])
    gamma, beta = (torch.from_numpy(v.numpy().astype(np.float64)) for v in (W[f"{BLOCKS[idx][0]}/norm/weight"],
                                                                                W[f"{BLOCKS[idx][0]}/norm/bias"]))
    refn = F.silu(F.group_norm(torch.from_numpy(out.astype(np.float64)), 32, gamma, beta, 1e-5)).numpy()
    en = rel(res["out_norm"], refn)
    print(f"st {name} [{variant}] P={P} qk3={int(qk)} |mu|/sd {mus:.2f}: out rel L2 {e:.3e} max {emax:.3e} | "
          f"y proj_in {ey[0]:.3e} attn1 {ey[1]:.3e} attn2 {ey[2]:.3e} mlp {ey[3]:.3e} | added attn1 {ed[0]:.3e} "
          f"attn2 {ed[1]:.3e} mlp {ed[2]:.3e} proj_out {ed[3]:.3e} | LN sums {max(eln):.2e} | GN(out) {en:.2e}")
    tol = TOL[(P, variant)]
    assert np.isfinite(out).all() and out.shape == ref.shape
    for stage, v, bar in zip(("proj_in", "attn1", "attn2", "mlp"), ey, tol["y"]):
        assert v < bar, (name, variant, f"y after {stage}", v)
    for stage, v, bar in zip(("attn1", "attn2", "mlp", "proj_out"), ed, tol["add"]):
        assert v < bar, (name, variant, f"what {stage} adds", v)
    assert e < tol["out"][0] and emax < tol["out"][1], (name, variant, e, emax)
    for i, v in enumerate(eln):
        assert v < TOL_LN, (name, variant, f"norm{i + 1} statistics", v)
    assert en < 2e-6, (name, variant, en)
    if act16:
        assert np.array_equal(res["out16"], split22(out).astype(np.float32)), "the output's fp16 hi + lo copy is not the split of out"
    else:
        assert not res["out16"].any()
    expect_trace(name, res["trace"], opts)
    return res


@pytest.mark.parametrize("name", list(CASES))
def test_spatial_transformer_default(ctx, blocks, name):
    check(ctx, blocks[CASES[name][0]], name, "default")


@pytest.mark.parametrize("name", L01)
def test_spatial_transformer_single_fp16_qk(ctx, blocks, name):
    """levels 0-1 with the attention on single fp16 q / k (the 1 x 1 logits product)"""
    check(ctx, blocks[CASES[name][0]], name, "attn_split=0", attn_split=0)


@pytest.mark.parametrize("name", L2MID)
def test_spatial_transformer_precision3(ctx, blocks, name):
    """3-pass GEMMs on the single-pass levels; q / k stay single fp16 at dpad 160"""
    check(ctx, blocks[CASES[name][0]], name, "precision=3", precision=3)


@pytest.mark.parametrize("name", ["l0", "l0_96x64"])
def test_spatial_transformer_precision1(ctx, blocks, name):
    """1-pass GEMMs on level 0: the folded consumers read fp16 y and use the hi column sums; q / k keep their hi + lo pairs"""
    check(ctx, blocks[CASES[name][0]], name, "precision=1", precision=1)


@pytest.mark.parametrize("name", list(CASES))
def test_spatial_transformer_no_gn_epilogue(ctx, blocks, name):
    check(ctx, blocks[CASES[name][0]], name, "gn_epilogue=0", gn_epilogue=0)


@pytest.mark.parametrize("r", [4, 16])
@pytest.mark.parametrize("name", ["l0", "l2"])
def test_spatial_transformer_row_offset(ctx, blocks, name, r):
    """token rows with |mean| / std ~ r at every LayerNorm: the cancellation edge of the folded LayerNorm (r = 0 is the
    default case)"""
    idx = CASES[name][0]
    bname, c, _ = BLOCKS[idx]
    W = dict(blocks[idx])
    x, ctxt, lens = case_inputs(name)
    # y0 rows of this input without the shift: their median std sets the offset
    with torch.no_grad():
        _, ys = S.spatial_transformer(W, bname, torch.from_numpy(split22(x)), torch.from_numpy(ctxt.astype(np.float64)), lens)
    sd = float(np.median(ys[0].std(1).numpy()))
    key = f"{bname}/proj_in/bias"
    b0 = W[key].numpy().astype(np.float32)
    b = (b0 + np.float32(r * sd)).astype(np.float32)
    W[key] = torch.from_numpy(b.astype(np.float64))
    ctx.set_tensor(key, b)
    ctx.finalize_weights()
    try:
        check(ctx, W, name, f"r={r}", r_key=r)
    finally:
        ctx.set_tensor(key, b0)
        ctx.finalize_weights()


@pytest.mark.parametrize("name", ["l0", "mid_n3"])
def test_spatial_transformer_repeatable(ctx, blocks, name):
    """GroupNorm and split-K tickets come back clean, nothing reads stale arena contents: a second run is bit-identical"""
    idx, *_, act16 = CASES[name]
    x, ctxt, lens = case_inputs(name)
    a = ctx.test_spatial_transformer(idx, x, ctxt, lens, act16=act16)
    b = ctx.test_spatial_transformer(idx, x, ctxt, lens, act16=act16)
    for k in ("out", "out16", "out_norm", "y", "ln"):
        assert np.array_equal(a[k], b[k]), k


def test_spatial_transformer_rejects_bad_arguments(ctx, blocks):
    from stable_diffusion_burn_b200._lib import SdbError
    x = np.zeros((1, 320, 8, 8), np.float32)
    cx = np.zeros((1, 5, 768), np.float32)
    with pytest.raises(SdbError, match="index"):
        ctx.test_spatial_transformer(16, x, cx, [5])
    with pytest.raises(SdbError, match="channel count"):
        ctx.test_spatial_transformer(2, x, cx, [5])
    with pytest.raises(SdbError, match="lengths"):
        ctx.test_spatial_transformer(0, x, cx, [6])
    with pytest.raises(SdbError, match="multiple of 8"):
        ctx.test_spatial_transformer(0, np.zeros((1, 320, 3, 3), np.float32), cx, [5])
