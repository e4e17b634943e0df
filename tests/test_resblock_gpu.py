"""The ResBlock's GroupNorm, channel-concat and skip-conv paths against an fp64 reference of the same block.

Each case runs one UNet ResBlock (unet/mod.rs:712-734) or VAE ResnetBlock (autoencoder/mod.rs:513-528) through
sdb_test_resblock: the model's own packers, staging and launch heuristics, with the inputs staged the way the model's producers
leave them. The entry also reports what ran (GroupNorm path, skip form, per-GEMM tile / split-K choice), and every case asserts
it reached the path it claims, so a later heuristic change cannot route a case around its path unnoticed.

The reference (`ref_block`) is built from torch primitives in fp64. For 1- and 2-pass products it rounds the conv operands to
fp16 where the kernel does: 1 pass rounds the GroupNorm + SiLU outputs, the raw skip input and the weights; 2 passes the weights
only. 3 passes are compared with the exact fp64 block.

The inputs carry their own sensitivity: every image has its own scale and offset (statistics leaking between the two images of
an 8x8 tile show), every channel an offset of about 4 standard deviations (the sum-of-squares cancellation), and x1 a scale and
offset unlike x0's (mixing up the two sources of the concat moves the groups that straddle it)."""
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.sd_oracle import _round

pytestmark = pytest.mark.gpu

# relative L2 bars: 3-pass against the exact block, 1- and 2-pass against the operand-rounding reference
TOL_L2 = {1: 3e-4, 2: 3e-4, 3: 5e-5}
TOL_MAX3 = 2e-4  # 3-pass: max |out - ref| / max |ref|


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def split22(x):
    """hi + lo of the fp16 pair a producer's epilogue writes (what an identity 3-pass producer hands on)."""
    hi = x.astype(np.float16).astype(np.float32)
    return hi.astype(np.float64) + (x - hi).astype(np.float16).astype(np.float64)


def activation(rng, n, c, h, w, scale, centre):
    """per-image scale / offset, per-channel offset ~4 sigma around `centre`"""
    img_s = scale * (1.0 + 0.3 * np.arange(n))
    img_o = 0.5 * (-1.0) ** np.arange(n)
    ch = centre + 0.3 * rng.standard_normal(c)
    z = rng.standard_normal((n, c, h, w))
    return ((z + ch[None, :, None, None]) * img_s[:, None, None, None] + img_o[:, None, None, None]).astype(np.float32)


# name: n, C0, C1, Cout, H, W, skip, emb, passes, x0 with producer statistics, x1 with producer statistics, what it reaches
# (GroupNorm paths of norm1 / norm2 at the default options, split-K on conv1 / conv2, M-tile images per tile)
CASES = {
    "l0_320_fused": (2, 320, 0, 320, 64, 64, False, True, 3, False, True, dict(gn=("fused", "apply"))),
    "l1_320_640": (2, 320, 0, 640, 32, 32, True, True, 3, True, True, dict(gn=("apply", "apply"))),
    "l2_640_1280": (2, 640, 0, 1280, 16, 16, True, True, 1, True, True, dict(gn=("apply", "apply"))),
    "l3_1280_8x8": (2, 1280, 0, 1280, 8, 8, False, True, 1, True, True, dict(gn=("apply", "apply"), split=True, TN=2)),
    "l3_cat_n3": (3, 1280, 1280, 1280, 8, 8, True, True, 1, True, True, dict(gn=("apply", "apply"), split=True, TN=2)),
    "l2_cat_straddle": (2, 1280, 640, 1280, 16, 16, True, True, 1, True, True, dict(gn=("apply", "apply"), split=True)),
    "l1_cat_straddle": (2, 1280, 640, 640, 32, 32, True, True, 3, True, True, dict(gn=("apply", "apply"))),
    "l0_cat_straddle": (1, 640, 320, 320, 64, 64, True, True, 3, True, True, dict(gn=("apply", "apply"))),
    "l0_cat_conv_in": (2, 320, 320, 320, 64, 64, True, True, 3, True, False, dict(gn=("fused", "apply"))),
    "l1_cat_768px": (2, 1280, 640, 640, 24, 24, True, True, 3, True, True, dict(gn=("apply", "apply"))),
    "vae_512": (1, 512, 0, 512, 64, 64, False, False, 3, True, True, dict(gn=("apply", "apply"))),
    "vae_fold_nin": (1, 512, 0, 256, 96, 192, True, False, 1, True, True, dict(gn=("apply+fold", "apply+fold"))),
}
SKIP_CASES = [k for k, v in CASES.items() if v[6]]
TWO_PASS_CASES = ["l2_cat_straddle", "l0_cat_conv_in"]


def make_inputs(name):
    n, c0, c1, co, h, w, skip, emb, *_ = CASES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    cin = c0 + c1
    d = {}
    d["x0"] = activation(rng, n, c0, h, w, 1.0, 4.0)
    d["x1"] = activation(rng, n, c1, h, w, 2.5, -3.0) if c1 else None
    d["norm1"] = ((1 + 0.1 * rng.standard_normal(cin)).astype(np.float32), (0.1 * rng.standard_normal(cin)).astype(np.float32))
    d["conv1"] = ((rng.standard_normal((co, cin, 3, 3)) / np.sqrt(9 * cin)).astype(np.float32),
                  (0.1 * rng.standard_normal(co)).astype(np.float32))
    d["norm2"] = ((1 + 0.1 * rng.standard_normal(co)).astype(np.float32), (0.1 * rng.standard_normal(co)).astype(np.float32))
    d["conv2"] = ((rng.standard_normal((co, co, 3, 3)) / np.sqrt(9 * co)).astype(np.float32),
                  (0.1 * rng.standard_normal(co)).astype(np.float32))
    d["skip"] = ((rng.standard_normal((co, cin, 1, 1)) / np.sqrt(cin)).astype(np.float32),
                 (0.1 * rng.standard_normal(co)).astype(np.float32)) if skip else None
    # conv_in.bias + lin_embed(silu(emb)) of the UNet; the VAE block has none
    d["emb_bias"] = (0.5 * rng.standard_normal(co)).astype(np.float32) if emb else None
    return d


def block_input(name, d):
    """the values the block reads: hi + lo of the input behind a statistics-producing identity conv, else the fp32 tensor"""
    x0_stats, x1_stats = CASES[name][9], CASES[name][10]
    xs = [split22(d["x0"]) if x0_stats else d["x0"].astype(np.float64)]
    if d["x1"] is not None:
        xs.append(split22(d["x1"]) if x1_stats else d["x1"].astype(np.float64))
    return torch.from_numpy(np.concatenate(xs, axis=1))


def ref_block(x, d, passes):
    """fp64 ResBlock / ResnetBlock on the concatenated input x, operands rounded to fp16 where a `passes`-pass product does"""
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    act = (lambda v: _round(v, "fp16")) if passes == 1 else (lambda v: v)
    wgt = (lambda v: _round(v, "fp16")) if passes <= 2 else (lambda v: v)
    (g1, b1), (w1, cb1), (g2, b2), (w2, cb2) = d["norm1"], d["conv1"], d["norm2"], d["conv2"]
    h = F.silu(F.group_norm(x, 32, t(g1), t(b1), 1e-5))
    bias1 = t(d["emb_bias"]) if d["emb_bias"] is not None else t(cb1)
    h = F.conv2d(act(h), wgt(t(w1)), bias1, padding=1)
    h = F.silu(F.group_norm(h, 32, t(g2), t(b2), 1e-5))
    h = F.conv2d(act(h), wgt(t(w2)), t(cb2), padding=1)
    if d["skip"] is not None:
        return F.conv2d(act(x), wgt(t(d["skip"][0])), t(d["skip"][1])) + h
    return x + h


_CACHE = {}


def case_data(name, passes):
    """inputs and fp64 reference, computed once per (case, passes) for every option variant"""
    if name not in _CACHE:
        d = make_inputs(name)
        _CACHE[name] = (d, block_input(name, d), {})
    d, x, refs = _CACHE[name]
    if passes not in refs:
        with torch.no_grad():
            refs[passes] = ref_block(x, d, passes).numpy()
    return d, x, refs[passes]


def run(ctx, name, passes):
    d = make_inputs(name) if name not in _CACHE else _CACHE[name][0]
    x0_stats, x1_stats = CASES[name][9], CASES[name][10]
    return ctx.test_resblock(d["x0"], d["x1"], d["norm1"], d["conv1"], d["norm2"], d["conv2"], skip=d["skip"],
                             emb_bias=d["emb_bias"], passes=passes, x0_stats=x0_stats, x1_stats=x1_stats)


class Options:
    """set library options for one block, restore the defaults afterwards"""

    DEFAULTS = {"skip_merge": 1, "raw16": 1, "gn_epilogue": 1, "splitk": 1}

    def __init__(self, ctx, **kw):
        self.ctx, self.kw = ctx, kw

    def __enter__(self):
        for k, v in self.kw.items():
            self.ctx.set_option(k, v)

    def __exit__(self, *exc):
        for k in self.kw:
            self.ctx.set_option(k, self.DEFAULTS[k])


def check(ctx, name, passes, variant, **opts):
    d, x, ref = case_data(name, passes)
    with Options(ctx, **opts):
        out, out16, outn, tr = run(ctx, name, passes)
    e = rel(out, ref)
    emax = float(np.abs(out - ref).max() / np.abs(ref).max())
    # the output's own consumers: its fp16 copy and the GroupNorm staged from the statistics conv2 left, against fp64 of `out`
    gamma, beta = (torch.from_numpy(v.astype(np.float64)) for v in d["norm2"])
    refn = F.silu(F.group_norm(torch.from_numpy(out.astype(np.float64)), 32, gamma, beta, 1e-5)).numpy()
    en = rel(outn, refn)
    print(f"resblock {name} [{variant}] passes={passes}: rel L2 {e:.3e} max {emax:.3e} | GN(out) {en:.3e} | "
          f"gn {tr['gn']} skip {tr['skip']} gemms "
          + " ".join(f"{g['kind']}:BN{g['BN']}/s{g['split']}/{g['TN']}x{g['TH']}x{g['TW']}/xk{g['xk']}/a1_{g['a1']}" for g in tr["gemms"]))
    assert out.shape == ref.shape and np.isfinite(out).all()
    assert e < TOL_L2[passes], (name, variant, e)
    if passes == 3:
        assert emax < TOL_MAX3, (name, variant, emax)
    assert en < 2e-6, (name, variant, en)  # hi + lo of a GroupNorm whose statistics are fp64 folds of fp32 partials
    if opts.get("raw16", 1):
        assert np.array_equal(out16, split22(out).astype(np.float32)), "conv2's fp16 hi + lo copy is not the split of its fp32 output"
    else:
        assert not out16.any()
    return out, tr


def expect_trace(name, tr, opts):
    n, c0, c1, co, h, w, skip, emb, passes, x0s, x1s, exp = CASES[name]
    gn_epi = opts.get("gn_epilogue", 1)
    g1, g2 = exp["gn"] if gn_epi else ("fused", "fused")
    out_gn = ("apply+fold" if g2 == "apply+fold" else "apply") if gn_epi else "fused"
    assert tr["gn"] == [g1, g2, out_gn], (name, tr["gn"])
    if not skip:
        form = "none"
    elif opts.get("skip_merge", 1) and opts.get("raw16", 1):
        form = "merged"
    else:
        form = "separate"
    assert tr["skip"] == form, (name, tr["skip"])
    gemms = tr["gemms"]
    conv1, conv2 = gemms[0], gemms[-1]
    assert conv1["kind"] == 2 and conv2["kind"] == 2  # G_CONV3
    if form == "merged":
        assert conv2["xk"] == c0 + c1
    if form == "separate":
        sk = gemms[1]
        assert sk["kind"] == 1 and sk["xk"] == 0  # G_CONV1
        # the skip conv reads both sources directly when their fp16 copies exist, else one concatenated staging
        assert sk["a1"] == (c1 if opts.get("raw16", 1) else 0)
    if gn_epi:
        assert conv1["gn_slots"] > 0 and conv2["gn_slots"] > 0
    if exp.get("split") and opts.get("splitk", 1):
        assert conv1["split"] > 1 and conv2["split"] > 1, (name, conv1["split"], conv2["split"])
    if "TN" in exp:
        assert conv1["TN"] == exp["TN"] and conv2["TN"] == exp["TN"]


@pytest.mark.parametrize("name", list(CASES))
def test_resblock_default(ctx, name):
    passes = CASES[name][8]
    _, tr = check(ctx, name, passes, "default")
    expect_trace(name, tr, {})


@pytest.mark.parametrize("name", list(CASES))
def test_resblock_no_gn_epilogue(ctx, name):
    """every GroupNorm from the fused statistics + apply kernel (with two sources on the concat blocks)"""
    passes = CASES[name][8]
    _, tr = check(ctx, name, passes, "gn_epilogue=0", gn_epilogue=0)
    expect_trace(name, tr, {"gn_epilogue": 0})


@pytest.mark.parametrize("name", SKIP_CASES)
def test_resblock_separate_skip(ctx, name):
    """skip conv as its own GEMM (two-source A operand on the concat blocks), conv2 accumulating onto it in place"""
    passes = CASES[name][8]
    _, tr = check(ctx, name, passes, "skip_merge=0", skip_merge=0)
    expect_trace(name, tr, {"skip_merge": 0})


@pytest.mark.parametrize("name", SKIP_CASES)
def test_resblock_no_raw16(ctx, name):
    """no fp16 copies from the producers: the skip input is staged from fp32 as one concatenated operand"""
    passes = CASES[name][8]
    _, tr = check(ctx, name, passes, "raw16=0", raw16=0)
    expect_trace(name, tr, {"raw16": 0})


@pytest.mark.parametrize("name", TWO_PASS_CASES)
def test_resblock_two_pass(ctx, name):
    _, tr = check(ctx, name, 2, "2-pass")
    expect_trace(name, tr, {})


def test_resblock_unsplit_two_images_per_tile(ctx):
    """the 8x8 concat block without split-K: GroupNorm partials of tiles holding 2 images written by the plain epilogue, the
    second image of the last tile masked (n = 3)"""
    name = "l3_cat_n3"
    _, tr = check(ctx, name, CASES[name][8], "splitk=0", splitk=0)
    expect_trace(name, tr, {"splitk": 0})
    assert all(g["split"] == 1 for g in tr["gemms"])


def test_resblock_repeatable(ctx):
    """split-K tile tickets and GroupNorm rendezvous tickets come back clean: a second run is bit-identical"""
    name = "l3_cat_n3"
    passes = CASES[name][8]
    a = run(ctx, name, passes)
    b = run(ctx, name, passes)
    for u, v in zip(a[:3], b[:3]):
        assert np.array_equal(u, v)
    with Options(ctx, gn_epilogue=0):
        c = run(ctx, "l0_cat_conv_in", 3)
        e = run(ctx, "l0_cat_conv_in", 3)
    for u, v in zip(c[:3], e[:3]):
        assert np.array_equal(u, v)


# ---------------------------------------------------------------- GroupNorm of cat([x0, x1]) in isolation
# n, C0, C1, H, W: the decoder's concat widths (groups of 60 / 30 straddling the boundary at C = 1920 / 960), equal halves,
# a single source, the VAE's 256-channel halves, and maps with more than 128 producer slots per image (pre-fold); then single
# sources from 64 channels (groups of 2) to 1920 (groups of 60) and from 4x4 to 64x64 maps
GN_CAT = [(2, 1280, 640, 16, 16), (1, 640, 320, 32, 32), (2, 320, 320, 64, 64), (3, 1280, 1280, 8, 8), (2, 640, 0, 16, 16),
          (1, 256, 256, 32, 32), (1, 320, 320, 128, 160), (1, 256, 256, 96, 192),
          (2, 320, 0, 16, 16), (1, 64, 0, 8, 8), (2, 960, 0, 8, 8), (1, 128, 0, 64, 64), (1, 1920, 0, 4, 4)]
# mode 1 only: the identity producer's GEMM leaves no GroupNorm partials for a 64-wide tile (64 channels) or for tiles of more
# than 4 images (4x4 maps), so the staging takes the fused path there
GN_CAT_FUSED_ONLY = [(1, 64, 0, 8, 8), (1, 1920, 0, 4, 4)]


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("n,c0,c1,h,w,mode", [(*s, m) for s in GN_CAT for m in (1, 2) if m == 1 or s not in GN_CAT_FUSED_ONLY])
def test_groupnorm_cat(ctx, n, c0, c1, h, w, mode, silu):
    rng = np.random.default_rng(1000 * c0 + c1 + h)
    x0 = activation(rng, n, c0, h, w, 1.0, 4.0)
    x1 = activation(rng, n, c1, h, w, 2.5, -3.0) if c1 else None
    c = c0 + c1
    g = (1 + 0.1 * rng.standard_normal(c)).astype(np.float32); b = (0.1 * rng.standard_normal(c)).astype(np.float32)
    # mode 2 reads the producers' outputs: hi + lo of the inputs
    xs = [split22(x0) if mode == 2 else x0.astype(np.float64)]
    if x1 is not None:
        xs.append(split22(x1) if mode == 2 else x1.astype(np.float64))
    x = torch.from_numpy(np.concatenate(xs, axis=1))
    ref = F.group_norm(x, 32, torch.from_numpy(g).double(), torch.from_numpy(b).double(), 1e-5)
    if silu:
        ref = F.silu(ref)
    out, tr = ctx.test_groupnorm_cat(x0, x1, g, b, silu=silu, mode=mode)
    e = rel(out, ref.numpy())
    print(f"GN cat n={n} {c0}+{c1} {h}x{w} mode {mode} silu {silu}: {tr['gn']} rel L2 {e:.3e}")
    if mode == 1:
        assert tr["gn"] == ["fused"]
    if mode == 2:
        assert tr["gn"] == ["apply+fold" if h * w > 128 * 128 else "apply"]
    assert e < 5e-6
