"""The autoencoder's stages, and the two CUDA-core convs the UNet shares with it, against fp64 references of the same operations.

Each case runs one stage through sdb_test_vae_stage: the context's own finalized weights and the launch code the model runs
(decoder conv_in with post_quant_conv and the pre-scale folded in, the 1-head mid attention of the decoder and the encoder, the
fused GroupNorm + SiLU + small-Cout conv_out of the decoder, UNet and encoder, the encoder's quant slice, the Cin = 4 / 8 / 9
conv_in kernels and the encoder's bottom/right-padded stride-2 downsamplers). The entry returns what ran, and every case asserts
from that trace that it reached the kernel variant, GroupNorm path or softmax instance it is there for.

The references are fp64 torch built from oracle/sd_oracle.py on the weights read back from the context. Where a product is
single-pass (precision = 1) they round its operands to fp16 as the kernels read them; the 3-pass products read hi + lo pairs (22
bits) and are taken as exact. The attention reference adds the v bias after P.V, as the kernel does
(tests/test_vae_stages_ref_cpu.py shows that this is the oracle's block).

The blocks under test get trained-checkpoint-like statistics on top of the synthetic stream: GroupNorm gamma in [0.4, 1.6] and
beta in [-0.4, 0.4], query / key weights x 1.7. Inputs give every image its own scale and every channel its own offset, so
GroupNorm statistics that leak between the images of a launch show; the r8 inputs have |mean| / std of about 8 in every group.

Bars: 3x the worst value measured on an H100 80GB HBM3 at a 700 W power limit, rounded up (see TOL)."""
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sd_oracle as O

pytestmark = pytest.mark.gpu

DEC, ENC = "autoencoder/decoder", "autoencoder/encoder"
ATTN = {"dec_attn": f"{DEC}/mid/attn", "enc_attn": f"{ENC}/mid/attn"}
ATTN_NEXT = {"dec_attn": f"{DEC}/mid/block_2/norm1", "enc_attn": f"{ENC}/mid/block_2/norm1"}
OUT = {"dec_out": (f"{DEC}/norm_out", f"{DEC}/conv_out", 128, 3), "unet_out": ("unet/norm_out", "unet/conv_out", 320, 4),
       "enc_out": (f"{ENC}/norm_out", f"{ENC}/conv_out", 512, 8)}
DOWN = {i: (f"{ENC}/blocks/{i}/downsampler/conv", f"{ENC}/blocks/{i + 1}/res1/norm1", c) for i, c in enumerate((128, 256, 512))}
KS_SMALL = {128: 4, 320: 5, 512: 4}  # channel groups of the small-image variant
PRE_SCALE = float(np.float32(1.0 / 0.18215))  # latent_to_image's pre-scale, rounded to f32 as the entry passes it

# Bars: 3x the worst value measured on an H100 80GB HBM3 (700 W power limit), rounded up; the worst measured value follows each.
#   attention: relative L2 of out - x (what the block adds; also per sample), of the attention output o before proj_out, and
#              max |out - ref| / max |ref|
#   conv:      relative L2 (also per image) and max |err| / max |ref| over every pixel
TOL = {
    ("attn", 3): dict(add=1.7e-4, o=1.6e-4, max=1.0e-4),     # 5.35e-5 / 5.25e-5 / 3.31e-5 (96x96)
    ("attn", 1): dict(add=9.0e-4, o=8.4e-4, max=2.1e-3),     # 2.99e-4 (a peaked sample) / 2.79e-4 / 6.78e-4 (peaked)
    "small_cout": dict(rel=3.9e-6, max=8.6e-6),              # 1.27e-6 / 2.84e-6 (encoder, large variant)
    "small_cout_r8": dict(rel=2.1e-5, max=1.7e-5),           # 6.69e-6 / 5.35e-6 (encoder): |mean| / std ~ 8
    "conv_in": dict(rel=5.3e-7, max=1.2e-6),                 # 1.74e-7 / 3.72e-7 (9-channel conv_in)
    ("down", 3): dict(rel=1.2e-5, max=1.3e-5),               # 3.92e-6 / 4.03e-6 (downsampler 0)
    ("down", 1): dict(rel=4.0e-6, max=4.9e-6),               # 1.32e-6 / 1.62e-6 (downsampler 0)
    "quant": dict(rel=2.0e-7, max=2.6e-7),                   # 6.36e-8 / 8.63e-8 (strided, scaled)
}
TOL_GN = 5.4e-6  # the next ResnetBlock's norm1 operand against fp64 GroupNorm of the stage's output: 1.78e-6 (r = 8)


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def relmax(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def split22(x):
    """hi + lo of x as the fp16 pair a 3-pass producer hands on (the values a stage with producer statistics sees)"""
    hi = x.astype(np.float16).astype(np.float32)
    return hi.astype(np.float64) + (x - hi).astype(np.float16).astype(np.float64)


def r16(a, on=True):
    return O._round(a, "fp16") if on else a


def activation(name, n, c, h, w, r=0.0):
    """every image its own scale, every channel its own offset; r > 0: every group's |mean| / std is about r"""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    img_s = (1.0 + 0.3 * np.arange(n))[:, None, None, None]
    x = rng.standard_normal((n, c, h, w)) + 0.5 * rng.standard_normal((1, c, 1, 1))
    if r:
        x = x + r
    return (x * img_s + 0.2 * np.arange(n)[:, None, None, None]).astype(np.float32)


# ------------------------------------------------------------------------------------------------ fp64 references
def ref_attention(P, name, x, rnd=False, rows=None):
    """conv_self_attention_block (autoencoder/mod.rs:562-608, 1 head, d = C) as the CUDA path computes it: q, k and V^T (no bias)
    from the GroupNorm'd input, P = softmax(q k^T / sqrt(C)), o = P V + b_v, out = x + proj_out(o). rnd: every product reads fp16
    operands and writes fp16 results, as at precision = 1. rows: the query rows to compute (attention and proj_out are
    row-independent once K and V exist). -> (out [n, C, rows], o [n, C, rows], P [n, rows, HW])"""
    n, c, hh, ww = x.shape
    hw = hh * ww
    rows = slice(None) if rows is None else rows
    h = r16(O.group_norm(P, f"{name}/norm", x), rnd).reshape(n, c, hw).transpose(1, 2)
    wt = lambda k: r16(P(f"{name}/{k}/weight").reshape(c, c), rnd)
    q = r16(h[:, rows] @ wt("q").T + P(f"{name}/q/bias"), rnd)
    k = r16(h @ wt("k").T + P(f"{name}/k/bias"), rnd)
    v = r16(h @ wt("v").T, rnd)
    s = q @ k.transpose(1, 2) / math.sqrt(c)
    p = torch.softmax(s, -1)
    o = r16(r16(p, rnd) @ v + P(f"{name}/v/bias"), rnd)
    po = o @ wt("proj_out").T + P(f"{name}/proj_out/bias")
    return x.reshape(n, c, hw)[:, :, rows] + po.transpose(1, 2), o.transpose(1, 2), p


def ref_norm_conv(P, norm, conv, x):
    return O.conv2d(P, conv, O.silu(O.group_norm(P, norm, x)), padding=1)


def ref_dec_in(P, lat, pre_scale):
    return O.conv2d(P, f"{DEC}/conv_in", O.conv2d(P, "autoencoder/post_quant_conv", lat * pre_scale), padding=1)


def ref_down(P, conv, x, rnd=False):
    """the bottom/right-padded stride-2 conv; oracle.padded_conv2d_s2 is tied to this form by tests/test_vae_encoder.py"""
    return F.conv2d(F.pad(r16(x, rnd), (0, 1, 0, 1)), r16(P(f"{conv}/weight"), rnd), P(f"{conv}/bias"), stride=2)


def ref_quant(P, y8, scale=1.0):
    return O.conv2d(P, "autoencoder/quant_conv", y8)[:, :4] * scale


def ref_gn_silu(P, norm, y):
    return O.silu(O.group_norm(P, norm, torch.from_numpy(y.astype(np.float64)))).numpy()


# ------------------------------------------------------------------------------------------------ fixture
NORMS = [f"{ATTN['dec_attn']}/norm", f"{ATTN['enc_attn']}/norm", f"{DEC}/norm_out", f"{ENC}/norm_out", "unet/norm_out"]
QK = [f"{a}/{k}/weight" for a in ATTN.values() for k in ("q", "k")]


def trained_like(ctx, get, set_):
    rng = np.random.default_rng(2025)
    shapes = dict(ctx.tensor_list())
    for norm in NORMS:
        c = shapes[f"{norm}/weight"][0]
        set_(f"{norm}/weight", rng.uniform(0.4, 1.6, c).astype(np.float32))
        set_(f"{norm}/bias", rng.uniform(-0.4, 0.4, c).astype(np.float32))
    for name in QK:
        set_(name, (1.7 * get(name)).astype(np.float32))


def params(ctx, prefixes):
    return O.Params({k: ctx.get_tensor(k, s) for k, s in ctx.tensor_list() if k.startswith(tuple(prefixes))}, dtype=torch.float64)


@pytest.fixture(scope="module")
def vae(ctx):
    ctx.init_synthetic(0)
    shapes = dict(ctx.tensor_list())
    trained_like(ctx, lambda k: ctx.get_tensor(k, shapes[k]), ctx.set_tensor)
    ctx.finalize_weights()
    P = params(ctx, ("autoencoder/", "unet/norm_out", "unet/conv_out", "unet/input_blocks/conv/"))
    torch.set_num_threads(max(1, torch.get_num_threads()))
    yield P
    for k in ("precision",):
        ctx.set_option(k, 0)
    ctx.init_synthetic(0)
    ctx.finalize_weights()


class Precision:
    def __init__(self, ctx, p):
        self.ctx, self.p = ctx, p

    def __enter__(self):
        self.ctx.set_option("precision", self.p)

    def __exit__(self, *exc):
        self.ctx.set_option("precision", 0)


# ------------------------------------------------------------------------------------------------ attention
# name: H, W, n, the query-row stride of the reference
ATTN_CASES = {
    "hw64_n3": (8, 8, 3, 1),       # two images per proj_out tile, the last tile half masked
    "hw64_n7": (8, 8, 7, 1),       # 18 GEMMs and 7 softmax launches in one call, each with its own trace record
    "16x16_n4": (16, 16, 4, 1),    # a full decode chunk: samples 1-3 of the per-sample loop
    "12x16": (12, 16, 2, 1),       # HW = 192: 1.5 proj_out tiles per image, which leaves no partials (the consumer's GroupNorm
                                   # runs fused); H*W must be a multiple of 64 (P is the P.V product's 64-channel operand)
    "64x64": (64, 64, 1, 1),       # HW = 4096, the top of the PER = 16 softmax
    "65x64": (65, 64, 1, 3),       # HW = 4160, the bottom of PER = 36
    "96x96": (96, 96, 1, 37),      # HW = 9216, the limit
}


def expect_attention_trace(tr, h, w, n, passes, stats):
    hw = h * w
    g = tr["gemms"]
    assert len(g) == 3 + 2 * n + 1, len(g)
    assert [x["kind"] for x in g] == [1, 1, 0] + [0, 0] * n + [0]
    assert all(x["passes"] == passes for x in g), [x["passes"] for x in g]
    # proj_out's GroupNorm partials: whole 128-row tiles of one image, or 2 / 4 images per tile
    slots = hw // 128 if hw % 128 == 0 else (1 if 128 % hw == 0 and hw >= 32 else 0)
    assert g[-1]["gn_slots"] == slots and ("gn" in g[-1]["epi"]) == (slots > 0) and "res32" in g[-1]["epi"], g[-1]
    assert tr["softmax"] == [16 if hw <= 4096 else 36] * n, tr["softmax"]
    assert tr["gn"][1] == ("apply" if slots else "fused"), tr["gn"]
    if not stats:
        assert tr["gn"][0] == "fused", tr["gn"]
    return slots


_REF = {}


def attn_check(ctx, P, stage, case, passes, variant="default", r=0.0, x=None, key=None):
    h, w, n, stride = ATTN_CASES[case]
    hw = h * w
    if x is None:
        x = activation(f"{stage}/{case}/{r}", n, 512, h, w, r)
    with Precision(ctx, 1 if passes == 1 else 0):
        res = ctx.test_vae_stage(stage, x, stats=True)
    rows = slice(0, hw, stride)
    k = (stage, case, passes, r, key)
    if k not in _REF:
        with torch.no_grad():
            out, o, p = ref_attention(P, ATTN[stage], torch.from_numpy(split22(x)), passes == 1, rows)
        _REF[k] = (out.numpy(), o.numpy(), float(p.amax(-1).median()), float((p < 2.0 ** -24).double().mean()))
    ref, ref_o, pmax, under = _REF[k]
    xs = split22(x).reshape(n, 512, hw)[:, :, rows]
    out = res["out"].reshape(n, 512, hw)[:, :, rows]
    o = res["tap"].reshape(n, 512, hw)[:, :, rows]
    e_add, e_o, e_max = rel(out - xs, ref - xs), rel(o, ref_o), relmax(out, ref)
    per_sample = [rel(out[s] - xs[s], ref[s] - xs[s]) for s in range(n)]
    slots = expect_attention_trace(res["trace"], h, w, n, passes, True)
    en = rel(res["out_norm"], ref_gn_silu(P, ATTN_NEXT[stage], res["out"]))
    print(f"vae {stage} {case} [{variant}] P={passes} softmax PER {res['trace']['softmax'][0]} proj_out slots {slots} "
          f"gn {res['trace']['gn']} median max P {pmax:.3f} P<2^-24 {under:.2f}: added rel L2 {e_add:.3e} "
          f"(per sample {' '.join(f'{v:.2e}' for v in per_sample)}) o {e_o:.3e} max {e_max:.3e} | norm1 {en:.2e}")
    tol = TOL[("attn", passes)]
    assert np.isfinite(res["out"]).all()
    assert max(per_sample) < tol["add"] and e_add < tol["add"], (stage, case, variant, per_sample)
    assert e_o < tol["o"] and e_max < tol["max"], (stage, case, variant, e_o, e_max)
    assert en < TOL_GN, (stage, case, variant, en)
    return res, pmax, under


@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("case", list(ATTN_CASES))
@pytest.mark.parametrize("stage", list(ATTN))
def test_vae_attention(ctx, vae, stage, case, passes):
    attn_check(ctx, vae, stage, case, passes)


@pytest.mark.parametrize("stage", list(ATTN))
def test_vae_attention_cancellation(ctx, vae, stage):
    """|mean| / std ~ 8 in every group of the attention input: the sum / sum-of-squares cancellation of its GroupNorm"""
    attn_check(ctx, vae, stage, "16x16_n4", 3, "r=8", r=8.0)


def _with_tensors(ctx, P, updates, fn):
    """run fn(P') with the tensors in `updates` replaced on the context and in a copy of P, then restore both"""
    saved = {k: P(k).numpy().astype(np.float32) for k in updates}
    P2 = O.Params({}, dtype=torch.float64)
    P2.t = dict(P.t)
    for k, v in updates.items():
        P2.t[k] = torch.from_numpy(v.astype(np.float64))
        ctx.set_tensor(k, v)
    ctx.finalize_weights()
    try:
        return fn(P2)
    finally:
        for k, v in saved.items():
            ctx.set_tensor(k, v)
        ctx.finalize_weights()


@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("stage", list(ATTN))
def test_vae_attention_peaked(ctx, vae, stage, passes):
    """q / k weights x 4 (on top of x 1.7): softmax rows nearly one-hot, P ~ 1 on the hi / lo split and most exponentials below
    fp16's smallest subnormal"""
    name = ATTN[stage]
    up = {f"{name}/{k}/weight": (vae(f"{name}/{k}/weight").numpy() * (4.0 / 1.7)).astype(np.float32) for k in ("q", "k")}
    _, pmax, under = _with_tensors(ctx, vae, up, lambda P2: attn_check(ctx, P2, stage, "16x16_n4", passes, "peaked", key="peaked"))
    assert pmax > 0.9 and under > 0.5, (pmax, under)


@pytest.mark.parametrize("stage", list(ATTN))
def test_vae_attention_large_v_bias(ctx, vae, stage):
    """a v bias 10x the v projection: it is added once, after P.V, and only sum(P) = 1 keeps it exact"""
    name = ATTN[stage]
    h, w, n, _ = ATTN_CASES["hw64_n3"]
    x = activation(f"{stage}/vbias", n, 512, h, w)
    with torch.no_grad():
        g = O.group_norm(vae, f"{name}/norm", torch.from_numpy(split22(x))).reshape(n, 512, h * w)
        v = torch.einsum("oc,ncp->nop", vae(f"{name}/v/weight").reshape(512, 512), g)
    vrms = float(v.pow(2).mean().sqrt())
    sign = np.where(np.random.default_rng(3).random(512) < 0.5, -1.0, 1.0)
    up = {f"{name}/v/bias": (10.0 * vrms * sign).astype(np.float32)}
    _with_tensors(ctx, vae, up, lambda P2: attn_check(ctx, P2, stage, "hw64_n3", 3, "v bias x10", x=x, key="vbias"))


def test_vae_attention_trace_overflow(ctx, vae):
    """dec_attn at 8x8 with n = 30 records 96 launches (64 GEMMs, 30 softmaxes, 2 GroupNorm stagings), more than SDB_TRACE_INTS
    holds: the call fails with the record count and the capacity instead of truncating, and the next call on the context runs"""
    x = activation("dec_attn/overflow", 30, 512, 8, 8)
    with pytest.raises(RuntimeError, match=r"96 records do not fit SDB_TRACE_INTS \(63 records\)"):
        ctx.test_vae_stage("dec_attn", x, stats=True)
    attn_check(ctx, vae, "dec_attn", "hw64_n3", 3)


# ------------------------------------------------------------------------------------------------ small-Cout conv
def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def small_cout_case(case, c):
    """(n, H, W, stats, r, expected variant): n is picked from the SM count so both sides of the 2 * SMs tile threshold run"""
    tiles = lambda n, h, w: n * -(-w // 32) * -(-h // 8)
    two = 2 * sm_count()
    if case == "small":        # ragged H (odd), W % 32 != 0, images with their own statistics, the statistics kernel
        n, h, w, st, r = 2, 13, 40, False, 0.0
    elif case == "small_r8":   # |mean| / std ~ 8, producer partials
        n, h, w, st, r = 3, 11, 24, True, 8.0
    elif case == "large":      # 8-row tiles: the smallest n at 24 x 40 with n * tiles >= 2 * SMs, producer partials
        h, w, st, r = 24, 40, True, 0.0
        n = -(-two // tiles(1, h, w))
    else:                      # "fold": more than 128 producer slots per image, the 64:1 pre-fold of Fwd::stats
        n, h, w, st, r = 2, 120, 152, True, 0.0
    variant = (2, 32, KS_SMALL[c]) if tiles(n, h, w) < two else (8, 16, 1)
    return n, h, w, st, r, variant


@pytest.mark.parametrize("case", ["small", "small_r8", "large", "fold"])
@pytest.mark.parametrize("stage", list(OUT))
def test_small_cout_conv(ctx, vae, stage, case):
    norm, conv, c, cout = OUT[stage]
    n, h, w, stats, r, variant = small_cout_case(case, c)
    x = activation(f"{stage}/{case}", n, c, h, w, r)
    res = ctx.test_vae_stage(stage, x, stats=stats)
    tr = res["trace"]
    assert tr["conv"] == [variant], (tr["conv"], variant)
    want = "sums:fold" if case == "fold" else ("sums:partials" if stats else "sums:stats")
    assert tr["gn"] == [want], tr["gn"]
    xs = split22(x) if stats else x.astype(np.float64)
    with torch.no_grad():
        ref = ref_norm_conv(vae, norm, conv, torch.from_numpy(xs)).numpy()
    out = res["out"]
    err = np.abs(out.astype(np.float64) - ref) / np.abs(ref).max()
    border = np.zeros((h, w), bool)
    border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = True
    per_image = [rel(out[s], ref[s]) for s in range(n)]
    e, emax = rel(out, ref), float(err.max())
    print(f"vae {stage} {case} n={n} {h}x{w} variant {variant} gn {tr['gn']}: rel L2 {e:.3e} max {emax:.3e} | border rows "
          f"{float(err[:, :, [0, -1], :].max()):.2e} cols {float(err[:, :, :, [0, -1]].max()):.2e} interior "
          f"{float(err[:, :, ~border].max()):.2e} | worst image {max(per_image):.2e}")
    tol = TOL["small_cout_r8" if r else "small_cout"]
    assert max(per_image) < tol["rel"] and e < tol["rel"] and emax < tol["max"], (stage, case, per_image, emax)


# ------------------------------------------------------------------------------------------------ encoder quant slice
@pytest.mark.parametrize("strided", [False, True])
def test_quant_slice(ctx, vae, strided):
    """quant_conv 8 -> 8 and the slice [0, 4): plain, and into channels 1-4 of the inpainting tensor [n, 5, H, W], scaled by
    0.18215, with channel 0 (the mask's place) as a canary that must come back untouched"""
    n, h, w = 3, 5, 12
    x = activation("enc_out/quant", n, 512, h, w)
    quant = None
    if strided:
        quant = np.random.default_rng(9).standard_normal((n, 5, h, w)).astype(np.float32)
    scale = float(np.float32(0.18215))
    res = ctx.test_vae_stage("enc_out", x, scale=scale, stats=False, quant=quant)
    y8 = torch.from_numpy(res["out"].astype(np.float64))
    with torch.no_grad():
        ref = ref_quant(vae, y8, scale if strided else 1.0).numpy()
    got = res["tap"][:, 1:] if strided else res["tap"]
    e, emax = rel(got, ref), relmax(got, ref)
    print(f"vae quant slice strided={strided}: rel L2 {e:.3e} max {emax:.3e}")
    if strided:
        assert np.array_equal(res["tap"][:, 0], quant[:, 0]), "the strided slice wrote outside channels 1-4"
    assert e < TOL["quant"]["rel"] and emax < TOL["quant"]["max"], (e, emax)


# ------------------------------------------------------------------------------------------------ conv_in
def conv_in_check(res, ref, what):
    out = res["out"]
    e, emax = rel(out, ref), relmax(out, ref)
    per_image = [rel(out[s], ref[s]) for s in range(out.shape[0])]
    print(f"vae {what}: rel L2 {e:.3e} max {emax:.3e} worst image {max(per_image):.2e}")
    tol = TOL["conv_in"]
    assert max(per_image) < tol["rel"] and emax < tol["max"], (what, per_image, emax)
    assert not res["trace"]["gemms"] and not res["trace"]["conv"]


@pytest.mark.parametrize("pre_scale", [1.0, PRE_SCALE])
def test_decoder_conv_in(ctx, vae, pre_scale):
    """post_quant_conv and the pre-scale folded into conv_in's gather; HW = 35: a ragged last 32-pixel CTA"""
    lat = activation("dec_in", 2, 4, 5, 7)
    res = ctx.test_vae_stage("dec_in", lat, scale=pre_scale, stats=False)
    with torch.no_grad():
        ref = ref_dec_in(vae, torch.from_numpy(lat.astype(np.float64)), pre_scale).numpy()
    conv_in_check(res, ref, f"dec_in pre_scale {pre_scale:.9g}")


def test_encoder_conv_in(ctx, vae):
    """3 -> 128 on the Cin = 4 kernel: the padded fourth weight channel is zero, so a nonzero fourth plane changes nothing"""
    img = activation("enc_in", 2, 4, 20, 28)
    res = ctx.test_vae_stage("enc_in", img, stats=False)
    with torch.no_grad():
        ref = O.conv2d(vae, f"{ENC}/conv_in", torch.from_numpy(img[:, :3].astype(np.float64)), padding=1).numpy()
    conv_in_check(res, ref, "enc_in")


def unet_conv_in_check(c, P, n, h, w, cond_ch, want_mod):
    x = activation(f"unet_in/{cond_ch}", n, 4, h, w)
    cond = activation(f"unet_in/cond/{cond_ch}", n, cond_ch, h, w) if cond_ch else None
    res = c.test_vae_stage("unet_in", x, cond=cond, stats=False)
    assert res["trace"]["cond_mod"] == want_mod, res["trace"]
    full = x.astype(np.float64)
    if cond_ch:  # sample s reads the conditioning of sample s % m
        full = np.concatenate([full, cond[np.arange(n) % want_mod].astype(np.float64)], 1)
    with torch.no_grad():
        ref = O.conv2d(P, "unet/input_blocks/conv", torch.from_numpy(full), padding=1).numpy()
    conv_in_check(res, ref, f"unet_in cin {4 + cond_ch} n={n} cond_mod {want_mod}")
    assert np.array_equal(res["out16"], split22(res["out"]).astype(np.float32)), "the fp16 hi + lo copy is not the split of out"


def test_unet_conv_in(ctx, vae):
    unet_conv_in_check(ctx, vae, 3, 12, 20, 0, 0)


@pytest.mark.parametrize("kind,cond_ch,want_mod", [("inpaint", 5, 2), ("pix2pix", 4, 4)])
def test_unet_conv_in_conditioned(kind, cond_ch, want_mod):
    """the 9-channel (inpainting: both CFG halves read one conditioning copy) and 8-channel (InstructPix2Pix: every sample its
    own) conv_in, n = 4 with distinct conditioning per sample"""
    from stable_diffusion_burn_b200 import _lib
    c = _lib.Context(0, **{kind: True})
    try:
        c.init_synthetic(0)
        c.finalize_weights()
        P = params(c, ("unet/input_blocks/conv/",))
        unet_conv_in_check(c, P, 4, 12, 20, cond_ch, want_mod)
    finally:
        c.close()


# ------------------------------------------------------------------------------------------------ downsampler
DOWN_CASES = {0: (2, 10, 14), 1: (2, 18, 10), 2: (3, 6, 10)}  # n, H, W: odd-sized outputs


@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("i", [0, 1, 2])
def test_encoder_downsampler(ctx, vae, i, passes):
    conv, nxt, c = DOWN[i]
    n, h, w = DOWN_CASES[i]
    x = activation(f"down{i}", n, c, h, w)
    with Precision(ctx, 1 if passes == 1 else 0):
        res = ctx.test_vae_stage(f"enc_down{i}", x, stats=True)
    g = res["trace"]["gemms"]
    assert len(g) == 1 and g[0]["kind"] == 5 and g[0]["passes"] == passes and g[0]["N"] == c, g
    with torch.no_grad():
        ref = ref_down(vae, conv, torch.from_numpy(split22(x)), passes == 1).numpy()
    out = res["out"]
    assert out.shape == (n, c, h // 2, w // 2)
    e, emax = rel(out, ref), relmax(out, ref)
    per_image = [rel(out[s], ref[s]) for s in range(n)]
    gn_path = res["trace"]["gn"]
    en = rel(res["out_norm"], ref_gn_silu(vae, nxt, out))
    print(f"vae enc_down{i} P={passes} {n}x{c}x{h}x{w} -> {h // 2}x{w // 2} slots {g[0]['gn_slots']} gn {gn_path}: rel L2 {e:.3e} "
          f"max {emax:.3e} worst image {max(per_image):.2e} | norm1 {en:.2e}")
    tol = TOL[("down", passes)]
    assert max(per_image) < tol["rel"] and emax < tol["max"], (i, passes, per_image, emax)
    assert en < TOL_GN, en
    assert gn_path == (["apply"] if g[0]["gn_slots"] else ["fused"]), gn_path


# ------------------------------------------------------------------------------------------------ entry checks
def test_autoencoder_latent_limits_refused_before_launch(ctx, vae):
    """a latent the mid attention cannot take (H*W % 64 != 0, or H*W > 9216 = 96 x 96) is refused before anything runs"""
    from stable_diffusion_burn_b200 import synth
    from stable_diffusion_burn_b200._lib import SdbError
    n0 = ctx.launch_count()
    for h, w in ((6, 6), (12, 20)):  # H*W % 64 != 0: 12 x 20 used to fail inside the attention after conv_in and block_1 ran
        with pytest.raises(SdbError, match="multiple of 64"):
            ctx.decode_latent(np.zeros((1, 4, h, w), np.float32))
        assert ctx.launch_count() == n0
    with pytest.raises(SdbError, match="multiple of 64"):
        ctx.encode_image(np.zeros((1, 3, 72, 64), np.float32))  # a 9 x 8 latent
    assert ctx.launch_count() == n0
    cx = synth.make_context(1, 5, seed=1)
    un = synth.make_context(1, 5, seed=2)[0]
    with pytest.raises(SdbError, match="768x768 px"):
        ctx.sample_image(cx, un, 7.5, 1, H=128, W=128)
    assert ctx.launch_count() == n0
    with pytest.raises(SdbError, match="768x768 px"):
        ctx.img2img(np.zeros((1, 1024, 1024, 3), np.uint8), cx, un, 7.5, 1, 1.0)
    assert ctx.launch_count() == n0
    with pytest.raises(SdbError, match="768x768 px"):
        ctx.latent_to_image(np.zeros((1, 4, 104, 96), np.float32))
    assert ctx.launch_count() == n0
    lat = ctx.sample_latent(cx, un, 7.5, 1, H=128, W=128)  # no decode: the UNet alone takes a 1024 px latent
    assert lat.shape == (1, 4, 128, 128) and np.isfinite(lat).all()
    assert ctx.launch_count() > n0
