"""GPU parity of the full path through the C ABI against the committed oracle fixtures (tests/golden) and
against the live oracle at small sizes. Tolerance (BASELINE.json north_star): UNet-step tensors within 1e-3
relative of the reference (here: relative L2 and max-abs/max-ref both <= 1e-3); decoded pixels within 1 LSB."""
import os

import numpy as np
import pytest
import torch

from stable_diffusion_burn_b200 import synth, topology

import attn_profiles as AP

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
UNET_TOL = 1.0e-3


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def relmax(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.fixture(scope="module")
def sd(ctx):
    ctx.init_synthetic(0)
    ctx.finalize_weights()
    return ctx


# ------------------------------------------------------------------ fused attention vs reference formula
ATTN = [  # n, Nq, Nk, C, heads
    (2, 256, 256, 320, 8), (1, 1024, 1024, 320, 8), (2, 256, 256, 640, 8), (2, 64, 64, 1280, 8), (1, 256, 256, 1280, 8),
    (2, 256, 77, 320, 8), (2, 64, 13, 1280, 8), (1, 1024, 2, 640, 8), (1, 4096, 4096, 320, 8), (1, 200, 300, 640, 8),
    (2, 1024, 1024, 640, 8), (2, 256, 300, 1280, 8),
]


@pytest.mark.parametrize("n,Nq,Nk,C,heads", ATTN)
def test_attention(ctx, n, Nq, Nk, C, heads):
    from oracle import sd_oracle as O
    rng = np.random.default_rng(Nq + Nk + C)
    q = rng.standard_normal((n, Nq, C)).astype(np.float32)
    k = rng.standard_normal((n, Nk, C)).astype(np.float32)
    v = rng.standard_normal((n, Nk, C)).astype(np.float32)
    # the kernel consumes fp16 v (and P); q / k are fp16 hi + lo pairs (exact logits) for the head dims of the UNet's 3-pass
    # levels (40, 80) and single fp16 values elsewhere: compare against the oracle formula on inputs rounded the same way
    split = (C // heads) in (40, 80)
    q16, k16 = ((torch.from_numpy(a).double() if split else torch.from_numpy(a).half().double()) for a in (q, k))
    v16 = torch.from_numpy(v).half().double()
    ref = O.qkv_attention(q16, k16, v16, heads).numpy()
    out = ctx.test_attention(q, k, v, heads)
    assert rel(out, ref) < 1e-3 and relmax(out, ref) < 2e-3
    if split:  # and the single-operand kernel stays reachable (attn_split = 0)
        ctx.set_option("attn_split", 0)
        try:
            q16, k16 = (torch.from_numpy(a).half().double() for a in (q, k))
            assert rel(ctx.test_attention(q, k, v, heads), O.qkv_attention(q16, k16, v16, heads).numpy()) < 1e-3
        finally:
            ctx.set_option("attn_split", 1)


def _attn_ref(q, k, v, heads, split, kvlen=None, mask=None):
    """fp64 attention on operands rounded the way the kernel consumes them: q / k exact with the split product, else fp16;
    v fp16. kvlen: sample s sees only its first kvlen[s] keys."""
    from oracle import sd_oracle as O
    q64, k64 = ((torch.from_numpy(a).double() if split else torch.from_numpy(a).half().double()) for a in (q, k))
    v64 = torch.from_numpy(v).half().double()
    if kvlen is None:
        return O.qkv_attention(q64, k64, v64, heads, mask=mask).numpy()
    return np.concatenate([O.qkv_attention(q64[s:s + 1], k64[s:s + 1, :L], v64[s:s + 1, :L], heads, mask=mask).numpy()
                           for s, L in enumerate(kvlen)])


def _check_attn(name, out, ref):
    e2, em = rel(out, ref), relmax(out, ref)
    print(f"{name}: rel L2 {e2:.3e} max/max {em:.3e}")
    assert np.isfinite(out).all() and e2 < 1e-3 and em < 2e-3, name


def _kvlen_inputs(rng, n, Nq, Nk, C, lens):
    """q, k, v with the rows past each sample's length zeroed, and k, v with those rows holding large finite values instead"""
    q = rng.standard_normal((n, Nq, C)).astype(np.float32)
    k = rng.standard_normal((n, Nk, C)).astype(np.float32)
    v = rng.standard_normal((n, Nk, C)).astype(np.float32)
    kj, vj = k.copy(), v.copy()
    for s, L in enumerate(lens):
        k[s, L:] = 0.0
        v[s, L:] = 0.0
        sign = lambda: rng.choice(np.float32([-1.0, 1.0]), (Nk - L, C))
        kj[s, L:] = sign() * rng.uniform(6.0, 8.0, (Nk - L, C))
        vj[s, L:] = sign() * rng.uniform(2.0e4, 3.0e4, (Nk - L, C))
    return q, k, v, kj, vj


# per-sample key lengths: n = len(lens); Nk is the padded key count of the batch
ATTN_KVLEN = [  # Nq, Nk, C, heads, lens
    (4096, 96, 320, 8, [2, 77]),  # level 0 of the guided (CFG) batch: unconditional | prompt keys, padded to 96
    (1024, 96, 640, 8, [2, 77]),
    (256, 96, 1280, 8, [1, 63, 64, 65, 77]),  # d = 160: both sides of the 64-key sub-tile boundary
    (200, 300, 320, 8, [1, 128, 129, 300]),  # key-tile boundary and a partial last tile
]


@pytest.mark.parametrize("Nq,Nk,C,heads,lens", ATTN_KVLEN)
def test_attention_kvlen(ctx, Nq, Nk, C, heads, lens):
    """sample s attends only to its first lens[s] keys; whatever the rows past them hold (here up to |k| = 8, |v| = 3e4),
    the output is bit-identical to the run where they are zero: masked keys are dropped by select before the max and the sum"""
    rng = np.random.default_rng(Nq + Nk + C + len(lens))
    q, k, v, kj, vj = _kvlen_inputs(rng, len(lens), Nq, Nk, C, lens)
    d = C // heads
    for split in ((1, 0) if d in (40, 80) else (1,)):
        ctx.set_option("attn_split", split)
        try:
            out = ctx.test_attention(q, k, v, heads, kvlen=lens)
            junk = ctx.test_attention(q, kj, vj, heads, kvlen=lens)
        finally:
            ctx.set_option("attn_split", 1)
        _check_attn(f"kvlen {lens} d={d} split={split}", out, _attn_ref(q, k, v, heads, split and d in (40, 80), kvlen=lens))
        assert np.array_equal(out, junk), (lens, split)


def test_attention_rejects_bad_arguments(ctx):
    from stable_diffusion_burn_b200._lib import SdbError
    q = np.zeros((2, 8, 320), np.float32)
    kv = np.zeros((2, 16, 320), np.float32)
    for lens in ([0, 16], [1, 17], [-1, 4]):  # the kernel would clamp these; the entry refuses them
        with pytest.raises(SdbError, match="kvlen"):
            ctx.test_attention(q, kv, kv, 8, kvlen=lens)
    # the causal mask is applied inside the first key tile only: longer causal sequences are refused on the host
    x = np.zeros((2, 129, 768), np.float32)
    for vt in (True, False):
        with pytest.raises(SdbError, match="at most 128 keys"):
            ctx.test_attention(x, x, x, 12, causal=True, v_transposed=vt)


@pytest.mark.parametrize("L", [1, 2, 8, 20, 77])
def test_attention_clip(ctx, L):
    """the CLIP text encoder's attention: d = 64, causal, V transposed, single fp16 q / k"""
    from oracle import sd_oracle as O
    rng = np.random.default_rng(100 + L)
    n, C, heads = 2, 768, 12
    q, k, v = (rng.standard_normal((n, L, C)).astype(np.float32) for _ in range(3))
    out = ctx.test_attention(q, k, v, heads, causal=True, v_transposed=True)
    _check_attn(f"clip L={L}", out, _attn_ref(q, k, v, heads, False, mask=O.attn_decoder_mask(L, torch.float64)))


RESCALE = [(p, d) for p, (_, dims) in AP.PROFILES.items() for d in dims]


@pytest.mark.parametrize("profile,d", RESCALE)
def test_attention_rescale(ctx, profile, d):
    """logit profiles that make the lazy rescale of the running maximum fire (or stay off) in known ways
    (tests/attn_profiles.py; tests/test_attn_profiles_cpu.py checks each profile against the kernel's rule)"""
    q, k, v = AP.make_case(profile, d)
    _check_attn(f"rescale {profile} d={d}", ctx.test_attention(q, k, v, AP.HEADS), _attn_ref(q, k, v, AP.HEADS, d in (40, 80)))


# ------------------------------------------------------------------ UNet::forward
@pytest.mark.parametrize("case,x,t,c", [
    ("kat_zeros", lambda: np.zeros((1, 4, 64, 64), np.float32), 1, lambda: synth.kat_context()),
    ("sin_ramp", lambda: synth.sin_ramp((1, 4, 64, 64)), 500, lambda: synth.make_context(1, 13)),
    ("randn_t999", lambda: synth.make_latent(1, 64, 64), 999, lambda: synth.make_context(1, 13)),
    ("batch2_32", lambda: synth.make_latent(2, 32, 32, seed=7), 321, lambda: synth.make_context(2, 5, seed=5)),
])
def test_unet_forward_golden(sd, case, x, t, c):
    g = np.load(os.path.join(GOLD, f"unet_{case}.npz"))
    out = sd.unet_forward(x(), t, c())
    e2, em = rel(out, g["out"]), relmax(out, g["out"])
    print(f"unet {case}: rel L2 {e2:.3e} max/max {em:.3e}")
    assert np.isfinite(out).all()
    assert e2 < UNET_TOL and em < UNET_TOL


def test_unet_precision_modes(sd):
    """3-pass everywhere is fp32-class; 1-pass everywhere shows the fp16 operand-rounding floor (reported, not required)."""
    g = np.load(os.path.join(GOLD, "unet_batch2_32.npz"))
    x, c = synth.make_latent(2, 32, 32, seed=7), synth.make_context(2, 5, seed=5)
    try:
        sd.set_option("precision", 3)
        e3 = rel(sd.unet_forward(x, 321, c), g["out"])
        sd.set_option("precision", 1)
        e1 = rel(sd.unet_forward(x, 321, c), g["out"])
    finally:
        sd.set_option("precision", 0)
    print(f"precision sweep: 3-pass {e3:.3e}  1-pass {e1:.3e}")
    assert e3 < 3e-4 and e1 < 5e-3


# ------------------------------------------------------------------ Autoencoder::decode_latent
def test_decode_golden_16(sd):
    g = np.load(os.path.join(GOLD, "vae_16.npz"))
    img = sd.decode_latent(synth.make_latent(1, 16, 16, seed=21))
    e2, em = rel(img, g["img"]), relmax(img, g["img"])
    print(f"vae16: rel L2 {e2:.3e} max/max {em:.3e}")
    assert e2 < 1e-3 and em < 2e-3


def test_decode_golden_64(sd):
    g = np.load(os.path.join(GOLD, "vae_64.npz"))
    img = sd.decode_latent(synth.make_latent(1, 64, 64, seed=22))
    assert img.shape == (1, 3, 512, 512)
    e2 = rel(img[:, :, ::8, ::8], g["img_sub"]); e3 = rel(img[:, :, 250:254, :], g["img_rows"])
    print(f"vae64: rel L2 sub {e2:.3e} rows {e3:.3e}")
    assert e2 < 1e-3 and e3 < 1e-3
    assert abs(float(img.mean()) - float(g["mean"])) < 1e-3 * max(1.0, abs(float(g["std"])))


# ------------------------------------------------------------------ sampler end to end (config C1: 1 step)
def _u8_ok(got, want):
    d = np.abs(got.astype(np.int16) - want.astype(np.int16))
    return float((d <= 1).mean()), int(d.max())


def test_sample_one_step_golden(sd):
    g = np.load(os.path.join(GOLD, "sample_1step.npz"))
    ctx_t = synth.make_context(1, 13); unc = synth.make_context(1, 2, seed=99)[0]; init = synth.make_latent(1, 64, 64)
    lat = sd.sample_latent(ctx_t, unc, 7.5, 1, init_latent=init)
    e = rel(lat, g["latent"])
    print(f"1-step latent rel L2 {e:.3e}")
    assert e < 1e-3
    rgb = sd.sample_image(ctx_t, unc, 7.5, 1, init_latent=init)
    assert rgb.shape == (1, 512, 512, 3) and rgb.dtype == np.uint8
    frac, dmax = _u8_ok(rgb, g["u8"])
    print(f"1-step u8: within 1 LSB {frac:.5f}, max diff {dmax}")
    assert frac >= 0.999 and dmax <= 3


def test_sample_two_steps_batch2_golden(sd):
    g = np.load(os.path.join(GOLD, "sample_2step_b2.npz"))
    ctx_t = synth.make_context(2, 7, seed=3); unc = synth.make_context(1, 2, seed=99)[0]; init = synth.make_latent(2, 32, 32, seed=31)
    lat = sd.sample_latent(ctx_t, unc, 5.0, 2, init_latent=init)
    e = rel(lat, g["latent"])
    print(f"2-step b2 latent rel L2 {e:.3e}")
    assert e < 2e-3
    rgb = sd.sample_image(ctx_t, unc, 5.0, 2, init_latent=init)
    frac, dmax = _u8_ok(rgb[:, ::2, ::2, :], g["u8"])
    print(f"2-step b2 u8: within 1 LSB {frac:.5f}, max diff {dmax}")
    assert frac >= 0.998 and dmax <= 4


def test_graph_replay_is_deterministic(sd):
    ctx_t = synth.make_context(1, 13); unc = synth.make_context(1, 2, seed=99)[0]; init = synth.make_latent(1, 32, 32, seed=5)
    a = sd.sample_latent(ctx_t, unc, 7.5, 4, init_latent=init)
    b = sd.sample_latent(ctx_t, unc, 7.5, 4, init_latent=init)
    sd.set_option("graphs", 0)
    try:
        c = sd.sample_latent(ctx_t, unc, 7.5, 4, init_latent=init)
    finally:
        sd.set_option("graphs", 1)
    assert np.array_equal(a, b) and np.array_equal(a, c)


def test_error_paths(sd):
    ctx_t = synth.make_context(1, 13); unc = synth.make_context(1, 2, seed=99)[0]
    with pytest.raises(Exception):
        sd.sample_latent(ctx_t, unc, 7.5, 2000, init_latent=synth.make_latent(1, 32, 32))  # step_by(0) in the reference
    with pytest.raises(Exception):
        sd.unet_forward(np.zeros((1, 4, 16, 16), np.float32), 1, synth.kat_context())  # deepest level would have 4 tokens
    with pytest.raises(Exception):
        sd.unet_forward(np.zeros((1, 4, 12, 12), np.float32), 1, synth.kat_context())  # not a multiple of 8


def test_option_keys(ctx):
    """sdb_set_option takes the run configurations and test hooks of sdb200.h; the design switches and tuning constants that
    were once options are unknown keys, so a caller still setting one learns that it no longer does anything"""
    from stable_diffusion_burn_b200._lib import SdbError
    for key in ("attn_regsplit", "prefetch_w", "mlp_passes", "splitk_min_iters", "splitk_chunk", "gn_apply_ctas", "gn_min_pix"):
        with pytest.raises(SdbError, match="unknown option"):
            ctx.set_option(key, 1)
    kept = dict(precision=0, graphs=1, splitk=1, emb_hoist=1, attn_split=1, raw16=1, skip_merge=1, gn_epilogue=1)
    for key, default in kept.items():
        ctx.set_option(key, default)


# ------------------------------------------------------------------ BASELINE configs 3-5 as parity cases
def test_unet_768px_golden(sd):
    """config C4 geometry: 96x96 latent (768x768 px): 9216 / 2304 / 576 / 144 tokens per level, non power-of-two tiles."""
    g = np.load(os.path.join(GOLD, "unet_768px.npz"))
    out = sd.unet_forward(synth.make_latent(1, 96, 96, seed=96), 777, synth.make_context(1, 9, seed=96))
    e2, em = rel(out, g["out"]), relmax(out, g["out"])
    print(f"unet 96x96: rel L2 {e2:.3e} max/max {em:.3e}")
    assert e2 < UNET_TOL and em < UNET_TOL


def test_batch_invariance(sd):
    """configs C3/C5 run batches of 8 per GPU: an image must not depend on what else is in its batch."""
    ctx_t = synth.make_context(8, 11, seed=41); unc = synth.make_context(1, 2, seed=99)[0]; init = synth.make_latent(8, 32, 32, seed=51)
    full = sd.sample_latent(ctx_t, unc, 7.5, 2, init_latent=init)
    for i in (0, 5):
        one = sd.sample_latent(ctx_t[i:i + 1], unc, 7.5, 2, init_latent=init[i:i + 1])
        e = rel(full[i:i + 1], one)
        print(f"batch invariance image {i}: rel L2 {e:.3e}")
        # Not bit-exact: the batch size changes the split-K factors, which changes the low-order bits of fp32 sums
        # (tensor-core accumulation error ~1.2e-9*K, tools/diag_split.py); downstream fp16 operand roundings then
        # decorrelate, so two batch shapes differ by about one rounding-noise amplitude — each stays within 1e-3 of the oracle.
        assert e < 1e-3


def test_time_embedding_hoist_bit_identical(sd):
    """sample_latent computes the time-embedding rows of all timesteps once per call (gemv_rows_kernel) instead of three GEMVs
    inside every step; the rows - and therefore the latents - are bit-identical to the per-step path (emb_hoist = 0), for a
    schedule whose length is not a multiple of the 5 rows a CTA handles, and again on a second call with another schedule."""
    c = synth.make_context(1, 9, seed=3); unc = synth.make_context(1, 2, seed=99)[0]; init = synth.make_latent(1, 32, 32, seed=8)
    for steps in (7, 3):
        new = sd.sample_latent(c, unc, 7.5, steps, init_latent=init, H=32, W=32)
        sd.set_option("emb_hoist", 0)
        try:
            old = sd.sample_latent(c, unc, 7.5, steps, init_latent=init, H=32, W=32)
        finally:
            sd.set_option("emb_hoist", 1)
        assert np.isfinite(new).all() and np.array_equal(new, old), steps


def test_decode_batch8(sd):
    lat = synth.make_latent(8, 16, 16, seed=61)
    imgs = sd.decode_latent(lat)
    one = sd.decode_latent(lat[6:7])
    assert imgs.shape == (8, 3, 128, 128) and np.isfinite(imgs).all()
    assert rel(imgs[6:7], one) < 1e-3
