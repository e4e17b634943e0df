"""LoRA adapters on the GPU (DESIGN.md §7 f8) through the C ABI: the merge through every packer against set_tensor of the
numpy-merged weight, the merge precision against fp64, restoring the base, the step-graph cache, adapters across base changes,
the Python loader and the errors."""
import zlib

import numpy as np
import pytest

from stable_diffusion_burn_b200 import _lib, lora, pipeline, synth, topology

pytestmark = pytest.mark.gpu
PARAMS = {n: s for n, s, _, _ in topology.all_params()}
ST0 = "unet/input_blocks/rt1/transformer"
STEPS, SCALE = 2, 5.0


@pytest.fixture(scope="module")
def sd(ctx):
    ctx.init_synthetic(0)
    ctx.finalize_weights()
    yield ctx
    ctx.lora_remove(-1)  # later modules share the session's context
    ctx.lora_apply()
    ctx.set_option("graphs", 1)
    ctx.finalize_weights()


@pytest.fixture(scope="module")
def inputs():
    return dict(ctx=synth.make_context(1, 7, seed=3), unc=synth.make_context(1, 2, seed=99)[0],
                noise=synth.make_latent(1, 32, 32, seed=41),
                tok=np.array([[49406, 320, 1125, 539, 320, 2368, 49407, 0, 0, 0]], np.int32),
                lat=synth.make_latent(1, 8, 8, seed=5))


def outputs(sd, x, decode=False):
    out = dict(latent=sd.sample_latent(x["ctx"], x["unc"], SCALE, STEPS, init_latent=x["noise"]), clip=sd.clip_forward(x["tok"]))
    if decode:
        out["img"] = sd.decode_latent(x["lat"])
    return out


def same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in a)


@pytest.fixture(scope="module")
def base(sd, inputs):
    return outputs(sd, inputs, decode=True)


def geom(reg):
    s = PARAMS[reg]
    return (s[1], s[0]) if len(s) == 2 else (s[0], int(np.prod(s[1:])))  # (out, fan-in)


def dyadic_term(reg, rank, seed):
    """Factors whose products and sums are exact in fp32: down = k / 8, up = k / 2^11 with |k| <= 8."""
    out, fan_in = geom(reg)
    g = np.random.default_rng(seed)
    down = (g.integers(-8, 9, (rank, fan_in)) / 8.0).astype(np.float32)
    up = (g.integers(-8, 9, (out, rank)) / 2048.0).astype(np.float32)
    return down, up


def merged(w, terms):
    """numpy float32(W + sum s (up . down)) in the registry layout; terms: (down, up, alpha, multiplier)."""
    d = sum(lora.delta(dn, up, a, m, shape=w.shape) for dn, up, a, m in terms)
    return (w.astype(np.float64) + d).astype(np.float32)


KINDS = {
    "self_qkv": [f"{ST0}/transformer/attn1/{n}/weight" for n in ("query", "key", "value")],
    "cross_q": [f"{ST0}/transformer/attn2/query/weight"],
    "cross_kv": [f"{ST0}/transformer/attn2/{n}/weight" for n in ("key", "value")],
    "attn_out": [f"{ST0}/transformer/attn1/out/weight", f"{ST0}/transformer/attn2/out/weight"],
    "geglu": [f"{ST0}/transformer/mlp/geglu/proj/weight"],
    "ff": [f"{ST0}/transformer/mlp/lin/weight"],
    "proj_in_out": [f"{ST0}/proj_in/weight", f"{ST0}/proj_out/weight"],
    "res_conv3x3": ["unet/input_blocks/rt1/res/conv_in/weight", "unet/output_blocks/rt7/res/conv_out/weight"],
    "skip_1x1": ["unet/input_blocks/rt3/res/skip_connection/weight"],
    "lin_embed": ["unet/input_blocks/rt1/res/lin_embed/weight", "unet/middle_block/res2/lin_embed/weight"],
    "down_conv": ["unet/input_blocks/d1/weight"],
    "upsample_conv": ["unet/output_blocks/rtu2/upsample/conv/weight"],
    "clip_qk": ["clip/blocks/0/attn/query/weight", "clip/blocks/0/attn/key/weight"],
    "clip_v_out": ["clip/blocks/1/attn/value/weight", "clip/blocks/1/attn/out/weight"],
    "clip_fc": ["clip/blocks/2/mlp/fc1/weight", "clip/blocks/2/mlp/fc2/weight"],
}


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_exact_merge_through_packers(sd, inputs, base, kind):
    """Dyadic factors: sampling and CLIP through the merged packing equal, bit for bit, the same context after set_tensor of the
    numpy-merged weights and a finalize. Removing the adapter and applying restores the base outputs."""
    regs = KINDS[kind]
    terms = {}
    for i, reg in enumerate(regs):
        rank = 2 + i
        down, up = dyadic_term(reg, rank, seed=zlib.crc32(reg.encode()))
        alpha = rank / 2.0  # s = 0.5: exact
        terms[reg] = (down, up, alpha)
        sd.lora_add(0, reg, down, up, alpha)
    sd.lora_apply()
    got = outputs(sd, inputs)
    w = {reg: sd.get_tensor(reg, PARAMS[reg]) for reg in regs}
    want_w = {reg: merged(w[reg], [terms[reg] + (1.0,)]) for reg in regs}
    for reg in regs:
        assert np.array_equal(sd.get_merged_tensor(reg, PARAMS[reg]), want_w[reg]), (kind, reg)
        assert np.array_equal(sd.get_tensor(reg, PARAMS[reg]), w[reg]), (kind, reg)  # the master copy stays the base
    assert not same(got, base), kind  # the adapter changes something
    sd.lora_remove(0)
    sd.lora_apply()
    assert same(outputs(sd, inputs), base), kind
    try:
        for reg in regs:
            sd.set_tensor(reg, want_w[reg])
        sd.finalize_weights()
        ref = outputs(sd, inputs)
    finally:
        for reg in regs:
            sd.set_tensor(reg, w[reg])
        sd.finalize_weights()
    for k in ("latent", "clip"):
        assert np.array_equal(got[k], ref[k]), (kind, k, float(np.abs(got[k] - ref[k]).max()))


@pytest.mark.parametrize("rank", [1, 4, 64, 128])
def test_merge_precision(sd, rank):
    """Random factors, two adapters on one tensor, negative multipliers: W_eff within the fp32 bound
    2^-23 (|W| + 2 r sum_t |s up . down|) of fp64."""
    g = np.random.default_rng(rank)
    for reg in ("clip/blocks/4/mlp/fc1/weight", "unet/input_blocks/rt3/res/conv_in/weight"):
        out, fan_in = geom(reg)
        w = sd.get_tensor(reg, PARAMS[reg]).astype(np.float64)
        terms = []
        for ad, mult in ((3, -0.7), (5, 1.3)):
            down = g.standard_normal((rank, fan_in)).astype(np.float32)
            up = (g.standard_normal((out, rank)) * 0.01).astype(np.float32)
            alpha = float(g.uniform(0.5, 2.0) * rank)
            sd.lora_add(ad, reg, down, up, alpha)
            sd.lora_scale(ad, mult)
            terms.append((down, up, alpha, mult))
        sd.lora_apply()
        got = sd.get_merged_tensor(reg, PARAMS[reg]).astype(np.float64)
        sd.lora_remove(-1)
        sd.lora_apply()
        exact = w + sum(lora.delta(d, u, a, m, shape=w.shape) for d, u, a, m in terms)
        mag = sum(abs(float(np.float32(m * a / d.shape[0]))) * (np.abs(u.astype(np.float64)) @ np.abs(d.astype(np.float64)))
                  for d, u, a, m in terms)
        mag = mag.T.reshape(w.shape) if w.ndim == 2 else mag.reshape(w.shape)
        bound = 2.0 ** -23 * (np.abs(w) + 2 * rank * mag)
        # the scale itself is rounded to fp32: (float)(m alpha / r) differs from the fp64 scale by <= 2^-24 relative
        bound += 2.0 ** -24 * np.abs(exact - w)
        err = np.abs(got - exact)
        assert (err <= bound).all(), (reg, rank, float((err / np.maximum(bound, 1e-30)).max()))


def test_restore_base_by_remove_or_zero_scale(sd, inputs, base):
    """Apply, then scale to 0 and apply, then remove and apply: sampling, CLIP and decode equal the no-adapter run."""
    for reg, down, up, a in synth.make_lora(KINDS["geglu"] + KINDS["clip_fc"] + KINDS["down_conv"], 8, seed=1):
        sd.lora_add(7, reg, down, up, a)
    sd.lora_apply()
    assert not same(outputs(sd, inputs), {k: base[k] for k in ("latent", "clip")})
    sd.lora_scale(7, 0.0)
    sd.lora_apply()
    assert same(outputs(sd, inputs, decode=True), base)
    sd.lora_scale(7, 1.0)
    sd.lora_apply()
    sd.lora_remove(7)
    sd.lora_apply()
    assert same(outputs(sd, inputs, decode=True), base)


def test_step_graph_survives_apply(sd, inputs):
    """After a call that cached the step graph, applying an adapter leaves the graph cached (the next call makes the launch count
    of a cached replay) and the result equals the graphs-off result; A -> B -> A returns the first A result bit for bit."""
    run = lambda: sd.sample_latent(inputs["ctx"], inputs["unc"], SCALE, STEPS, init_latent=inputs["noise"])
    run()
    n0 = sd.launch_count()
    run()
    cached = sd.launch_count() - n0
    for ad, seed in ((1, 11), (2, 12)):
        for reg, down, up, a in synth.make_lora(KINDS["self_qkv"] + KINDS["res_conv3x3"] + KINDS["lin_embed"], 4, seed=seed):
            sd.lora_add(ad, reg, down, up, a)
    sd.lora_scale(2, 0.0)
    sd.lora_apply()
    n0 = sd.launch_count()
    ra = run()
    assert sd.launch_count() - n0 == cached
    sd.set_option("graphs", 0)
    try:
        assert np.array_equal(run(), ra)
    finally:
        sd.set_option("graphs", 1)
    sd.lora_scale(1, 0.0), sd.lora_scale(2, 1.0)
    sd.lora_apply()
    rb = run()
    assert not np.array_equal(rb, ra)
    sd.lora_scale(2, 0.0), sd.lora_scale(1, 1.0)
    sd.lora_apply()
    n0 = sd.launch_count()
    assert np.array_equal(run(), ra)
    assert sd.launch_count() - n0 == cached
    sd.lora_remove(-1)
    sd.lora_apply()


def test_adapters_survive_base_changes(sd, inputs):
    """A finalize with an adapter active gives the same result; set_tensor of a targeted base weight and a finalize merge the
    adapter onto the new base."""
    reg = KINDS["cross_q"][0]
    down, up = dyadic_term(reg, 4, seed=21)
    sd.lora_add(4, reg, down, up, 4.0)
    sd.lora_apply()
    a = outputs(sd, inputs)
    sd.finalize_weights()
    assert same(outputs(sd, inputs), a)
    w = sd.get_tensor(reg, PARAMS[reg])
    w2 = (w * np.float32(0.5)).astype(np.float32)
    try:
        sd.set_tensor(reg, w2)
        sd.finalize_weights()
        assert np.array_equal(sd.get_tensor(reg, PARAMS[reg]), w2)
        assert np.array_equal(sd.get_merged_tensor(reg, PARAMS[reg]), merged(w2, [(down, up, 4.0, 1.0)]))
        b = outputs(sd, inputs)
        sd.lora_remove(4)
        sd.lora_apply()
        sd.set_tensor(reg, merged(w2, [(down, up, 4.0, 1.0)]))
        sd.finalize_weights()
        assert same(outputs(sd, inputs), b)
    finally:
        sd.lora_remove(-1)
        sd.set_tensor(reg, w)
        sd.finalize_weights()


def test_python_loader_kohya_equals_peft(sd, inputs, base, tmp_path):
    """A kohya file and a PEFT file holding the same factors give identical outputs through StableDiffusion.load_lora."""
    from safetensors.numpy import save_file
    p = pipeline.StableDiffusion.__new__(pipeline.StableDiffusion)
    p.ctx = sd
    kohya = {v: k for k, v in lora.kohya_names().items()}
    peft = {v: k for k, v in lora.peft_names().items()}
    regs = KINDS["attn_out"] + KINDS["skip_1x1"] + KINDS["clip_qk"]
    fk, fp = {}, {}
    for reg, down, up, a in synth.make_lora(regs, 8, seed=3, alpha=4.0):
        shape = PARAMS[reg]
        d = down.reshape((8,) + tuple(shape[1:])) if len(shape) == 4 else down
        u = up.reshape(up.shape + (1, 1)) if len(shape) == 4 else up
        fk[kohya[reg] + ".lora_down.weight"], fk[kohya[reg] + ".lora_up.weight"] = d.astype(np.float16), u.astype(np.float16)
        fk[kohya[reg] + ".alpha"] = np.array(4.0, np.float16)
        # PEFT has no alpha: alpha = r = 8, so the up factor carries the 1/2 (in F32: halving an fp16 subnormal would round)
        fp[peft[reg] + ".lora_A.weight"] = d.astype(np.float16)
        fp[peft[reg] + ".lora_B.weight"] = u.astype(np.float16).astype(np.float32) * np.float32(0.5)
    save_file(fk, str(tmp_path / "k.safetensors"))
    save_file(fp, str(tmp_path / "p.safetensors"))
    p.load_lora(tmp_path / "k.safetensors", 0, multiplier=0.75)
    a = outputs(sd, inputs)
    p.unload_lora(0)
    p.load_lora(tmp_path / "p.safetensors", 0, multiplier=0.75)
    b = outputs(sd, inputs)
    assert same(a, b) and not same(a, base)
    p.set_lora_scale(0, 0.0)
    assert same(outputs(sd, inputs), {k: base[k] for k in ("latent", "clip")})
    with pytest.raises(ValueError, match="adapter 0 is in use"):  # nothing is added to the adapter already loaded
        p.load_lora(tmp_path / "k.safetensors", 0)
    p.set_lora_scale(0, 0.75)
    assert same(outputs(sd, inputs), b)
    # a file naming one module under both conventions is rejected before anything is added
    bad = dict(fk)
    bad[peft[regs[0]] + ".lora_A.weight"] = fk[kohya[regs[0]] + ".lora_down.weight"]
    save_file(bad, str(tmp_path / "bad.safetensors"))
    with pytest.raises(ValueError, match="more than once"):
        p.load_lora(tmp_path / "bad.safetensors", 1)
    # an add failing part way removes the new adapter's terms and applies nothing: nothing is left pending
    real_add, calls = sd.lora_add, []

    def failing_add(*args):
        calls.append(args)
        if len(calls) == 3:
            raise _lib.SdbError("injected failure")
        real_add(*args)

    sd.lora_add = failing_add
    try:
        with pytest.raises(_lib.SdbError, match="injected failure"):
            p.load_lora(tmp_path / "k.safetensors", 1)
    finally:
        del sd.lora_add
    assert sd.lora_adapters() == {0}
    assert same(outputs(sd, inputs), b)  # no sdb_lora_apply needed: the calls run
    p.unload_lora()
    assert same(outputs(sd, inputs), {k: base[k] for k in ("latent", "clip")})


def test_errors(sd, inputs, base):
    """Every rejection names its field and value and changes nothing; compute with pending changes names sdb_lora_apply."""
    reg = KINDS["ff"][0]
    out, fan_in = geom(reg)
    down, up = np.ones((2, fan_in), np.float32), np.ones((out, 2), np.float32)
    lib, h = sd.lib, sd.h
    f = _lib.ptr

    def err(rc):
        assert rc != 0
        return lib.sdb_last_error(h).decode()

    assert "unknown tensor 'nope'" in err(lib.sdb_lora_add(h, 0, b"nope", 2, f(down), f(up), 2.0))
    for bad in ("unet/input_blocks/conv/weight", "unet/lin1_time_embed/weight", "unet/conv_out/weight",
                f"{ST0}/norm/weight", f"{ST0}/transformer/attn1/out/bias", "clip/token_embedding/weight",
                "autoencoder/decoder/conv_in/weight"):
        assert "is not a LoRA target" in err(lib.sdb_lora_add(h, 0, bad.encode(), 2, f(down), f(up), 2.0)), bad
    assert "rank 0 must be >= 1" in err(lib.sdb_lora_add(h, 0, reg.encode(), 0, f(down), f(up), 2.0))
    assert "down is NULL" in err(lib.sdb_lora_add(h, 0, reg.encode(), 2, None, f(up), 2.0))
    assert "up is NULL" in err(lib.sdb_lora_add(h, 0, reg.encode(), 2, f(down), None, 2.0))
    for alpha in (float("nan"), float("inf"), 0.0, -1.0):
        assert "alpha" in err(lib.sdb_lora_add(h, 0, reg.encode(), 2, f(down), f(up), alpha)), alpha
    assert "adapter -2 must be >= 0" in err(lib.sdb_lora_add(h, -2, reg.encode(), 2, f(down), f(up), 2.0))
    assert "no adapter 0" in err(lib.sdb_lora_scale(h, 0, 1.0))
    assert "no adapter 9" in err(lib.sdb_lora_remove(h, 9))
    # nothing was added: nothing is pending
    assert same(outputs(sd, inputs), {k: base[k] for k in ("latent", "clip")})
    sd.lora_add(0, reg, down, up, 2.0)
    assert "already has a term for" in err(lib.sdb_lora_add(h, 0, reg.encode(), 2, f(down), f(up), 2.0))
    assert "multiplier nan must be finite" in err(lib.sdb_lora_scale(h, 0, float("nan")))
    with pytest.raises(_lib.SdbError, match="sdb_lora_apply"):
        sd.sample_latent(inputs["ctx"], inputs["unc"], SCALE, STEPS, init_latent=inputs["noise"])
    with pytest.raises(_lib.SdbError, match="sdb_lora_apply"):
        sd.clip_forward(inputs["tok"])
    with pytest.raises(_lib.SdbError, match="sdb_lora_apply"):
        sd.get_merged_tensor(reg, PARAMS[reg])
    sd.lora_remove(0)
    sd.lora_apply()
    assert same(outputs(sd, inputs), {k: base[k] for k in ("latent", "clip")})


def test_golden(sd):
    """tests/golden/lora_b1.npz (tests/golden/make_lora_golden.py): the oracle on the synthetic weights with a seeded adapter on one
    module of every target kind, merged in fp64. The adapter is regenerated here from its seed and applied; CLIP of the prompt
    and of the negative at the CLIP bar, then 4 DDIM steps from the stored contexts at the bars of
    test_sample_two_steps_batch2_golden."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import make_lora_golden as MG
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lora_b1.npz"))
    rel = lambda a, b: float(np.linalg.norm(np.float64(a) - b) / np.linalg.norm(np.float64(b)))
    for reg, down, up, a in synth.make_lora(MG.LORA_TARGETS, MG.RANK, seed=MG.SEED):
        sd.lora_add(11, reg, down, up, a)
    sd.lora_apply()
    try:
        ctx, unc = sd.clip_forward(g["tokens"]), sd.clip_forward(g["utokens"])
        ec, eu = rel(ctx, g["context"]), rel(unc, g["uncond"])
        lat = sd.sample_latent(g["context"], g["uncond"][0], MG.SCALE, MG.STEPS, init_latent=g["init"])
        rgb = sd.sample_image(g["context"], g["uncond"][0], MG.SCALE, MG.STEPS, init_latent=g["init"])
    finally:
        sd.lora_remove(11)
        sd.lora_apply()
    e = rel(lat, g["latent"])
    d = np.abs(rgb[:, ::2, ::2, :].astype(np.int16) - g["u8"].astype(np.int16))
    frac, dmax = float((d <= 1).mean()), int(d.max())
    print(f"lora golden: clip rel L2 {ec:.3e} / {eu:.3e}, latent rel L2 {e:.3e}, u8 within 1 LSB {frac:.5f}, max diff {dmax}")
    assert ec < 1e-3 and eu < 1e-3
    assert e < 2e-3
    assert frac >= 0.998 and dmax <= 4
