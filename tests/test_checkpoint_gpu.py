"""SD-1.x single-file .safetensors checkpoints on the GPU (DESIGN.md §7 f13): sdb_load_safetensors widens F32 / F16 / BF16 and
re-lays every tensor bit for bit, equals the dump-dir path on the same weights, loads 9- and 8-channel UNets, leaves a context
untouched when it rejects a file, swaps a VAE alone, keeps LoRA adapters, and from_checkpoint picks the context kind."""
import contextlib
import hashlib
import os

import numpy as np
import pytest

from stable_diffusion_burn_b200 import _lib, dumpdir, synth
from stable_diffusion_burn_b200.pipeline import StableDiffusion

from test_checkpoint_cpu import CONV_IN_KEY, encode, ldm_entries, sparse_checkpoint, write_safetensors

pytestmark = pytest.mark.gpu
DTYPES = ("F32", "F16", "BF16")
SCHED = "alpha_cumulative_products"
CONV_IN = "unet/input_blocks/conv/weight"
# F16 / BF16 bit patterns the widening must keep: +-0, subnormals, +-inf, quiet NaNs with payloads, extremes
F16_SPECIAL = np.array([0x0000, 0x8000, 0x0001, 0x83FF, 0x7C00, 0xFC00, 0x7E00, 0xFE01, 0x7BFF, 0x0400], np.uint16)
BF16_SPECIAL = np.array([0x0000, 0x8000, 0x0001, 0x807F, 0x7F80, 0xFF80, 0x7FC0, 0xFFC1, 0x7F7F, 0x0080], np.uint16)


def digest(a):
    return hashlib.sha1(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


def decode(raw: bytes, dtype, shape):
    """numpy's a.astype(np.float32) of the stored array"""
    if dtype == "F32":
        return np.frombuffer(raw, "<f4").astype(np.float32).reshape(shape)
    if dtype == "F16":
        return np.frombuffer(raw, "<f2").astype(np.float32).reshape(shape)
    return (np.frombuffer(raw, "<u2").astype(np.uint32) << np.uint32(16)).view(np.float32).reshape(shape)


@contextlib.contextmanager
def small_work(gb=4):
    """contexts beside the session's get a small work arena: the default one of each would take most of the card"""
    old = os.environ.get("SDB_WORK_GB")
    os.environ["SDB_WORK_GB"] = str(gb)
    try:
        yield
    finally:
        if old is None:
            del os.environ["SDB_WORK_GB"]
        else:
            os.environ["SDB_WORK_GB"] = old


def registry_digests(c):
    return {n: digest(c.get_tensor(n, s)) for n, s in c.tensor_list()}


@pytest.fixture(scope="module")
def ckpt(ctx, tmp_path_factory):
    """synth.make_params(0) (read back from the device: the synthetic stream is bit-identical on both sides) as a full LDM
    checkpoint: dtypes cycle F32 / F16 / BF16 over the keys, data in reverse key order, plus model_ema.* copies, an I64
    position_ids and an F16 alphas_cumprod. -> file, the registry arrays the load must give, their digests."""
    ctx.init_synthetic(0)
    shapes = dict(ctx.tensor_list())
    tensors, expect = [], {}
    for i, (key, reg, shape, tr) in enumerate(ldm_entries(4)):
        dt = DTYPES[i % 3]
        a = ctx.get_tensor(reg, shapes[reg])
        raw = encode(a.T if tr else a, dt)
        w = decode(raw, dt, shape)
        expect[reg] = np.ascontiguousarray(w.T) if tr else w
        tensors.append((key, dt, shape, raw))
    sched = synth.alpha_cumulative_products()
    tensors.append(("alphas_cumprod", "F16", (1000,), encode(sched, "F16")))
    expect[SCHED] = sched.astype(np.float16).astype(np.float32)
    for key, _, shape, raw in tensors[:3]:
        tensors.append(("model_ema." + key.replace(".", ""), "F16", shape, None))
    tensors.append(("cond_stage_model.transformer.text_model.embeddings.position_ids", "I64", (1, 77),
                    np.arange(77, dtype="<i8").tobytes()))
    tensors.sort(key=lambda t: t[0])
    path = write_safetensors(tmp_path_factory.mktemp("ckpt") / "full.safetensors", tensors,
                             data_order=[t[0] for t in reversed(tensors)])
    return dict(path=path, expect=expect, digests={n: digest(a) for n, a in expect.items()})


@pytest.fixture(scope="module")
def loaded(ctx, ckpt):
    ctx.init_synthetic(1)
    ctx.finalize_weights()
    ctx.load_safetensors(ckpt["path"])
    ctx.finalize_weights()
    yield ctx
    ctx.init_synthetic(0)  # the session context's usual weights for the modules after this one
    ctx.finalize_weights()


def test_full_checkpoint_bit_exact(loaded, ckpt):
    got = registry_digests(loaded)
    bad = [n for n in ckpt["digests"] if got[n] != ckpt["digests"][n]]
    assert not bad, bad[:10]
    assert len(got) == len(ckpt["digests"]) == 1131


def test_special_values_and_default_schedule(tmp_path):
    """A sparse file (zeros) whose only data are special bit patterns in an F16 copy, a BF16 copy and an F16 transpose, and no
    alphas_cumprod: those tensors widen bit for bit, every other reads +0, the schedule is the SD-1 default."""
    special = {"clip/position_embedding/weight": "F16", "unet/norm_out/weight": "BF16", "clip/blocks/0/attn/query/weight": "F16"}
    t, want = [], {}
    for k, reg, s, tr in ldm_entries(4):
        dt = special.get(reg, "BF16")
        raw = None
        if reg in special:
            sp = F16_SPECIAL if dt == "F16" else BF16_SPECIAL
            raw = np.resize(sp, int(np.prod(s))).astype("<u2").tobytes()
            w = decode(raw, dt, s)
            want[reg] = np.ascontiguousarray(w.T) if tr else w
        t.append((k, dt, s, raw))
    f = write_safetensors(tmp_path / "special.safetensors", t)
    with small_work():
        c = _lib.Context(0)
    try:
        c.init_synthetic(3)
        c.load_safetensors(f)
        for n, s in c.tensor_list():
            a = c.get_tensor(n, s).view(np.uint32)
            if n == SCHED:
                assert np.array_equal(a, synth.alpha_cumulative_products().view(np.uint32))
            elif n in want:
                assert np.array_equal(a, want[n].view(np.uint32)), n
            else:
                assert not a.any(), n
        assert np.isnan(want["unet/norm_out/weight"][6]) and np.signbit(want["clip/position_embedding/weight"].flat[1])
    finally:
        c.close()


def test_equals_dump_dir(loaded, ckpt, tmp_path_factory):
    root = str(tmp_path_factory.mktemp("dump"))
    dumpdir.save_dump_dir(root, ckpt["expect"])
    with small_work():
        other = _lib.Context(0)
    try:
        other.load_dump_dir(root)
        assert registry_digests(other) == ckpt["digests"]
        other.finalize_weights()
        tok = np.array([[49406, 320, 1125, 539, 320, 2368, 49407]], np.int32)
        ctx_ = synth.make_context(1, 7, seed=3)
        unc = synth.make_context(1, 2, seed=4)[0]
        lat = synth.make_latent(1, 32, 32, seed=5)
        for c in (loaded, other):
            c.set_sampler(0, 0.0, 0)
        outs = [(c.sample_latent(ctx_, unc, 7.5, 4, init_latent=lat, H=32, W=32), c.clip_forward(tok),
                 c.decode_latent(synth.make_latent(1, 8, 8, seed=6))) for c in (loaded, other)]
        for a, b in zip(*outs):
            assert np.array_equal(a, b)
    finally:
        other.close()


@pytest.mark.parametrize("width", [9, 8])
def test_conditioned_unets(ctx, tmp_path, width):
    g = np.random.default_rng(width)
    w = g.standard_normal((320, width, 3, 3)).astype(np.float32)
    t = [(k, "F16", s, encode(w, "F16") if k == CONV_IN_KEY else None) for k, _, s, _ in ldm_entries(width)]
    f = write_safetensors(tmp_path / "c.safetensors", t)
    four = sparse_checkpoint(tmp_path / "four.safetensors", 4)
    with small_work():
        c = _lib.Context(0, inpaint=width == 9, pix2pix=width == 8)
    try:
        c.init_synthetic(0)
        c.finalize_weights()
        x = synth.make_latent(1, 32, 32, seed=5)
        x = np.concatenate([x] * 3, axis=1)[:, :width]
        cx = synth.make_context(1, 5, seed=4)
        y0 = c.unet_forward(x, 500, cx)
        entry = "sdb_create_inpaint" if width == 9 else "sdb_create_pix2pix"
        with pytest.raises(_lib.SdbError, match=r"\[320,4,3,3\].*sdb_create\b"):
            c.load_safetensors(four)
        with pytest.raises(_lib.SdbError, match=rf"\[320,{width},3,3\].*{entry}"):
            ctx.load_safetensors(f)
        assert np.array_equal(c.unet_forward(x, 500, cx), y0)  # rejected: unchanged, still finalized
        c.load_safetensors(f)
        for n, s in c.tensor_list():
            a = c.get_tensor(n, s)
            if n == CONV_IN:
                assert np.array_equal(a, w.astype(np.float16).astype(np.float32))
            elif n != SCHED:
                assert not a.view(np.uint32).any(), n
        c.finalize_weights()
        assert np.isfinite(c.unet_forward(x, 500, cx)).all()
    finally:
        c.close()


def test_rejected_file_leaves_context_finalized(loaded, ckpt, tmp_path):
    cx, unc = synth.make_context(1, 5, seed=4), synth.make_context(1, 2, seed=8)[0]
    lat = synth.make_latent(1, 32, 32, seed=9)
    before = loaded.sample_latent(cx, unc, 7.5, 2, init_latent=lat, H=32, W=32)
    k_last = max(t[0] for t in ldm_entries(4))
    bad = [sparse_checkpoint(tmp_path / "shape.safetensors", change={k_last: ("F16", (3,))}),
           sparse_checkpoint(tmp_path / "dtype.safetensors", change={k_last: ("F64", ldm_entries(4)[-1][2])}),
           sparse_checkpoint(tmp_path / "drop.safetensors", drop=[k_last])]
    f = sparse_checkpoint(tmp_path / "trunc.safetensors")
    os.truncate(f, os.path.getsize(f) - 2)
    for b in bad + [f]:
        with pytest.raises(_lib.SdbError):
            loaded.load_safetensors(b)
    assert np.array_equal(loaded.sample_latent(cx, unc, 7.5, 2, init_latent=lat, H=32, W=32), before)


def test_vae_only_file(loaded, ckpt, tmp_path):
    g = np.random.default_rng(3)
    t, want = [], {}
    for k, reg, s, _ in ldm_entries(vae_only=True):
        a = g.standard_normal(s).astype(np.float32)
        raw = encode(a, "F16")
        want[reg] = decode(raw, "F16", s)
        t.append((k, "F16", s, raw))
    t.append(("loss.logvar", "F32", (), encode(np.zeros((), np.float32), "F32")))
    f = write_safetensors(tmp_path / "vae.safetensors", t)
    assert _lib.probe_safetensors(f) == (_lib.CKPT_VAE, 0)
    try:
        loaded.load_safetensors(f)
        got = registry_digests(loaded)
        for n, d in got.items():
            if n.startswith("autoencoder/"):
                assert d == digest(want[n]), n
            else:
                assert d == ckpt["digests"][n], n
        assert len(want) == sum(n.startswith("autoencoder/") for n in got)
    finally:
        loaded.load_safetensors(ckpt["path"])
        loaded.finalize_weights()


def test_lora_survives_the_load(loaded, ckpt):
    targets = ["unet/input_blocks/rt1/transformer/transformer/attn1/query/weight", "clip/blocks/3/mlp/fc1/weight",
               "unet/output_blocks/rt7/res/conv_in/weight"]
    terms = synth.make_lora(targets, 4, seed=2)
    x, cx = synth.make_latent(1, 32, 32, seed=5), synth.make_context(1, 5, seed=4)
    with small_work():
        b = _lib.Context(0)
    try:
        # adapter, then load, then finalize
        b.init_synthetic(1)
        b.finalize_weights()
        for reg, down, up, a in terms:
            b.lora_add(0, reg, down, up, a)
        b.lora_apply()
        b.load_safetensors(ckpt["path"])
        b.finalize_weights()
        # load, then adapter, then apply
        for reg, down, up, a in terms:
            loaded.lora_add(0, reg, down, up, a)
        loaded.lora_apply()
        for reg in targets:
            s = dict(b.tensor_list())[reg]
            assert np.array_equal(b.get_merged_tensor(reg, s), loaded.get_merged_tensor(reg, s)), reg
        assert np.array_equal(b.unet_forward(x, 500, cx), loaded.unet_forward(x, 500, cx))
    finally:
        b.close()
        loaded.lora_remove(-1)
        loaded.lora_apply()


def test_from_checkpoint(tmp_path):
    for width in (4, 9, 8):
        f = sparse_checkpoint(tmp_path / f"w{width}.safetensors", width)
        with small_work():
            sd = StableDiffusion.from_checkpoint(f)
        try:
            assert sd.ctx.unet_in_channels() == width
            assert not sd.ctx.get_tensor(CONV_IN, (320, width, 3, 3)).any()
        finally:
            sd.close()
    with pytest.raises(ValueError, match="VAE"):
        StableDiffusion.from_checkpoint(sparse_checkpoint(tmp_path / "vae.safetensors", vae_only=True))
