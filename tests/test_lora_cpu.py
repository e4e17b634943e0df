"""LoRA adapter files (DESIGN.md §7 f8): the safetensors reader, the kohya / PEFT name map and the alpha / r rule. No GPU."""
import re

import numpy as np
import pytest

from stable_diffusion_burn_b200 import lora, synth, topology

PARAMS = {n: s for n, s, _, _ in topology.all_params()}


def _geom(reg):
    s = PARAMS[reg]
    return (s[1], s[0]) if len(s) == 2 else (s[0], int(np.prod(s[1:])))  # (out, fan-in)


# ---------------------------------------------------------------------------------------------------------------- reader
@pytest.mark.parametrize("dtype", ["F32", "F16"])
def test_reader_matches_safetensors_numpy(tmp_path, dtype):
    from safetensors.numpy import load_file, save_file
    g = np.random.default_rng(1)
    npt = np.float32 if dtype == "F32" else np.float16
    data = {"a.lora_down.weight": g.standard_normal((4, 7)).astype(npt), "b": g.standard_normal((3, 2, 1, 5)).astype(npt),
            "alpha": np.array(8.0, npt), "empty": np.zeros((0, 3), npt)}
    p = tmp_path / "x.safetensors"
    save_file(data, str(p), metadata={"format": "pt"})
    ref = load_file(str(p))
    got = lora.read_safetensors(p)
    assert set(got) == set(ref)
    for k in ref:
        assert got[k].dtype == ref[k].dtype and got[k].shape == ref[k].shape, k
        np.testing.assert_array_equal(got[k], ref[k])


def test_reader_matches_safetensors_torch_bf16(tmp_path):
    import torch
    from safetensors.torch import load_file, save_file
    g = torch.Generator().manual_seed(2)
    data = {"x": torch.randn(5, 9, generator=g).to(torch.bfloat16), "y": torch.randn(16, 3, 3, 3, generator=g).to(torch.bfloat16)}
    p = tmp_path / "b.safetensors"
    save_file(data, str(p))
    ref = load_file(str(p))
    got = lora.read_safetensors(p)
    for k in ref:
        assert got[k].dtype == np.float32
        np.testing.assert_array_equal(got[k], ref[k].float().numpy())


def test_reader_rejects_other_dtypes(tmp_path):
    from safetensors.numpy import save_file
    p = tmp_path / "i.safetensors"
    save_file({"ids": np.arange(4, dtype=np.int64)}, str(p))
    with pytest.raises(ValueError, match="ids has dtype I64"):
        lora.read_safetensors(p)


# ---------------------------------------------------------------------------------------------------------------- names
def test_module_counts_from_topology():
    unet = set(lora.UNET_MODULES.values())
    st = [r for r in unet if "/transformer/" in r or r.endswith(("/proj_in/weight", "/proj_out/weight"))]
    res = [r for r in unet if r.endswith(("/conv_in/weight", "/conv_out/weight", "/skip_connection/weight", "/lin_embed/weight"))]
    rs = [r for r in unet if r not in st and r not in res]
    # from the topology: 16 transformers x 12 Linears / 1x1 convs, 22 ResBlocks x 3 + the skip convs, 3 down + 3 up convs
    n_st = sum(1 for n, *_ in topology.unet_params() if n.endswith("/proj_in/weight"))
    n_rb = sum(1 for n, *_ in topology.unet_params() if n.endswith("/lin_embed/weight"))
    n_skip = sum(1 for n, *_ in topology.unet_params() if n.endswith("/skip_connection/weight"))
    assert (n_st, n_rb, n_skip) == (16, 22, 14)
    assert len(st) == 12 * n_st == 192
    assert len(res) == 3 * n_rb + n_skip == 80
    assert sorted(rs) == sorted(n for n, *_ in topology.unet_params()
                                if re.fullmatch(r"unet/input_blocks/d\d/weight|unet/output_blocks/\w+/upsample/conv/weight", n))
    assert len(rs) == 6 and len(unet) == 278 == len(lora.UNET_MODULES)
    assert len(set(lora.CLIP_MODULES.values())) == len(lora.CLIP_MODULES) == 72


@pytest.mark.parametrize("table", ["kohya", "peft"])
def test_names_map_one_to_one_onto_targets(table):
    names = lora.kohya_names() if table == "kohya" else lora.peft_names()
    assert len(names) == 278 + 72
    assert len(set(names.values())) == len(names)  # one-to-one
    for mod, reg in names.items():
        assert reg in PARAMS, (mod, reg)
        assert lora.registry_name(mod) == reg
        # both orientations: a [r, fan-in] down and an [out, r] up of the module fit the registry weight
        out, fan_in = _geom(reg)
        shape = PARAMS[reg]
        d = lora.delta(np.ones((2, fan_in)), np.ones((out, 2)), 2.0, shape=shape)
        assert d.shape == shape


def test_clip_names_equal_transformers_linear_modules():
    from transformers import CLIPTextConfig, CLIPTextModel
    import torch
    with torch.device("meta"):
        m = CLIPTextModel(CLIPTextConfig())
        sd = CLIPTextModel(CLIPTextConfig(hidden_size=768, intermediate_size=3072, num_attention_heads=12))  # SD-v1 sizes
    lin = {n: mod for n, mod in m.named_modules() if isinstance(mod, torch.nn.Linear)}
    assert set(lin) == set(lora.CLIP_MODULES)
    lin = {n: mod for n, mod in sd.named_modules() if isinstance(mod, torch.nn.Linear)}
    assert set(lin) == set(lora.CLIP_MODULES)
    for n, mod in lin.items():
        assert _geom(lora.CLIP_MODULES[n]) == (mod.out_features, mod.in_features), n


SPOT = {
    "down_blocks.0.resnets.0.conv1": "unet/input_blocks/rt1/res/conv_in/weight",
    "down_blocks.0.attentions.1.transformer_blocks.0.attn1.to_q": "unet/input_blocks/rt2/transformer/transformer/attn1/query/weight",
    "down_blocks.1.resnets.0.conv_shortcut": "unet/input_blocks/rt3/res/skip_connection/weight",
    "down_blocks.2.downsamplers.0.conv": "unet/input_blocks/d3/weight",
    "down_blocks.3.resnets.0.conv1": "unet/input_blocks/r1/conv_in/weight",
    "down_blocks.3.resnets.1.time_emb_proj": "unet/input_blocks/r2/lin_embed/weight",
    "mid_block.resnets.1.conv2": "unet/middle_block/res2/conv_out/weight",
    "mid_block.attentions.0.transformer_blocks.0.ff.net.0.proj": "unet/middle_block/transformer/transformer/mlp/geglu/proj/weight",
    "mid_block.attentions.0.proj_out": "unet/middle_block/transformer/proj_out/weight",
    "up_blocks.0.resnets.0.conv_shortcut": "unet/output_blocks/r1/skip_connection/weight",
    "up_blocks.0.resnets.2.conv1": "unet/output_blocks/ru/res/conv_in/weight",
    "up_blocks.0.upsamplers.0.conv": "unet/output_blocks/ru/upsample/conv/weight",
    "up_blocks.1.attentions.2.transformer_blocks.0.attn2.to_out.0": "unet/output_blocks/rtu1/transformer/transformer/attn2/out/weight",
    "up_blocks.1.upsamplers.0.conv": "unet/output_blocks/rtu1/upsample/conv/weight",
    "up_blocks.2.resnets.2.time_emb_proj": "unet/output_blocks/rtu2/res/lin_embed/weight",
    "up_blocks.2.upsamplers.0.conv": "unet/output_blocks/rtu2/upsample/conv/weight",
    "up_blocks.3.attentions.2.transformer_blocks.0.ff.net.2": "unet/output_blocks/rt7/transformer/transformer/mlp/lin/weight",
    "up_blocks.3.resnets.0.conv_shortcut": "unet/output_blocks/rt5/res/skip_connection/weight",
}


@pytest.mark.parametrize("module", sorted(SPOT))
def test_spot_check(module):
    assert lora.UNET_MODULES[module] == SPOT[module]
    assert lora.registry_name("lora_unet_" + module.replace(".", "_")) == SPOT[module]
    assert lora.registry_name("unet." + module) == SPOT[module]


def test_irregular_blocks_have_no_extra_modules():
    assert not any(m.startswith("down_blocks.3.attentions") for m in lora.UNET_MODULES)
    assert not any(m.startswith("up_blocks.0.attentions") for m in lora.UNET_MODULES)
    assert not any(m.startswith("up_blocks.3.upsamplers") for m in lora.UNET_MODULES)
    assert not any(m.startswith("down_blocks.3.downsamplers") for m in lora.UNET_MODULES)
    assert "down_blocks.0.resnets.0.conv_shortcut" not in lora.UNET_MODULES  # 320 -> 320: no skip conv


@pytest.mark.parametrize("key,msg", [
    ("lora_unet_down_blocks_0_resnets_0_conv1.hada_w1_a", "LoHa / LoKr"),
    ("lora_unet_down_blocks_0_resnets_0_conv1.lokr_w1", "LoHa / LoKr"),
    ("lora_unet_down_blocks_0_resnets_0_conv1.dora_scale", "DoRA"),
    ("lora_unet_input_blocks_1_0_in_layers_2.lora_down.weight", "LDM-style"),
    ("lora_unet_down_blocks_0_norm1.lora_down.weight", "unknown module"),
    ("lora_unet_conv_in.lora_down.weight", "unknown module"),
    ("unet.down_blocks.9.resnets.0.conv1.lora_A.weight", "unknown module"),
    ("lora_te_text_model_embeddings_token_embedding.lora_down.weight", "unknown module"),
    ("lora_unet_down_blocks_0_resnets_0_conv1.weight", "not a lora_down"),
])
def test_rejected_keys(key, msg):
    with pytest.raises(ValueError, match=msg) as e:
        lora.lora_terms({key: np.zeros((1, 1), np.float32)})
    assert repr(key) in str(e.value)  # the whole key, quoted


def test_module_named_twice():
    d = np.zeros((4, 768), np.float32)
    with pytest.raises(ValueError, match="more than once") as e:
        lora.lora_terms({"lora_te_text_model_encoder_layers_0_mlp_fc1.lora_down.weight": d,
                         "text_encoder.text_model.encoder.layers.0.mlp.fc1.lora_A.weight": d})
    assert "'text_encoder.text_model.encoder.layers.0.mlp.fc1.lora_A.weight'" in str(e.value)


def test_missing_half_and_bad_shape():
    with pytest.raises(ValueError, match="needs both"):
        lora.lora_terms({"unet.mid_block.resnets.0.conv1.lora_A.weight": np.zeros((4, 1280 * 9), np.float32)})
    with pytest.raises(ValueError, match="do not fit"):
        lora.lora_terms({"unet.mid_block.resnets.0.conv1.lora_A.weight": np.zeros((4, 1280), np.float32),
                         "unet.mid_block.resnets.0.conv1.lora_B.weight": np.zeros((1280, 4), np.float32)})


# ---------------------------------------------------------------------------------------------------------------- alpha
def test_alpha_over_rank_rule():
    g = np.random.default_rng(3)
    reg = "clip/blocks/3/mlp/fc1/weight"
    down = g.standard_normal((8, 768)).astype(np.float32)
    up = g.standard_normal((3072, 8)).astype(np.float32)
    k = "lora_te_text_model_encoder_layers_3_mlp_fc1"
    (t,) = lora.lora_terms({k + ".lora_down.weight": down, k + ".lora_up.weight": up, k + ".alpha": np.array(4.0, np.float32)})
    assert t[0] == reg and t[3] == 4.0 and lora.lora_scale(t[3], 8) == np.float32(0.5)
    (p,) = lora.lora_terms({"text_encoder.text_model.encoder.layers.3.mlp.fc1.lora_A.weight": down,
                            "text_encoder.text_model.encoder.layers.3.mlp.fc1.lora_B.weight": up})
    assert p[3] == 8.0 and lora.lora_scale(p[3], 8) == np.float32(1.0)  # missing alpha: alpha = r
    assert lora.lora_scale(4.0, 8, multiplier=-0.75) == np.float32(-0.375)
    d = lora.delta(down, up, 4.0, shape=PARAMS[reg])
    np.testing.assert_allclose(d, 0.5 * (up.astype(np.float64) @ down.astype(np.float64)).T)
    # a conv: [r, in, k, k] down and [out, r, 1, 1] up flatten to the OIHW fan-in order
    k = "lora_unet_down_blocks_1_downsamplers_0_conv"
    (c,) = lora.lora_terms({k + ".lora_down.weight": np.ones((2, 640, 3, 3), np.float16),
                            k + ".lora_up.weight": np.ones((640, 2, 1, 1), np.float16)})
    assert c[0] == "unet/input_blocks/d2/weight" and c[1].shape == (2, 5760) and c[2].shape == (640, 2) and c[3] == 2.0


def test_make_lora_is_seeded_and_sized():
    reg = "unet/input_blocks/rt1/transformer/transformer/attn1/query/weight"
    (a,) = synth.make_lora([reg], 16, seed=5)
    (b,) = synth.make_lora([reg], 16, seed=5)
    for x, y in zip(a[1:3], b[1:3]):
        np.testing.assert_array_equal(x, y)
    w = synth.make_tensor(reg, PARAMS[reg], "lin_w", 320, 0)
    d = lora.delta(a[1], a[2], a[3], shape=PARAMS[reg])
    ratio = np.sqrt(np.mean(d ** 2)) / np.sqrt(np.mean(w.astype(np.float64) ** 2))
    assert 0.2 < ratio < 0.4, ratio


# ---------------------------------------------------------------------------------------------------------------- golden
def test_golden_fixture_rederived():
    """tests/golden/lora_b1.npz from its generator: the adapter merged in fp64 into the synthetic weights, the oracle's CLIP,
    4 DDIM steps and decode (about a minute)."""
    import os
    import sys
    import torch
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    sys.path.insert(0, gold)
    import make_lora_golden as MG
    assert os.path.getsize(os.path.join(gold, "lora_b1.npz")) < 1 << 20
    kinds = {r.rsplit("/", 2)[-2] if "/transformer/" not in r else r.split("/transformer/")[-1] for r in MG.LORA_TARGETS}
    assert len(MG.LORA_TARGETS) == len(set(MG.LORA_TARGETS)) == 24 and len(kinds) >= 16
    assert all(r in set(lora.UNET_MODULES.values()) | set(lora.CLIP_MODULES.values()) for r in MG.LORA_TARGETS)
    torch.set_num_threads(os.cpu_count() or 1)
    out = MG.compute()
    g = np.load(os.path.join(gold, "lora_b1.npz"))
    for k in ("tokens", "utokens", "init"):
        assert np.array_equal(out[k], g[k]), k
    rel = lambda a, b: float(np.linalg.norm(np.float64(a) - b) / np.linalg.norm(np.float64(b)))
    for k in ("context", "uncond", "latent"):
        assert rel(out[k], g[k]) < 1e-4, k
    d = np.abs(out["u8"].astype(np.int16) - g["u8"].astype(np.int16))
    assert (d <= 1).mean() >= 0.999 and d.max() <= 2
