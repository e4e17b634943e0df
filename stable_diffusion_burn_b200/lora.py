"""LoRA adapter files (DESIGN.md §7 f8): a dependency-free safetensors reader and the map from the kohya and diffusers/PEFT
key conventions to this project's registry names.

Supported conventions (restated from the kohya-ss and diffusers/PEFT layouts; no real adapter file exists offline):
  kohya   lora_unet_<module with '.' -> '_'>.lora_down.weight / .lora_up.weight / .alpha, lora_te_<CLIP module ...>
  PEFT    unet.<module>.lora_A.weight / .lora_B.weight, text_encoder.<module>...; a missing alpha means alpha = r
<module> is a path of the diffusers module tree (UNet2DConditionModel / CLIPTextModel). down is [r][fan-in] (a conv's
[r][in][k][k] flattens to OIHW order), up is [out][r] (or [out][r][1][1]). LoHa, LoKr, DoRA and the LDM-style
lora_unet_input_blocks_* names are rejected by key.
"""
from __future__ import annotations

import json
import struct

import numpy as np

from . import topology

# ------------------------------------------------------------------------------------------------------------------ reader
_DTYPES = {"F32": (np.float32, 4), "F16": (np.float16, 2), "BF16": (np.uint16, 2)}


def read_safetensors(path) -> dict:
    """name -> numpy array of a .safetensors file: F32 as float32, F16 as float16, BF16 widened exactly to float32. Other
    dtypes raise, naming the tensor."""
    with open(path, "rb") as f:
        data = f.read()
    if len(data) < 8:
        raise ValueError(f"{path}: not a safetensors file (shorter than its header length)")
    (hlen,) = struct.unpack("<Q", data[:8])
    if 8 + hlen > len(data):
        raise ValueError(f"{path}: header length {hlen} runs past the end of the file")
    header = json.loads(data[8:8 + hlen].decode("utf-8"))
    body = memoryview(data)[8 + hlen:]
    out = {}
    for name, info in header.items():
        if name == "__metadata__":
            continue
        dt = info["dtype"]
        if dt not in _DTYPES:
            raise ValueError(f"{path}: tensor {name} has dtype {dt}; supported: F32, F16, BF16")
        np_t, size = _DTYPES[dt]
        shape = tuple(int(s) for s in info["shape"])
        b, e = (int(x) for x in info["data_offsets"])
        if e - b != size * int(np.prod(shape, dtype=np.int64)) or e > len(body):
            raise ValueError(f"{path}: tensor {name}: data_offsets {b}..{e} do not hold {dt} {list(shape)}")
        a = np.frombuffer(body[b:e], dtype=np.dtype(np_t).newbyteorder("<")).reshape(shape)
        if dt == "BF16":
            a = (a.astype(np.uint32) << np.uint32(16)).view(np.float32)
        out[name] = a.astype(a.dtype.newbyteorder("="), copy=True)
    return out


# ------------------------------------------------------------------------------------------------------------ module table
_RESNET = {"conv1": "conv_in", "conv2": "conv_out", "conv_shortcut": "skip_connection", "time_emb_proj": "lin_embed"}
_ATTN = {"proj_in": "proj_in", "proj_out": "proj_out", "transformer_blocks.0.ff.net.0.proj": "transformer/mlp/geglu/proj",
         "transformer_blocks.0.ff.net.2": "transformer/mlp/lin"}
for _a in ("attn1", "attn2"):
    for _d, _r in (("to_q", "query"), ("to_k", "key"), ("to_v", "value"), ("to_out.0", "out")):
        _ATTN[f"transformer_blocks.0.{_a}.{_d}"] = f"transformer/{_a}/{_r}"
_CLIP = {"self_attn.q_proj": "attn/query", "self_attn.k_proj": "attn/key", "self_attn.v_proj": "attn/value",
         "self_attn.out_proj": "attn/out", "mlp.fc1": "mlp/fc1", "mlp.fc2": "mlp/fc2"}

# diffusers block -> (registry prefix of resnets.j, of attentions.j, of upsamplers.0 / downsamplers.0)
_I, _O = "unet/input_blocks", "unet/output_blocks"
_UNET_BLOCKS = {
    "down_blocks.0": ([f"{_I}/rt1/res", f"{_I}/rt2/res"], [f"{_I}/rt1/transformer", f"{_I}/rt2/transformer"],
                      ("downsamplers.0.conv", f"{_I}/d1")),
    "down_blocks.1": ([f"{_I}/rt3/res", f"{_I}/rt4/res"], [f"{_I}/rt3/transformer", f"{_I}/rt4/transformer"],
                      ("downsamplers.0.conv", f"{_I}/d2")),
    "down_blocks.2": ([f"{_I}/rt5/res", f"{_I}/rt6/res"], [f"{_I}/rt5/transformer", f"{_I}/rt6/transformer"],
                      ("downsamplers.0.conv", f"{_I}/d3")),
    "down_blocks.3": ([f"{_I}/r1", f"{_I}/r2"], [], None),
    "mid_block": (["unet/middle_block/res1", "unet/middle_block/res2"], ["unet/middle_block/transformer"], None),
    "up_blocks.0": ([f"{_O}/r1", f"{_O}/r2", f"{_O}/ru/res"], [], ("upsamplers.0.conv", f"{_O}/ru/upsample/conv")),
    "up_blocks.1": ([f"{_O}/rt1/res", f"{_O}/rt2/res", f"{_O}/rtu1/res"],
                    [f"{_O}/rt1/transformer", f"{_O}/rt2/transformer", f"{_O}/rtu1/transformer"],
                    ("upsamplers.0.conv", f"{_O}/rtu1/upsample/conv")),
    "up_blocks.2": ([f"{_O}/rt3/res", f"{_O}/rt4/res", f"{_O}/rtu2/res"],
                    [f"{_O}/rt3/transformer", f"{_O}/rt4/transformer", f"{_O}/rtu2/transformer"],
                    ("upsamplers.0.conv", f"{_O}/rtu2/upsample/conv")),
    "up_blocks.3": ([f"{_O}/rt5/res", f"{_O}/rt6/res", f"{_O}/rt7/res"],
                    [f"{_O}/rt5/transformer", f"{_O}/rt6/transformer", f"{_O}/rt7/transformer"], None),
}


def _build_modules():
    params = {n: s for n, s, _, _ in topology.all_params()}
    unet, clip = {}, {}

    def put(table, module, reg):
        if f"{reg}/weight" in params:  # a ResBlock without a channel change has no skip_connection
            table[module] = f"{reg}/weight"

    for blk, (resnets, attns, resample) in _UNET_BLOCKS.items():
        for j, reg in enumerate(resnets):
            for d, r in _RESNET.items():
                put(unet, f"{blk}.resnets.{j}.{d}", f"{reg}/{r}")
        for j, reg in enumerate(attns):
            for d, r in _ATTN.items():
                put(unet, f"{blk}.attentions.{j}.{d}", f"{reg}/{r}")
        if resample:
            put(unet, f"{blk}.{resample[0]}", resample[1])
    for i in range(topology.CLIP_LAYERS):
        for d, r in _CLIP.items():
            put(clip, f"text_model.encoder.layers.{i}.{d}", f"clip/blocks/{i}/{r}")
    return unet, clip, params


UNET_MODULES, CLIP_MODULES, _PARAMS = _build_modules()  # diffusers module path -> registry weight name
_KOHYA = {**{"lora_unet_" + m.replace(".", "_"): r for m, r in UNET_MODULES.items()},
          **{"lora_te_" + m.replace(".", "_"): r for m, r in CLIP_MODULES.items()}}
_PEFT = {**{"unet." + m: r for m, r in UNET_MODULES.items()}, **{"text_encoder." + m: r for m, r in CLIP_MODULES.items()}}
_SUFFIXES = {".lora_down.weight": "down", ".lora_up.weight": "up", ".lora_A.weight": "down", ".lora_B.weight": "up",
             ".alpha": "alpha"}
_LDM_PREFIXES = ("lora_unet_input_blocks_", "lora_unet_middle_block_", "lora_unet_output_blocks_", "lora_unet_out_",
                 "lora_unet_time_embed_")


def kohya_names() -> dict:
    """kohya module name -> registry weight name, for every target."""
    return dict(_KOHYA)


def peft_names() -> dict:
    """PEFT module name (unet.* / text_encoder.*) -> registry weight name, for every target."""
    return dict(_PEFT)


def registry_name(module: str) -> str:
    """Registry weight name of a kohya or PEFT module name (no suffix); raises ValueError naming an unknown module."""
    r = _KOHYA.get(module) or _PEFT.get(module)
    if r is None:
        raise ValueError(f"LoRA key {module!r}: unknown module (no SD-v1 UNet / CLIP target of that name)")
    return r


def lora_scale(alpha, rank, multiplier=1.0) -> np.float32:
    """The scale the device applies to a term: (float)(multiplier * alpha / r), computed in double."""
    return np.float32(float(multiplier) * float(alpha) / int(rank))


def lora_terms(tensors: dict) -> list:
    """Adapter file tensors -> [(registry weight name, down [r, fan-in] f32, up [out, r] f32, alpha)], sorted by registry name.
    A missing alpha means alpha = r. Unsupported or unknown keys raise ValueError naming the key."""
    mods = {}
    for key, a in tensors.items():
        if any(s in key for s in ("hada_", "lokr_")):
            raise ValueError(f"LoRA key {key!r}: LoHa / LoKr adapters are not supported")
        if "dora_scale" in key:
            raise ValueError(f"LoRA key {key!r}: DoRA adapters are not supported")
        if key.startswith(_LDM_PREFIXES):
            raise ValueError(f"LoRA key {key!r}: LDM-style module names are not supported (use the diffusers-style kohya "
                             "names lora_unet_down_blocks_* / lora_unet_up_blocks_* / lora_unet_mid_block_*)")
        suf = next((s for s in _SUFFIXES if key.endswith(s)), None)
        if suf is None:
            raise ValueError(f"LoRA key {key!r}: not a lora_down / lora_up / lora_A / lora_B weight or an alpha")
        module = key[:-len(suf)]
        try:
            reg = registry_name(module)
        except ValueError:
            raise ValueError(f"LoRA key {key!r}: unknown module {module!r} (no SD-v1 UNet / CLIP target of that name)") from None
        m = mods.setdefault(reg, {"key": module})
        if _SUFFIXES[suf] in m:
            raise ValueError(f"LoRA key {key!r}: names the {_SUFFIXES[suf]} of {reg} more than once (also as {m['key']!r})")
        m[_SUFFIXES[suf]] = np.asarray(a)
    out = []
    for reg, m in sorted(mods.items()):
        if "down" not in m or "up" not in m:
            raise ValueError(f"LoRA module {m['key']!r}: needs both a down (lora_down / lora_A) and an up (lora_up / lora_B) "
                             "weight")
        down = m["down"].astype(np.float32)
        up = m["up"].astype(np.float32)
        r = down.shape[0]
        down = down.reshape(r, -1)
        up = up.reshape(up.shape[0], -1)
        shape = _PARAMS[reg]
        out_dim, fan_in = (shape[1], shape[0]) if len(shape) == 2 else (shape[0], int(np.prod(shape[1:])))
        if down.shape[1] != fan_in or up.shape != (out_dim, r):
            raise ValueError(f"LoRA module {m['key']!r}: down {list(m['down'].shape)} / up {list(m['up'].shape)} do not fit "
                             f"{reg} ({out_dim} outputs, fan-in {fan_in})")
        alpha = float(np.asarray(m["alpha"], np.float64).reshape(-1)[0]) if "alpha" in m else float(r)
        if not (np.isfinite(alpha) and alpha > 0):
            raise ValueError(f"LoRA module {m['key']!r}: alpha {alpha} must be finite and > 0")
        out.append((reg, down, up, alpha))
    return out


def delta(down, up, alpha, multiplier=1.0, shape=None) -> np.ndarray:
    """fp64 s (up . down) in the registry layout of a weight of `shape` ([in, out] Linear: transposed; OIHW conv)."""
    s = float(multiplier) * float(alpha) / down.shape[0]
    d = s * (np.asarray(up, np.float64) @ np.asarray(down, np.float64))  # [out, fan-in]
    if shape is None:
        return d
    return d.T.reshape(shape) if len(shape) == 2 else d.reshape(shape)
