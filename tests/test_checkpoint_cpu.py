"""SD-1.x single-file .safetensors checkpoints (DESIGN.md §7 f13), without a GPU: the LDM key map of
tests/golden/ldm_keymap.json.gz (derived from the reference's own converter by tests/ref_shim/make_ckpt_map.py) against the
registry, and sdb_probe_safetensors — the loader's complete validation — on files written by the numpy writer below."""
import gzip
import json
import os
import struct

import numpy as np
import pytest

from stable_diffusion_burn_b200 import _lib, topology

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "tests", "golden", "ldm_keymap.json.gz"), "rb") as _f:
    KEYMAP = json.loads(gzip.decompress(_f.read()))  # LDM key -> [registry name, LDM shape, "copy" | "transpose"]
CONV_IN_KEY = "model.diffusion_model.input_blocks.0.0.weight"
ITEM = {"F32": 4, "F16": 2, "BF16": 2, "F64": 8, "I64": 8, "U8": 1}


# ------------------------------------------------------------------------------------------------------------ the writer
def ldm_entries(width=4, vae_only=False, old_clip=False):
    """[(LDM key, registry name, LDM shape, transposed)] of a full checkpoint with a `width`-channel conv_in, or of a VAE-only
    file (the autoencoder keys without first_stage_model.)."""
    out = []
    for key, (reg, shape, op) in KEYMAP.items():
        if key == CONV_IN_KEY:
            shape = [320, width, 3, 3]
        if vae_only:
            if not key.startswith("first_stage_model."):
                continue
            key = key[len("first_stage_model."):]
        elif old_clip:
            key = key.replace("cond_stage_model.transformer.text_model.", "cond_stage_model.transformer.")
        out.append((key, reg, tuple(shape), op == "transpose"))
    return out


def encode(a, dtype):
    """the little-endian bytes of fp32 array `a` stored as `dtype` (BF16: the upper half of each fp32, i.e. truncated)"""
    a = np.ascontiguousarray(a, np.float32)
    if dtype == "F32":
        return a.astype("<f4").tobytes()
    if dtype == "F16":
        return a.astype("<f2").tobytes()
    if dtype == "BF16":
        return (a.view(np.uint32) >> np.uint32(16)).astype("<u2").tobytes()
    raise ValueError(dtype)


def widened(a, dtype):
    """what the loader makes of encode(a, dtype): numpy's exact widening to fp32"""
    a = np.ascontiguousarray(a, np.float32)
    if dtype == "F16":
        return a.astype(np.float16).astype(np.float32)
    if dtype == "BF16":
        return ((a.view(np.uint32) >> np.uint32(16)) << np.uint32(16)).view(np.float32)
    return a


def write_safetensors(path, tensors, data_order=None, metadata=None):
    """tensors: [(key, dtype, shape, fp32 array or raw bytes or None)]. The header lists them in order; their data lies in
    `data_order` (keys; default: header order). None writes no bytes: the file is extended with truncate, so a body that is
    mostly None stays sparse on disk and reads as zeros."""
    size = {k: int(np.prod(s, dtype=np.int64)) * ITEM.get(dt, 1) for k, dt, s, _ in tensors}  # other dtypes: 1 byte each
    offs, off = {}, 0
    for k in data_order or [t[0] for t in tensors]:
        offs[k] = (off, off + size[k])
        off += size[k]
    header = {"__metadata__": metadata} if metadata is not None else {}
    for k, dt, s, _ in tensors:
        header[k] = {"dtype": dt, "shape": list(s), "data_offsets": list(offs[k])}
    hb = json.dumps(header).encode()
    hb += b" " * (-len(hb) % 8)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(hb)) + hb)
        base = 8 + len(hb)
        for k, dt, _, a in tensors:
            if a is not None:
                f.seek(base + offs[k][0])
                f.write(a if isinstance(a, bytes) else encode(a, dt))
        f.truncate(base + off)
    return str(path)


def read_header(path):
    with open(path, "rb") as f:
        (n,) = struct.unpack("<Q", f.read(8))
        h = json.loads(f.read(n))
    h.pop("__metadata__", None)
    return h


def write_raw(path, header: bytes, body_bytes=0, hlen=None):
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(header) if hlen is None else hlen) + header)
        f.truncate(8 + len(header) + body_bytes)
    return str(path)


def sparse_checkpoint(path, width=4, dtype="F16", extra=(), drop=(), change=None, metadata=None, **kw):
    """a full (or VAE-only) checkpoint header over a sparse body; extra: more (key, dtype, shape, data) entries; drop: keys to
    leave out; change: {key: (dtype, shape)}"""
    change = change or {}
    t = [(k, *change.get(k, (dtype, s)), None) for k, _, s, _ in ldm_entries(width, **kw) if k not in drop]
    return write_safetensors(path, t + list(extra), metadata=metadata)


# ------------------------------------------------------------------------------------------------------------ the map
def test_keymap_covers_the_registry_once():
    reg = {n: (tuple(s), k) for n, s, k, _ in topology.all_params()}
    seen = {}
    for key, (name, shape, op) in KEYMAP.items():
        assert name in reg, (key, name)
        assert name not in seen, (name, key, seen.get(name))
        seen[name] = key
        rshape, kind = reg[name]
        assert op == ("transpose" if kind == "lin_w" else "copy"), (key, op, kind)
        assert tuple(shape) == (rshape[::-1] if op == "transpose" else rshape), (key, shape, rshape)
    assert set(seen) == set(reg), set(reg) - set(seen)
    assert len(KEYMAP) == 1130 and "alpha_cumulative_products" not in seen
    # the irregular parts of the LDM layout
    assert KEYMAP["first_stage_model.decoder.up.3.block.0.conv1.weight"][0] == "autoencoder/decoder/blocks/0/res1/conv1/weight"
    assert KEYMAP["first_stage_model.decoder.up.1.upsample.conv.weight"][0] == "autoencoder/decoder/blocks/2/upsampler/weight"
    for key, reg_ in (("output_blocks.2.1.conv", "output_blocks/ru/upsample/conv"),
                      ("output_blocks.5.2.conv", "output_blocks/rtu1/upsample/conv"),
                      ("output_blocks.8.2.conv", "output_blocks/rtu2/upsample/conv"),
                      ("input_blocks.3.0.op", "input_blocks/d1"), ("input_blocks.6.0.op", "input_blocks/d2"),
                      ("input_blocks.9.0.op", "input_blocks/d3"), ("time_embed.0", "lin1_time_embed"),
                      ("time_embed.2", "lin2_time_embed"), ("out.0", "norm_out"), ("out.2", "conv_out")):
        assert KEYMAP[f"model.diffusion_model.{key}.weight"][0] == f"unet/{reg_}/weight"


# ------------------------------------------------------------------------------------------------------------ probing
@pytest.mark.parametrize("width", [4, 8, 9])
def test_probe_full_checkpoint(tmp_path, width):
    f = sparse_checkpoint(tmp_path / "m.safetensors", width)
    assert _lib.probe_safetensors(f) == (_lib.CKPT_FULL, width)


def test_probe_vae_only_and_old_clip_spelling(tmp_path):
    f = sparse_checkpoint(tmp_path / "vae.safetensors", vae_only=True,
                          extra=[("loss.logvar", "F32", (), None), ("loss.discriminator.main.0.weight", "F16", (64, 3, 4, 4), None)])
    assert _lib.probe_safetensors(f) == (_lib.CKPT_VAE, 0)
    f = sparse_checkpoint(tmp_path / "old.safetensors", old_clip=True, metadata={"format": "pt"})
    assert _lib.probe_safetensors(f) == (_lib.CKPT_FULL, 4)


def test_ignored_keys_are_parsed_not_mapped(tmp_path):
    extra = [("model_ema.diffusion_modeltime_embed0weight", "F32", (1280, 320), None), ("model_ema.num_updates", "I64", (), None),
             ("cond_stage_model.transformer.text_model.embeddings.position_ids", "I64", (1, 77), None),
             ("betas", "F64", (1000,), None), ("first_stage_model.loss.logvar", "F32", (), None),
             ("alphas_cumprod", "F16", (1000,), None), ("some.other", "F4_E2M1", (3,), None)]
    f = sparse_checkpoint(tmp_path / "m.safetensors", dtype="BF16", extra=extra)
    assert _lib.probe_safetensors(f) == (_lib.CKPT_FULL, 4)


def _rejects(f, *needles):
    with pytest.raises(_lib.SdbError) as e:
        _lib.probe_safetensors(f)
    msg = str(e.value)
    for n in needles:
        assert n in msg, (n, msg)
    return msg


def test_errors_name_the_key(tmp_path):
    p = lambda name: tmp_path / name
    k_bias = "model.diffusion_model.out.2.bias"
    k_q = "cond_stage_model.transformer.text_model.encoder.layers.3.self_attn.q_proj.weight"
    _rejects(sparse_checkpoint(p("unmapped"), extra=[("model.diffusion_model.foo.weight", "F16", (3,), None)]),
             "model.diffusion_model.foo.weight")
    _rejects(sparse_checkpoint(p("unmapped_vae"), vae_only=True, extra=[("decoder.mid.attn_2.q.weight", "F16", (3,), None)]),
             "decoder.mid.attn_2.q.weight")
    _rejects(sparse_checkpoint(p("missing"), drop=[k_bias]), "missing", k_bias, "unet/conv_out/bias")
    _rejects(sparse_checkpoint(p("shape"), change={k_q: ("F16", (768, 769))}), k_q, "[768,769]", "[768,768]")
    _rejects(sparse_checkpoint(p("dtype"), change={k_q: ("F64", (768, 768))}), k_q, "F64")
    _rejects(sparse_checkpoint(p("sched"), extra=[("alphas_cumprod", "F32", (999,), None)]), "alphas_cumprod", "[999]")
    _rejects(sparse_checkpoint(p("twice"), extra=[(k_q.replace("text_model.", ""), "F16", (768, 768), None)]),
             "given twice", k_q)
    _rejects(sparse_checkpoint(p("width"), width=5), CONV_IN_KEY, "[320,5,3,3]")
    _rejects(sparse_checkpoint(p("sd2"), extra=[("cond_stage_model.model.ln_final.weight", "F16", (1024,), None)]),
             "cond_stage_model.model.ln_final.weight", "SD-2")
    _rejects(sparse_checkpoint(p("sdxl"), extra=[("conditioner.embedders.0.transformer.x", "F16", (4,), None)]),
             "conditioner.embedders.0.transformer.x", "SDXL")
    # a truncated file: the tensors past the new end lie outside it
    f = sparse_checkpoint(p("trunc"))
    os.truncate(f, os.path.getsize(f) - 1000)
    header = read_header(f)
    last = max(header, key=lambda k: header[k]["data_offsets"][1])
    _rejects(f, last, "outside")


def _one(dtype="F32", shape=(2,), offs=(0, 8), key="model.diffusion_model.out.2.bias"):
    return json.dumps({key: {"dtype": dtype, "shape": list(shape), "data_offsets": list(offs)}}).encode()


def test_malformed_headers(tmp_path):
    p = lambda name: str(tmp_path / name)
    k = "model.diffusion_model.out.2.bias"
    with open(p("short"), "wb") as f:
        f.write(b"\x10\x00\x00")
    _rejects(p("short"), "shorter than the header length")
    _rejects(write_raw(p("past"), b"{}", hlen=4096), "4096", "past the end")
    _rejects(write_raw(p("limit"), b"{}", hlen=100 * 2**20 + 1), str(100 * 2**20 + 1), "100 MB")
    _rejects(write_raw(p("nonjson"), b"not json at all!"), "malformed")
    _rejects(write_raw(p("trailing"), _one() + b" x", 8), "trailing")
    _rejects(write_raw(p("array"), b"[1, 2]"), "malformed")
    _rejects(write_raw(p("nested"), json.dumps({k: {"dtype": "F32", "shape": [2], "data_offsets": [0, 8],
                                                    "extra": {"a": 1}}}).encode(), 8), k, "extra")
    _rejects(write_raw(p("nested_shape"), json.dumps({k: {"dtype": "F32", "shape": [[2]], "data_offsets": [0, 8]}}).encode(), 8),
             k, "shape")
    _rejects(write_raw(p("meta"), json.dumps({"__metadata__": {"a": {"b": "c"}}}).encode()), "__metadata__")
    _rejects(write_raw(p("float"), _one(shape=(2.0,)), 8), k, "integer")
    _rejects(write_raw(p("neg"), _one(offs=(-8, 0)), 8), k, "negative")
    _rejects(write_raw(p("overflow"), _one().replace(b"[0, 8]", b"[0, 99999999999999999999]"), 8), k, "overflow")
    _rejects(write_raw(p("outside"), _one(offs=(8, 16)), 8), k, "outside")
    _rejects(write_raw(p("size"), _one(offs=(0, 6)), 8), k, "6 bytes", "8 bytes")
    _rejects(write_raw(p("dup"), b'{"a": {"dtype": "F32", "shape": [], "data_offsets": [0, 4]}, "a": '
                                 b'{"dtype": "F32", "shape": [], "data_offsets": [0, 4]}}', 4), "a given twice")
    _rejects(write_raw(p("nomodel"), _one(key="foo"), 8), "no SD-1.x checkpoint keys")
