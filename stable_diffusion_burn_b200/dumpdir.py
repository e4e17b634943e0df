"""Dump-dir weight format of the reference (SURVEY §8f row f2): writer and numpy reader.

Layout (writer python/save.py, reader src/model/load.rs:17-160): a directory tree whose directory names are the Rust
field names; every tensor is a 1-D float32 .npy holding [dims..., values...] (save.py:10-15), every scalar is
[1.0, value] (save.py:6-8). Linear weights are stored [in,out] (save.py:19), conv weights OIHW together with
stride/padding/dilation/kernel_size/n_group/n_channels_in/n_channels_out (save.py:52-68); norms carry eps (+ n_group,
n_channel for GroupNorm); attention blocks carry n_head; clip/ carries n_layer; the root carries n_steps and
alphas_cumprod (src/model/stablediffusion/load.rs:20-21).

The CUDA library reads this tree natively (sdb_load_dump_dir, csrc/dumpdir.cu). This module is the other direction
(parameter dict -> tree, used by the tests and to convert any name->array dict into the reference's format) plus a
plain numpy reader for the CPU oracle.
"""
from __future__ import annotations

import os

import numpy as np

from . import topology

SCHEDULE_FILE = "alphas_cumprod"
SCHEDULE_NAME = "alpha_cumulative_products"


def save_scalar(value, name: str, path: str) -> None:
    np.save(os.path.join(path, name + ".npy"), np.array([1.0, float(value)], np.float32))


def save_tensor(array, name: str, path: str) -> None:
    a = np.asarray(array, np.float32)
    np.save(os.path.join(path, name + ".npy"),
            np.concatenate([np.asarray(a.shape, np.float32), a.reshape(-1)]).astype(np.float32))


def read_tensor(file: str) -> np.ndarray:
    """[dims..., values...] -> array; the rank is not stored, so it is inferred as the only D with prod(v[:D]) == len - D
    (the reference knows D statically, load.rs:17-28)."""
    v = np.load(file)
    if v.dtype != np.float32 or v.ndim != 1:
        raise ValueError(f"{file}: dump-dir tensors are 1-D float32")
    for d in range(1, 5):
        dims = v[:d]
        if np.all(dims == np.floor(dims)) and np.all(dims >= 0) and int(np.prod(dims.astype(np.int64))) == v.size - d:
            return v[d:].reshape(dims.astype(np.int64))
    raise ValueError(f"{file}: no leading shape matches the payload length")


CONV_IN = "unet/input_blocks/conv/weight"


def _norm_dirs():
    """(dir, channels, is_group_norm) for every norm on the path."""
    out = []
    for n, s, k, _ in topology.all_params():
        if k == "norm_g":
            d = n.rsplit("/", 1)[0]
            layer = ("/transformer/norm1", "/transformer/norm2", "/transformer/norm3")
            is_ln = d.endswith(layer) or d.startswith("clip/")
            out.append((d, s[0], not is_ln))
    return out


def conv_stride(name: str) -> int:
    """Stride of the conv whose weight tensor is `name`: the three UNet downsamplers are stride 2 (unet/mod.rs:44-53)."""
    d = name.rsplit("/", 1)[0]
    return 2 if d in ("unet/input_blocks/d1", "unet/input_blocks/d2", "unet/input_blocks/d3") else 1


def save_dump_dir(root: str, params: dict, eps: float | dict = 1e-5) -> None:
    """Writes `params` (registry name -> array, incl. "alpha_cumulative_products") as the reference's dump-dir; a 9- or
    8-channel conv_in writes the inpainting (DESIGN.md §7 f9) or InstructPix2Pix (f10) registry."""
    width = np.shape(params[CONV_IN])[1] if CONV_IN in params else 4
    eps_of = (lambda d: eps.get(d, 1e-5)) if isinstance(eps, dict) else (lambda d: eps)
    os.makedirs(root, exist_ok=True)
    save_scalar(1000, "n_steps", root)
    save_tensor(params[SCHEDULE_NAME], SCHEDULE_FILE, root)
    for name, shape, kind, _ in topology.conv_in_width_params(width):
        if name not in params:
            continue  # optional tensor left out on purpose (bias / GroupNorm affine)
        d, leaf = name.rsplit("/", 1)
        path = os.path.join(root, d)
        os.makedirs(path, exist_ok=True)
        a = np.asarray(params[name], np.float32)
        assert tuple(a.shape) == tuple(shape), name
        save_tensor(a, leaf, path)
        if kind == "conv_w":
            cout, cin, k, _ = shape
            s = conv_stride(name)
            pad = k // 2
            if d.endswith("/downsampler/conv"):  # save_padded_conv2d (python/save.py:70-97): inner conv saved with padding (0,0)
                s, pad = 2, 0
                outer = os.path.dirname(path)
                save_tensor(np.array([cin, cout], np.float32), "channels", outer)
                save_scalar(k, "kernel_size", outer)
                save_scalar(2, "stride", outer)
                save_tensor(np.array([0, 1, 0, 1], np.float32), "padding", outer)
            for fname, val in (("stride", s), ("padding", pad), ("dilation", 1), ("kernel_size", k)):
                save_tensor(np.array([val, val], np.float32), fname, path)
            save_scalar(1, "n_group", path)
            save_scalar(cin, "n_channels_in", path)
            save_scalar(cout, "n_channels_out", path)
    for d, c, group in _norm_dirs():
        path = os.path.join(root, d)
        os.makedirs(path, exist_ok=True)
        save_scalar(eps_of(d), "eps", path)
        if group:
            save_scalar(32, "n_group", path)
            save_scalar(c, "n_channel", path)
    for name, _, _, _ in topology.all_params():
        if name.endswith("/query/weight"):
            d = name[: -len("/query/weight")]
            os.makedirs(os.path.join(root, d), exist_ok=True)
            save_scalar(12 if d.startswith("clip/") else 8, "n_head", os.path.join(root, d))
    for d in ("clip", "autoencoder/decoder", "autoencoder/encoder"):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    save_scalar(4, "n_block", os.path.join(root, "autoencoder/encoder"))
    save_scalar(12, "n_layer", os.path.join(root, "clip"))
    save_scalar(4, "n_block", os.path.join(root, "autoencoder/decoder"))


def load_dump_dir(root: str) -> dict:
    """numpy reader (for the oracle): registry name -> array, optional tensors filled like the reference does. A 9- or
    8-channel conv_in reads the inpainting or InstructPix2Pix registry."""
    out = {SCHEDULE_NAME: read_tensor(os.path.join(root, SCHEDULE_FILE + ".npy"))}
    group = {d for d, _, g in _norm_dirs() if g}
    conv_in = os.path.join(root, CONV_IN + ".npy")
    width = read_tensor(conv_in).shape[1] if os.path.exists(conv_in) else 4
    for name, shape, kind, _ in topology.conv_in_width_params(width):
        f = os.path.join(root, name + ".npy")
        if os.path.exists(f):
            a = read_tensor(f)
            if tuple(a.shape) != tuple(shape):
                raise ValueError(f"{f}: shape {a.shape} != {shape}")
            out[name] = a
        elif kind in ("conv_b", "lin_b") or (kind == "norm_b" and name.rsplit("/", 1)[0] in group):
            out[name] = np.zeros(shape, np.float32)
        elif kind == "norm_g" and name.rsplit("/", 1)[0] in group:
            out[name] = np.ones(shape, np.float32)
        else:
            raise FileNotFoundError(f)
    return out
