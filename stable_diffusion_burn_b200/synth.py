"""Deterministic synthetic weights and inputs (no checkpoints exist offline).

Weights are a pure function of (tensor name, element index, seed) through a 32-bit
integer hash, so the numpy generator here and the device generator in
csrc/synth.cu (sdb_init_synthetic) produce bit-identical fp32 values.

  h   = mix32(idx ^ mix32(fnv1a32(name) + seed))
  u   = (h >> 8) * 2^-24                  in [0,1), exact in fp32
  val = (2u - 1) * bound + offset         (fp32 ops, one rounding each)

bound/offset per kind (fan_in = Cin*k*k for conv, in-features for Linear):
  conv_w, lin_w : bound = sqrt(3)/sqrt(fan_in)  (unit-gain uniform), offset 0
  conv_b, lin_b : bound = 1/sqrt(fan_in), offset 0
  norm_g        : bound = 0.1, offset 1
  norm_b        : bound = 0.1, offset 0
  emb           : bound = sqrt(3), offset 0     (token / position embeddings)
"""
from __future__ import annotations

import math
import numpy as np

from . import topology

M32 = np.uint32(0xFFFFFFFF)


def fnv1a32(name: str) -> int:
    h = 0x811C9DC5
    for b in name.encode("utf-8"):
        h ^= b
        h = (h * 0x01000193) & 0xFFFFFFFF
    return h


def _mix32_scalar(x: int) -> int:
    x &= 0xFFFFFFFF
    x ^= x >> 16
    x = (x * 0x85EBCA6B) & 0xFFFFFFFF
    x ^= x >> 13
    x = (x * 0xC2B2AE35) & 0xFFFFFFFF
    x ^= x >> 16
    return x


def _mix32(x: np.ndarray) -> np.ndarray:
    x = x.astype(np.uint32, copy=True)
    x ^= x >> np.uint32(16)
    x *= np.uint32(0x85EBCA6B)
    x ^= x >> np.uint32(13)
    x *= np.uint32(0xC2B2AE35)
    x ^= x >> np.uint32(16)
    return x


def tensor_key(name: str, seed: int) -> int:
    return _mix32_scalar((fnv1a32(name) + seed) & 0xFFFFFFFF)


def uniform01(name: str, count: int, seed: int) -> np.ndarray:
    """fp32 U[0,1) stream for a tensor name."""
    key = np.uint32(tensor_key(name, seed))
    idx = np.arange(count, dtype=np.uint32)
    with np.errstate(over="ignore"):
        h = _mix32(idx ^ key)
    return (h >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)


def kind_bound_offset(kind: str, fan_in: int):
    if kind in ("conv_w", "lin_w"):
        return np.float32(math.sqrt(3.0) / math.sqrt(fan_in)), np.float32(0.0)
    if kind in ("conv_b", "lin_b"):
        return np.float32(1.0 / math.sqrt(fan_in)), np.float32(0.0)
    if kind == "norm_g":
        return np.float32(0.1), np.float32(1.0)
    if kind == "norm_b":
        return np.float32(0.1), np.float32(0.0)
    if kind == "emb":  # unit variance, like burn's N(0,1) embedding initialiser
        return np.float32(math.sqrt(3.0)), np.float32(0.0)
    raise ValueError(kind)


def make_tensor(name: str, shape, kind: str, fan_in: int, seed: int) -> np.ndarray:
    n = int(np.prod(shape))
    u = uniform01(name, n, seed)
    bound, off = kind_bound_offset(kind, fan_in)
    v = (u * np.float32(2.0) - np.float32(1.0)) * bound + off
    return v.astype(np.float32).reshape(shape)


def alpha_cumulative_products() -> np.ndarray:
    """SD-v1 'scaled_linear' schedule: betas = linspace(sqrt(8.5e-4), sqrt(1.2e-2), 1000)^2.

    In the reference this is a loaded Param (stablediffusion/mod.rs:44, load.rs:21); the
    values here are the ones an SD-v1.4 dump would contain (computed in f64, stored f32).
    """
    betas = np.linspace(math.sqrt(0.00085), math.sqrt(0.012), 1000, dtype=np.float64) ** 2
    return np.cumprod(1.0 - betas).astype(np.float32)


def make_params(seed: int = 0, which=None, inpaint=False, pix2pix=False) -> dict:
    """name -> np.float32 array for every tensor on the path (≈3.6 GB fp32 in total). inpaint: the 9-channel registry, pix2pix:
    the 8-channel one; their tensors other than unet/input_blocks/conv/weight equal the 4-channel ones (the stream is keyed by
    name)."""
    plist = topology.all_params(inpaint, pix2pix) if which is None else which
    out = {n: make_tensor(n, s, k, f, seed) for (n, s, k, f) in plist}
    out["alpha_cumulative_products"] = alpha_cumulative_products()
    return out


def realistic_stats(params: dict, seed: int = 7) -> dict:
    """Reshapes the i.i.d. synthetic weights towards the statistics of a trained SD-v1 checkpoint (none exists offline): per
    output channel gains drawn log-normal (sigma 0.5: a few channels 3-5x the rest, i.e. outlier activations), GroupNorm /
    LayerNorm gamma in [0.4, 1.6] and beta in +-0.4, sharper attention logits (query / key weights x 1.7), larger biases.
    A pure function of (name, channel, seed) — the GPU test applies the same transform before sdb_set_tensor."""
    out = {}
    for name, a in params.items():
        a = np.asarray(a, np.float32)
        leaf = name.rsplit("/", 1)[-1]
        parent = name.rsplit("/", 1)[0]
        if name == "alpha_cumulative_products" or "embedding" in name:
            out[name] = a
            continue
        is_norm = any(k in parent.rsplit("/", 1)[-1] for k in ("norm", "_ln", "layer_norm"))
        if is_norm:
            u = uniform01(name + "#r", a.size, seed).reshape(a.shape)
            out[name] = (0.4 + 1.2 * u).astype(np.float32) if leaf == "weight" else ((u * 2 - 1) * np.float32(0.4)).astype(np.float32)
            continue
        if leaf == "weight" and a.ndim in (2, 4):
            n_out = a.shape[1] if a.ndim == 2 else a.shape[0]  # Linear [in,out], conv OIHW
            u1 = uniform01(parent + "#g1", n_out, seed).astype(np.float64)
            u2 = uniform01(parent + "#g2", n_out, seed).astype(np.float64)
            z = np.sqrt(-2.0 * np.log(np.maximum(u1, 1e-7))) * np.cos(2 * np.pi * u2)  # Box-Muller
            g = np.exp(0.5 * z)
            g = (g / np.sqrt(np.mean(g * g))).astype(np.float32)  # unit RMS gain: the layer's output scale is kept
            if parent.endswith(("/query", "/key")):
                g = g * np.float32(1.7)
            out[name] = (a * (g[None, :] if a.ndim == 2 else g[:, None, None, None])).astype(np.float32)
        elif leaf == "bias":
            out[name] = (a * np.float32(3.0)).astype(np.float32)
        else:
            out[name] = a
    return out


def make_lora(targets, rank: int, seed: int = 0, alpha=None) -> list:
    """A seeded synthetic LoRA adapter (DESIGN.md §7 f8): for each registry weight name in `targets`, counter-hash factors
    down [rank][fan-in] ~ U(-1, 1) and up [out][rank] ~ U(-1, 1) * b, with b chosen so that the RMS of s (up . down) is about
    0.3 of the synthetic weight's RMS (1 / sqrt(fan-in)). alpha defaults to rank (s = 1). -> [(name, down, up, alpha)]."""
    shapes = {n: (s, k) for n, s, k, _ in topology.all_params()}
    out = []
    for name in targets:
        shape, kind = shapes[name]
        o, f = (shape[1], shape[0]) if kind == "lin_w" else (shape[0], int(np.prod(shape[1:])))
        a = float(rank if alpha is None else alpha)
        s = a / rank
        b = np.float32(0.3 * 3.0 / (math.sqrt(rank) * math.sqrt(f) * s))  # RMS(up.down) = sqrt(r) * (1/sqrt3) * (b/sqrt3)
        down = (uniform01(name + "#lora_down", rank * f, seed) * np.float32(2.0) - np.float32(1.0)).reshape(rank, f)
        up = ((uniform01(name + "#lora_up", o * rank, seed) * np.float32(2.0) - np.float32(1.0)) * b).reshape(o, rank)
        out.append((name, down.astype(np.float32), up.astype(np.float32), a))
    return out


# ---------------------------------------------------------------- inputs ----
def make_latent(n: int, h: int, w: int, seed: int = 1234) -> np.ndarray:
    """N(0,1) init latent [n,4,h,w]; image i uses stream seed+i (SURVEY §8d)."""
    out = np.empty((n, 4, h, w), np.float32)
    for i in range(n):
        out[i] = np.random.Generator(np.random.Philox(seed + i)).standard_normal((4, h, w), dtype=np.float32)
    return out


def randn_stream(count: int, k0: int, k1: int) -> np.ndarray:
    """The device's counter-hash Box-Muller N(0,1) stream (csrc/kernels.cu: randn_at), element i of `count`:
    u1 = ((mix32(i ^ k0) >> 8) + 1) 2^-24, u2 = (mix32(i * 0x9E3779B9 ^ k1) >> 8) 2^-24, sqrt(-2 ln u1) cos(2 pi u2) in float32.
    u1 and u2 are exact; the device's logf / cosf and numpy's differ by a few ulp."""
    i = np.arange(count, dtype=np.uint64).astype(np.uint32)
    with np.errstate(over="ignore"):
        a = _mix32(i ^ np.uint32(k0))
        b = _mix32((i * np.uint32(0x9E3779B9)) ^ np.uint32(k1))
    u1 = ((a >> np.uint32(8)) + np.uint32(1)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    u2 = (b >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    r = np.sqrt(np.float32(-2.0) * np.log(u1))
    return (r * np.cos(np.float32(6.283185307179586) * u2)).astype(np.float32)


def init_noise_keys(seed: int):
    """Key of the init latent the sampling entries draw for `seed` (csrc/kernels.cu: init_noise_keys)."""
    return ((seed & 0xFFFFFFFF) * 2654435761 + 1) & 0xFFFFFFFF, ((seed >> 32) & 0xFFFFFFFF) ^ 0x5BD1E995


def seeded_latents(seeds, h: int, w: int) -> np.ndarray:
    """The init latents [n,4,h,w] of a batch call (DESIGN.md §7 f7): request i is the stream the device draws for seeds[i] at
    n = 1, element j < 4hw at index j (csrc/kernels.cu: randn_seeds_kernel). To a few ulp, like randn_stream."""
    return np.stack([randn_stream(4 * h * w, *init_noise_keys(int(s))).reshape(4, h, w) for s in seeds])


def step_noise_keys(noise_seed: int, t: int):
    """Key of stochastic DDIM's noise at timestep t (csrc/kernels.cu: step_noise_keys): the init-latent key of noise_seed mixed
    with the timestep value; k1 also takes k0, so that seeds differing in their low word only do not share k1 (the angle of every
    Box-Muller pair)."""
    k0 = (((noise_seed & 0xFFFFFFFF) * 2654435761 + 1) & 0xFFFFFFFF) ^ _mix32_scalar(0x3C6EF372 + t)
    k1 = (((noise_seed >> 32) & 0xFFFFFFFF) ^ 0x5BD1E995) ^ _mix32_scalar(k0 ^ 0xA54FF53A)
    return k0, k1


def step_noise(noise_seed: int, t: int, shape) -> np.ndarray:
    """Stochastic DDIM's per-step noise z [shape] at timestep t, keyed by (noise_seed, t, flat element index in the call's
    [n,4,H,W] latent): a batch member's noise depends on its position in the call. Mirror of sdb_test_step_noise."""
    n = int(np.prod(shape))
    return randn_stream(n, *step_noise_keys(noise_seed, t)).reshape(shape)


def make_context(n: int, L: int, seed: int = 77) -> np.ndarray:
    """Stand-in for CLIP output [n,L,768]: N(0,1) rows normalised to zero mean / unit variance."""
    g = np.random.Generator(np.random.Philox(seed))
    x = g.standard_normal((n, L, 768), dtype=np.float32)
    x = (x - x.mean(-1, keepdims=True)) / x.std(-1, keepdims=True)
    return x.astype(np.float32)


def kat_context() -> np.ndarray:
    """The reference author's eyeball probe: repeat([0.5,1.3],384) as [1,1,768] (python/dump.py:624-633)."""
    return np.tile(np.array([0.5, 1.3], np.float32), 384).reshape(1, 1, 768)


def sin_ramp(shape) -> np.ndarray:
    """RNG-free ramp sin(arange*10/n) (python/test_tiny.py:25)."""
    n = int(np.prod(shape))
    return np.sin(np.arange(n, dtype=np.float32) * np.float32(10.0 / n)).astype(np.float32).reshape(shape)
