"""CPU oracle of image-to-image / masked inpainting (DESIGN.md §7 f5) and the inputs of its fixture — TEST INFRASTRUCTURE ONLY.

The reference has no img2img. The functions below follow the semantics the CUDA path implements, on top of the reference
restatement in oracle/sd_oracle.py (encode_image, forward_diffuser, ddim_timesteps, sample_latent's step arithmetic).
The fixture tests/golden/img2img_b2.npz is written by tests/golden/make_img2img_golden.py from img2img_inputs() and IMG2IMG.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle.sd_oracle import ddim_timesteps, encode_image, forward_diffuser


# Built from the reference's encode_image
# (autoencoder/mod.rs:60-66), the latent scale of latent_to_image (stablediffusion/mod.rs:71) and sample_latent's schedule and
# DDIM step (stablediffusion/mod.rs:123-156). The elementwise formulas are evaluated in numpy float32, one rounding per
# operation (no fused multiply-add), which is what the kernels' __f*_rn intrinsics compute.
def image_u8_to_float(image_u8):
    """u8 [n,H,W,3] HWC RGB -> float32 NCHW [n,3,H,W], x = fl(fl(v / 127.5) - 1): the inverse of latent_to_image's
    (x + 1) / 2 * 255. No reference counterpart (the reference has no image input path)."""
    v = np.ascontiguousarray(np.asarray(image_u8, np.uint8).transpose(0, 3, 1, 2)).astype(np.float32)
    return np.subtract(np.divide(v, np.float32(127.5)), np.float32(1.0))


def mask_to_latent(mask_u8):
    """u8 [n,8H,8W] (255 = regenerate, 0 = keep) -> float32 [n,H,W]: w = fl(S / 16320), S the integer sum of each 8x8 block
    (the area mean of mask / 255). No reference counterpart."""
    m = np.asarray(mask_u8, np.uint8)
    n, hp, wp = m.shape
    S = m.reshape(n, hp // 8, 8, wp // 8, 8).astype(np.int64).sum(axis=(2, 4))
    return np.divide(S.astype(np.float32), np.float32(16320.0))


def img2img_start(strength, n_steps):
    """-> (first schedule index, ts): of the N timesteps of ddim_timesteps(n_steps), the last k = floor(strength * N) run.
    Rejects a strength that is not finite or not in (0, 1], and one that runs no step (below 1/N)."""
    ts, _ = ddim_timesteps(n_steps)
    N = len(ts)
    if not (math.isfinite(strength) and 0.0 < strength <= 1.0):
        raise ValueError("strength must be finite and in (0, 1]")
    k = int(math.floor(strength * N))
    if k == 0:
        raise ValueError(f"strength {strength} runs none of the {N} timesteps; the smallest valid strength is 1/{N}")
    return N - k, ts


def img2img_latent(P, context, uncond, scale, n_steps, image_u8, strength, noise, mask_u8=None, taps=None):
    """Image-to-image (mask_u8 None) or masked inpainting -> the final latent [n,4,H,W] (torch). NOT a reference function: the
    reference has no img2img (see the section comment). noise [n,4,H,W]; taps receives "z0" and, with a mask, "w".
    z0 = fl(encode_image(x) * 0.18215); start at t0 = ts[N-k] from fl(fl(sa z0) + fl(sb noise)), sa = sqrt(abar[t0]),
    sb = sqrt(1 - abar[t0]); each step is sample_latent's, then with a mask x = fl(fl(w nl) + fl(fl(1 - w) known)),
    known = fl(fl(sqrt(a_prev) z0) + fl(sqrt(1 - a_prev) noise))."""
    alphas = P("alpha_cumulative_products").to(torch.float32)
    first, ts = img2img_start(strength, n_steps)
    step = 1000 // n_steps
    x_img = torch.from_numpy(image_u8_to_float(image_u8))
    z0 = np.multiply(encode_image(P, x_img).to(torch.float32).numpy(), np.float32(0.18215))
    eps = np.asarray(noise, np.float32)
    w = mask_to_latent(mask_u8)[:, None] if mask_u8 is not None else None
    if taps is not None:
        taps["z0"] = z0
        if w is not None:
            taps["w"] = w[:, 0]
    a0 = float(alphas[ts[first]])
    sa, sb = np.float32(math.sqrt(a0)), np.float32(math.sqrt(1.0 - a0))
    latent = torch.from_numpy(np.add(np.multiply(sa, z0), np.multiply(sb, eps))).to(P.dtype)
    for t in ts[first:]:
        a_t = float(alphas[t])
        a_prev = float(alphas[t - step]) if t >= step else 1.0
        sqrt_noise = math.sqrt(1.0 - a_t)
        pred = forward_diffuser(P, latent, t, context, uncond, scale)
        predx0 = (latent - pred * sqrt_noise) / math.sqrt(a_t)
        dir_latent = pred * math.sqrt(1.0 - a_prev)
        latent = predx0 * math.sqrt(a_prev) + dir_latent
        if w is not None:
            ka, kb = np.float32(math.sqrt(a_prev)), np.float32(math.sqrt(1.0 - a_prev))
            known = np.add(np.multiply(ka, z0), np.multiply(kb, eps))
            nl = latent.to(torch.float32).numpy()
            latent = torch.from_numpy(np.add(np.multiply(w, nl), np.multiply(np.subtract(np.float32(1.0), w), known))).to(P.dtype)
    return latent


# ------------------------------------------------------------------------------------------------ fixture inputs
def img2img_inputs():
    """Inputs of the img2img fixture: two smooth 256x256 RGB patterns and their masks. Image 0: a rectangle to regenerate whose
    left edge ramps 0 -> 255 over 64 px; image 1: the left half kept, the right half regenerated but for one soft block."""
    y, x = np.mgrid[0:256, 0:256].astype(np.float64)
    img0 = np.stack([128 + 100 * np.sin(x / 23.0), 128 + 90 * np.cos(y / 31.0), 64 + 0.5 * (x + y) / 2], -1)
    r = np.hypot(x - 140, y - 100)
    img1 = np.stack([200 - 0.6 * r, 90 + 80 * np.sin(r / 17.0), 30 + 0.8 * y], -1)
    image = np.clip(np.rint(np.stack([img0, img1])), 0, 255).astype(np.uint8)
    mask = np.zeros((2, 256, 256), np.uint8)
    mask[0, 64:192, 48:208] = 255
    mask[0, 64:192, 48:112] = np.rint(np.linspace(0, 255, 64)).astype(np.uint8)[None, :]
    mask[1, :, 128:] = 255
    mask[1, 100:164, 150:214] = 90
    return image, mask


IMG2IMG = dict(n_steps=4, strength=0.5, scale=5.0)  # k = 2: t = 499, 249
