"""The image and mask conversions of image-to-image / masked inpainting (DESIGN.md §7 f5) and the inputs of its fixture — TEST
INFRASTRUCTURE ONLY.

The reference has no img2img. Its oracle is tests/sampler_oracle.py: sampler_img2img_latent, built from the reference's
encode_image (autoencoder/mod.rs:60-66), the latent scale of latent_to_image (stablediffusion/mod.rs:71) and sample_latent's
schedule and DDIM step (stablediffusion/mod.rs:123-156), on the conversions below. The elementwise formulas are evaluated in
numpy float32, one rounding per operation (no fused multiply-add), which is what the kernels' __f*_rn intrinsics compute.
The fixture tests/golden/img2img_b2.npz is written by tests/golden/make_img2img_golden.py from img2img_inputs() and IMG2IMG.
"""
from __future__ import annotations

import numpy as np


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
