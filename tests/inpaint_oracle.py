"""CPU oracle of inpainting with a 9-channel UNet (DESIGN.md §7 f9) and the cases of its fixture — TEST INFRASTRUCTURE ONLY.

An inpainting checkpoint's UNet reads cat(x_t, latent mask, masked-image latent) (the order of diffusers' inpainting pipeline and
of the original LDM LatentInpaintDiffusion). The reference has no such model; the functions below follow the semantics the CUDA
path implements, on top of tests/img2img_oracle.py (conversion), tests/sampler_oracle.py (strength rule, z0, start latent, the
step loop) and oracle/sd_oracle.py (encode_image, forward_diffuser, whose UNet takes whatever conv_in holds). Elementwise rules
are evaluated in numpy float32, one rounding per operation. The fixture tests/golden/inpaint_b2.npz is written by
tests/golden/make_inpaint_golden.py from img2img_inputs() and INPAINT_CASES.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.sd_oracle import encode_image, forward_diffuser

import img2img_oracle as IO
import sampler_oracle as SO


def binary_mask(mask_u8):
    """u8 [n,8H,8W] -> bool, m = (mask >= 128): diffusers' mask >= 0.5 on mask / 255."""
    return np.asarray(mask_u8, np.uint8) >= 128


def latent_mask(mask_u8):
    """float32 [n,H,W]: the nearest pick m[8h][8w] (F.interpolate(mask, size=(H, W)) in its default nearest mode)."""
    return binary_mask(mask_u8)[:, ::8, ::8].astype(np.float32)


def masked_image(image_u8, mask_u8):
    """float32 NCHW [n,3,8H,8W]: x = fl(fl(v / 127.5) - 1), exactly 0 where the mask regenerates."""
    x = IO.image_u8_to_float(image_u8)
    return np.where(binary_mask(mask_u8)[:, None], np.float32(0.0), x).astype(np.float32)


def inpaint_cond(P, image_u8, mask_u8):
    """The UNet's extra input channels [n,5,H,W]: the latent mask, then z_m = fl(encode_image(x_m) * 0.18215)."""
    z_m = SO.scaled_latent(encode_image(P, torch.from_numpy(masked_image(image_u8, mask_u8))))
    return np.concatenate([latent_mask(mask_u8)[:, None], z_m], 1)


def inpaint_latent(P, context, uncond, scale, n_steps, image_u8, strength, noise, mask_u8, kind=SO.DDIM, eta=0.0, noise_seed=0,
                   taps=None):
    """Inpainting with a 9-channel UNet -> the final latent [n,4,H,W] (torch). P holds a [320,9,3,3] conv_in. The start latent,
    the strength rule and z0 (the unmasked image) are img2img's; both CFG halves of every step read cat(x_t, cond); the step is
    the sampler's update with no blend. taps receives "z0", "m_lat" and "z_m"."""
    if mask_u8 is None:
        raise ValueError("inpainting with a 9-channel UNet needs a mask")
    SO.check_sampler(kind, eta)
    first, ts = SO.img2img_start(strength, n_steps)
    z0 = SO.scaled_latent(encode_image(P, torch.from_numpy(IO.image_u8_to_float(image_u8))))
    cond = inpaint_cond(P, image_u8, mask_u8)
    if taps is not None:
        taps["z0"], taps["m_lat"], taps["z_m"] = z0, cond[:, 0], cond[:, 1:]
    a0 = float(P("alpha_cumulative_products").to(torch.float32)[ts[first]])
    start = SO.start_latent(a0, z0, np.asarray(noise, np.float32))
    cond_t = torch.from_numpy(cond).to(P.dtype)
    guide = lambda x, t: forward_diffuser(P, torch.cat([x, cond_t], 1), t, context, uncond, scale)
    return SO.guided_latent(P, n_steps, start, guide, kind, eta, noise_seed, first)


def zero_extension(conv_in4):
    """A [320,9,3,3] conv_in whose channels 0-3 are `conv_in4` and 4-8 zero: the 4-channel UNet bit for bit."""
    w = np.zeros((conv_in4.shape[0], 9, 3, 3), np.float32)
    w[:, :4] = conv_in4
    return w


# ------------------------------------------------------------------------------------------------ fixture
INPAINT = dict(n_steps=4, scale=5.0)
INPAINT_CASES = {"ddim_s1": dict(kind=SO.DDIM, strength=1.0), "dpmpp_s05": dict(kind=SO.DPMPP_2M, strength=0.5)}
