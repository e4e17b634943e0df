"""CPU oracle of InstructPix2Pix image editing with an 8-channel UNet (DESIGN.md §7 f10) and the cases of its fixture — TEST
INFRASTRUCTURE ONLY.

InstructPix2Pix (Brooks et al. 2023) conditions an SD-1.x UNet on the input image: conv_in reads cat(x_t, c_I), c_I the VAE
posterior mode of the image, unscaled. Each step evaluates the UNet three times and combines the results with a text and an
image scale, as the original edit_cli.py and diffusers' StableDiffusionInstructPix2PixPipeline do. The reference has no such
model; the functions below follow the semantics the CUDA path implements, on top of tests/img2img_oracle.py (the image
conversion), tests/sampler_oracle.py (the step loop) and oracle/sd_oracle.py (encode_image and unet_forward, whose conv_in
takes whatever width P holds). The fixture tests/golden/pix2pix_b2.npz is written by tests/golden/make_pix2pix_golden.py from
PIX2PIX_CASES.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle.sd_oracle import encode_image, unet_forward

import img2img_oracle as IO
import sampler_oracle as SO


def image_latent(P, image_u8):
    """c_I [n,4,H,W] (torch, P's dtype): encode_image(x) with x = fl(fl(v / 127.5) - 1), UNSCALED (no 0.18215)."""
    return encode_image(P, torch.from_numpy(IO.image_u8_to_float(image_u8)).to(P.dtype))


def check_scales(text_scale, image_scale):
    """The argument rule of sdb_edit_image: both scales finite, named in the error."""
    for name, v in (("text_scale", text_scale), ("image_scale", image_scale)):
        if not math.isfinite(v):
            raise ValueError(f"{name} = {v} is not finite")


def three_way(e_u, e_i, e_t, text_scale, image_scale):
    """pred = e_U + s_T (e_T - e_I) + s_I (e_I - e_U), left to right, one rounding per operation in the tensors' dtype."""
    return (e_u + (e_t - e_i) * text_scale) + (e_i - e_u) * image_scale


def pix2pix_latent(P, ctx, unc, text_scale, image_scale, n_steps, image_u8, latent0, kind=SO.DDIM, eta=0.0, noise_seed=0,
                   taps=None):
    """InstructPix2Pix editing -> the final latent [n,4,H,W] (torch). P holds a [320,8,3,3] conv_in; ctx [n,L,768] the
    instructions, unc [Lu,768] the negative broadcast over the batch; latent0 [n,4,H,W] the start latent at t = 999. Each step:
    e_T = UNet(cat(x, c_I), ctx), e_I = UNet(cat(x, c_I), unc), e_U = UNet(cat(x, 0), unc), combined by three_way, then the
    sampler's update. taps receives "c_I" (float32 numpy)."""
    check_scales(text_scale, image_scale)
    c_i = image_latent(P, image_u8)
    if taps is not None:
        taps["c_I"] = c_i.to(torch.float32).numpy()
    ctx = torch.as_tensor(ctx).to(P.dtype)
    u_ctx = torch.as_tensor(unc).to(P.dtype).unsqueeze(0).repeat(c_i.shape[0], 1, 1)
    zero = torch.zeros_like(c_i)

    def guide(x, t):
        xi = torch.cat([x, c_i], 1)
        e_t = unet_forward(P, xi, t, ctx)
        e_i = unet_forward(P, xi, t, u_ctx)
        e_u = unet_forward(P, torch.cat([x, zero], 1), t, u_ctx)
        return three_way(e_u, e_i, e_t, text_scale, image_scale)

    return SO.guided_latent(P, n_steps, latent0, guide, kind, eta, noise_seed)


def zero_extension(conv_in4):
    """A [320,8,3,3] conv_in whose channels 0-3 are `conv_in4` and 4-7 zero: the image latent has no effect."""
    w = np.zeros((conv_in4.shape[0], 8, 3, 3), np.float32)
    w[:, :4] = conv_in4
    return w


# ------------------------------------------------------------------------------------------------ fixture
PIX2PIX = dict(n_steps=4, text_scale=5.0, image_scale=1.5)
PIX2PIX_CASES = {"ddim": dict(kind=SO.DDIM), "dpmpp": dict(kind=SO.DPMPP_2M)}
