"""Writes tests/golden/img2img_b2.npz (and no other fixture) from the img2img oracle (tests/sampler_oracle.py:
sampler_img2img_latent, DDIM) on the synthetic weights (seed 0): n = 2, 256x256 px (32x32 latent), L = 7, Lu = 2, cfg 5.0,
4 steps at strength 0.5 (k = 2: t = 499, 249).
Stores the inputs (images, masks, noise), z0, the latent mask w, the final latent and the u8 output at a stride of 2.
Run from the repo root:  python tests/golden/make_img2img_golden.py
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import sd_oracle as O  # noqa: E402
from stable_diffusion_burn_b200 import synth  # noqa: E402
import img2img_oracle as IO  # noqa: E402
import sampler_oracle as SO  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def main():
    torch.set_num_threads(os.cpu_count())
    P = O.Params(synth.make_params(0))
    image, mask = IO.img2img_inputs()
    ctx = torch.from_numpy(synth.make_context(2, 7, seed=3))
    unc = torch.from_numpy(synth.make_context(1, 2, seed=99))[0]
    noise = synth.make_latent(2, 32, 32, seed=41)
    cfg = IO.IMG2IMG
    taps = {}
    t1 = time.time()
    with torch.no_grad():
        lat = SO.sampler_img2img_latent(P, ctx, unc, cfg["scale"], cfg["n_steps"], image, cfg["strength"], noise, mask_u8=mask,
                                        taps=taps)
        u8 = O.to_u8(O.latent_to_image_f32(P, lat))
    print("img2img", time.time() - t1, flush=True)
    np.savez_compressed(os.path.join(OUT, "img2img_b2.npz"), image=image, mask=mask, noise=noise, z0=taps["z0"], w=taps["w"],
                        latent=lat.numpy(), u8=u8[:, ::2, ::2, :].copy())


if __name__ == "__main__":
    main()
