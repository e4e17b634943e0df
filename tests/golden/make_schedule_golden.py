"""Writes tests/golden/schedule_b2.npz (and no other fixture) from the Karras-schedule oracle (tests/schedule_oracle.py) on the
synthetic weights (seed 0), the sampler_b2 inputs on the Karras grid (DESIGN.md §7 f15): n = 2, 32x32 latents (256x256 px), L = 7,
Lu = 2, cfg 5.0, 4 steps (t = 999, 687.1533, 145.9392, 0):
  ddim    DDIM eta = 0 (k-diffusion's Euler) txt2img
  eta     DDIM eta = 0.7, noise_seed 11 (Euler ancestral), txt2img
  dpmpp   DPM-Solver++(2M) txt2img
  inpaint DPM-Solver++(2M) masked inpainting of the img2img_inputs() images at strength 0.75 (the last 3 steps)
from the start latent / noise synth.make_latent(2, 32, 32, seed=41). Stores each final latent and its u8 image at a stride of 2.
Run from the repo root:  python tests/golden/make_schedule_golden.py
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
import schedule_oracle as KO  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def compute(P):
    cfg = SO.SAMPLER_CASES
    ctx = torch.from_numpy(synth.make_context(2, 7, seed=3))
    unc = torch.from_numpy(synth.make_context(1, 2, seed=99))[0]
    noise = synth.make_latent(2, 32, 32, seed=41)
    image, mask = IO.img2img_inputs()
    out = dict(noise=noise)
    lat0 = lambda: torch.from_numpy(noise)
    with torch.no_grad():
        runs = {
            "ddim": lambda: KO.karras_latent(P, ctx, unc, cfg["scale"], cfg["n_steps"], lat0()),
            "eta": lambda: KO.karras_latent(P, ctx, unc, cfg["scale"], cfg["n_steps"], lat0(), SO.DDIM, cfg["eta"],
                                            cfg["noise_seed"]),
            "dpmpp": lambda: KO.karras_latent(P, ctx, unc, cfg["scale"], cfg["n_steps"], lat0(), SO.DPMPP_2M),
            "inpaint": lambda: KO.karras_img2img_latent(P, ctx, unc, cfg["scale"], cfg["n_steps"], image, cfg["strength"], noise,
                                                        mask_u8=mask, kind=SO.DPMPP_2M),
        }
        for name, fn in runs.items():
            t1 = time.time()
            lat = torch.as_tensor(fn())
            u8 = O.to_u8(O.latent_to_image_f32(P, lat))
            print(name, f"{time.time() - t1:.1f} s", flush=True)
            out[f"{name}_latent"] = lat.numpy()
            out[f"{name}_u8"] = u8[:, ::2, ::2, :].copy()
    return out


def main():
    torch.set_num_threads(os.cpu_count())
    out = compute(O.Params(synth.make_params(0)))
    np.savez_compressed(os.path.join(OUT, "schedule_b2.npz"), **out)


if __name__ == "__main__":
    main()
