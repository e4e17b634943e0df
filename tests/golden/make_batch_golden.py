"""Writes tests/golden/batch_hetero.npz (and no other fixture): three different requests of one batch call (DESIGN.md §7 f7), each
run through the sampler oracle (tests/sampler_oracle.py) on its own at n = 1, on the synthetic weights (seed 0), 32x32 latents
(256x256 px), 4 steps (t = 999, 749, 499, 249):
  request 0  L = 5,  the shared 2-token negative, scale 7.5
  request 1  L = 13, its own 9-token negative,     scale 1.0
  request 2  L = 77, the shared 2-token negative, scale 3.0
each with its own seed (its start latent / noise, synth.seeded_latents) and noise seed. Runs:
  ddim     DDIM (eta = 0) txt2img
  dpmpp    DPM-Solver++(2M) txt2img
  eta      DDIM eta = 0.7 txt2img, the step noise keyed per request by its noise seed
  inpaint  DPM-Solver++(2M) masked inpainting at strength 0.75 of the img2img_inputs() images 0, 1, 0 under masks 0, 1, 1
Stores the start latents, each final latent and its u8 image at a stride of 2.
Run from the repo root:  python tests/golden/make_batch_golden.py
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
BATCH_CASES = dict(n_steps=4, H=32, W=32, lens=(5, 13, 77), ulens=(2, 9, 2), scales=(7.5, 1.0, 3.0), seeds=(101, 102, 2 ** 33 + 103),
                   noise_seeds=(201, 202, 203), eta=0.7, strength=0.75, images=(0, 1, 0), masks=(0, 1, 1))


def requests():
    """-> (contexts [L_i, 768], negatives [Lu_i, 768], start latents [3, 4, 32, 32]) of BATCH_CASES."""
    cfg = BATCH_CASES
    shared = synth.make_context(1, 2, seed=99)[0]
    ctxs = [synth.make_context(1, L, seed=300 + i)[0] for i, L in enumerate(cfg["lens"])]
    uncs = [shared if Lu == 2 else synth.make_context(1, Lu, seed=400 + i)[0] for i, Lu in enumerate(cfg["ulens"])]
    return ctxs, uncs, synth.seeded_latents(cfg["seeds"], cfg["H"], cfg["W"])


def compute(P):
    cfg = BATCH_CASES
    ctxs, uncs, noise = requests()
    image, mask = IO.img2img_inputs()
    out = dict(noise=noise)
    steps = cfg["n_steps"]
    with torch.no_grad():
        def txt(i, kind, eta=0.0):
            return SO.sampler_latent(P, torch.from_numpy(ctxs[i][None]), torch.from_numpy(uncs[i]), cfg["scales"][i], steps,
                                     torch.from_numpy(noise[i:i + 1]), kind, eta, cfg["noise_seeds"][i])

        def inpaint(i):
            return SO.sampler_img2img_latent(P, torch.from_numpy(ctxs[i][None]), torch.from_numpy(uncs[i]), cfg["scales"][i], steps,
                                             image[cfg["images"][i]][None], cfg["strength"], noise[i:i + 1],
                                             mask_u8=mask[cfg["masks"][i]][None], kind=SO.DPMPP_2M)

        runs = {"ddim": lambda i: txt(i, SO.DDIM), "dpmpp": lambda i: txt(i, SO.DPMPP_2M),
                "eta": lambda i: txt(i, SO.DDIM, cfg["eta"]), "inpaint": inpaint}
        for name, fn in runs.items():
            t1 = time.time()
            lat = torch.cat([fn(i) for i in range(3)])
            u8 = O.to_u8(O.latent_to_image_f32(P, lat))
            print(name, f"{time.time() - t1:.1f} s", flush=True)
            out[f"{name}_latent"] = lat.numpy()
            out[f"{name}_u8"] = u8[:, ::2, ::2, :].copy()
    return out


def main():
    torch.set_num_threads(os.cpu_count())
    out = compute(O.Params(synth.make_params(0)))
    np.savez_compressed(os.path.join(OUT, "batch_hetero.npz"), **out)


if __name__ == "__main__":
    main()
