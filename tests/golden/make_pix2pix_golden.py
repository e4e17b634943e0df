"""Writes tests/golden/pix2pix_b2.npz (and no other fixture) from the InstructPix2Pix oracle (tests/pix2pix_oracle.py) on the
8-channel synthetic weights (seed 0): n = 2, 256x256 px (32x32 latent), the images of img2img_inputs(), L = 7, Lu = 2, text
scale 5.0, image scale 1.5, 4 steps; DDIM and DPM-Solver++(2M) from one seeded start latent. Stores the inputs, the unscaled
image latent c_I, each case's final latent and its u8 output at a stride of 2.
Run from the repo root:  python tests/golden/make_pix2pix_golden.py
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
import pix2pix_oracle as PO  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def main():
    torch.set_num_threads(os.cpu_count())
    P = O.Params(synth.make_params(0, pix2pix=True))
    image, _ = IO.img2img_inputs()
    ctx = synth.make_context(2, 7, seed=3)
    unc = synth.make_context(1, 2, seed=99)[0]
    latent0 = synth.make_latent(2, 32, 32, seed=43)
    out = dict(image=image, latent0=latent0)
    for name, case in PO.PIX2PIX_CASES.items():
        taps = {}
        t1 = time.time()
        with torch.no_grad():
            lat = PO.pix2pix_latent(P, ctx, unc, PO.PIX2PIX["text_scale"], PO.PIX2PIX["image_scale"], PO.PIX2PIX["n_steps"], image,
                                    latent0, kind=case["kind"], taps=taps)
            u8 = O.to_u8(O.latent_to_image_f32(P, lat))
        print(name, time.time() - t1, flush=True)
        out["c_I"] = taps["c_I"]
        out[f"latent_{name}"] = lat.numpy()
        out[f"u8_{name}"] = u8[:, ::2, ::2, :].copy()
    np.savez_compressed(os.path.join(OUT, "pix2pix_b2.npz"), **out)


if __name__ == "__main__":
    main()
