"""Writes tests/golden/inpaint_b2.npz (and no other fixture) from the inpainting oracle (tests/inpaint_oracle.py) on the 9-channel
synthetic weights (seed 0): n = 2, 256x256 px (32x32 latent), the images and soft masks of img2img_inputs(), L = 7, Lu = 2, cfg
5.0, 4 steps; DDIM at strength 1.0 and DPM-Solver++(2M) at 0.5. Stores the inputs, the latent mask, z_m, each case's final latent
and its u8 output at a stride of 2.
Run from the repo root:  python tests/golden/make_inpaint_golden.py
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
import inpaint_oracle as NO  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def main():
    torch.set_num_threads(os.cpu_count())
    P = O.Params(synth.make_params(0, inpaint=True))
    image, mask = IO.img2img_inputs()
    ctx = torch.from_numpy(synth.make_context(2, 7, seed=3))
    unc = torch.from_numpy(synth.make_context(1, 2, seed=99))[0]
    noise = synth.make_latent(2, 32, 32, seed=41)
    out = dict(image=image, mask=mask, noise=noise)
    for name, case in NO.INPAINT_CASES.items():
        taps = {}
        t1 = time.time()
        with torch.no_grad():
            lat = NO.inpaint_latent(P, ctx, unc, NO.INPAINT["scale"], NO.INPAINT["n_steps"], image, case["strength"], noise, mask,
                                    kind=case["kind"], taps=taps)
            u8 = O.to_u8(O.latent_to_image_f32(P, lat))
        print(name, time.time() - t1, flush=True)
        out["m_lat"], out["z_m"] = taps["m_lat"], taps["z_m"]
        out[f"latent_{name}"] = lat.numpy()
        out[f"u8_{name}"] = u8[:, ::2, ::2, :].copy()
    np.savez_compressed(os.path.join(OUT, "inpaint_b2.npz"), **out)


if __name__ == "__main__":
    main()
