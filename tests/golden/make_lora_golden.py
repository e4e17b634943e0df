"""Writes tests/golden/lora_b1.npz (and no other fixture): the synthetic weights (seed 0) with a seeded synthetic LoRA adapter
(synth.make_lora, rank 8, seed 8, alpha = r) on one module of every target kind (DESIGN.md §7 f8), merged in fp64 and rounded to
fp32, run through the oracle: prompt tokens -> CLIP (prompt and the empty negative) -> 4 DDIM steps at 32x32 latents (256x256 px),
scale 5.0 -> the u8 image. Stores the tokens, the start latent, both CLIP outputs, the final latent and the u8 image at a stride
of 2. The GPU test regenerates the adapter from (LORA_TARGETS, RANK, SEED).
Run from the repo root:  python tests/golden/make_lora_golden.py
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import sd_oracle as O  # noqa: E402
from stable_diffusion_burn_b200 import lora, synth  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
RANK, SEED, STEPS, SCALE = 8, 8, 4, 5.0
ST = "unet/input_blocks/rt1/transformer"
LORA_TARGETS = [
    f"{ST}/transformer/attn1/query/weight", f"{ST}/transformer/attn1/key/weight", f"{ST}/transformer/attn1/value/weight",
    f"{ST}/transformer/attn1/out/weight", f"{ST}/transformer/attn2/query/weight", f"{ST}/transformer/attn2/key/weight",
    f"{ST}/transformer/attn2/value/weight", f"{ST}/transformer/attn2/out/weight", f"{ST}/transformer/mlp/geglu/proj/weight",
    f"{ST}/transformer/mlp/lin/weight", f"{ST}/proj_in/weight", f"{ST}/proj_out/weight",
    "unet/input_blocks/rt1/res/conv_in/weight", "unet/input_blocks/rt1/res/conv_out/weight",
    "unet/input_blocks/rt3/res/skip_connection/weight", "unet/input_blocks/rt1/res/lin_embed/weight",
    "unet/input_blocks/d1/weight", "unet/output_blocks/rtu2/upsample/conv/weight",
    "clip/blocks/0/attn/query/weight", "clip/blocks/0/attn/key/weight", "clip/blocks/0/attn/value/weight",
    "clip/blocks/0/attn/out/weight", "clip/blocks/0/mlp/fc1/weight", "clip/blocks/0/mlp/fc2/weight",
]
TOKENS = np.array([[49406, 320, 1125, 539, 320, 2368, 49407]], np.int64)
UTOKENS = np.array([[49406, 49407]], np.int64)


def merged_params():
    params = synth.make_params(0)
    for reg, down, up, alpha in synth.make_lora(LORA_TARGETS, RANK, seed=SEED):
        w = params[reg]
        params[reg] = (w.astype(np.float64) + lora.delta(down, up, alpha, shape=w.shape)).astype(np.float32)
    return params


def compute():
    P = O.Params(merged_params())
    init = synth.make_latent(1, 32, 32, seed=31)
    with torch.no_grad():
        ctx = O.clip_forward(P, torch.from_numpy(TOKENS))
        unc = O.clip_forward(P, torch.from_numpy(UTOKENS))
        lat = O.sample_latent(P, ctx, unc[0], SCALE, STEPS, torch.from_numpy(init))
        u8 = O.to_u8(O.latent_to_image_f32(P, lat))
    return dict(tokens=TOKENS.astype(np.int32), utokens=UTOKENS.astype(np.int32), init=init, context=ctx.numpy(),
                uncond=unc.numpy(), latent=lat.numpy(), u8=u8[:, ::2, ::2, :].copy())


def main():
    torch.set_num_threads(os.cpu_count())
    t0 = time.time()
    out = compute()
    print(f"oracle {time.time() - t0:.1f} s")
    np.savez_compressed(os.path.join(OUT, "lora_b1.npz"), **out)


if __name__ == "__main__":
    main()
