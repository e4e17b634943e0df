"""Generates tests/golden/*.npz from the CPU oracle (oracle/sd_oracle.py) on the synthetic weights (seed 0).

The oracle itself is pinned against the reference's own Python model (tests/test_ref_pin_cpu.py, tests/ref_shim/); these
fixtures are what the GPU suite holds the CUDA path to (erf GELU, like the Rust model), and the CPU suite re-derives a subset. Run from the repo root:  python tests/golden/make_golden.py
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import sd_oracle as O  # noqa: E402
from stable_diffusion_burn_b200 import synth  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
ONLY = set(sys.argv[1:])  # e.g. `make_golden.py batch2_32` regenerates only that UNet case (+ the 2-step sample)


CLIP_PROMPT = [49406, 550, 5810, 617, 8661, 2441, 13, 27, 347, 40786, 4160, 91, 285, 49407]  # arbitrary in-vocab ids, sot..eot


def clip_tokens():
    """Token batches of the CLIP fixture: a README-length prompt, the empty prompt, a full 77-id window, a ragged pair."""
    g = np.random.Generator(np.random.Philox(4242))
    full = np.concatenate([[49406], g.integers(0, 49406, 75), [49407]]).astype(np.int32)
    pair = np.stack([np.concatenate([[49406], g.integers(0, 49406, 9), [49407]]),
                     np.concatenate([[49406], g.integers(0, 49406, 4), [49407] * 6])]).astype(np.int32)
    return {"prompt": np.asarray(CLIP_PROMPT, np.int32)[None], "empty": np.asarray([[49406, 49407]], np.int32),
            "full77": full[None], "pair11": pair}


def clip_golden():
    from stable_diffusion_burn_b200 import topology
    P = O.Params(synth.make_params(0, which=topology.clip_params()))
    keep = {}
    with torch.no_grad():
        for name, tok in clip_tokens().items():
            y = O.clip_forward(P, torch.from_numpy(tok).long())
            keep["tok:" + name] = tok
            keep["out:" + name] = y.numpy()
            print("clip", name, tuple(y.shape), "rms", float(y.pow(2).mean().sqrt()), flush=True)
    np.savez_compressed(os.path.join(OUT, "clip.npz"), **keep)


def enc_images():
    """Inputs of the VAE-encoder fixture: the RNG-free ramp at 64x64 and a seeded batch of two 128x96 images."""
    g = np.random.Generator(np.random.Philox(777))
    return {"ramp64": synth.sin_ramp((1, 3, 64, 64)), "randn128x96": g.standard_normal((2, 3, 128, 96), dtype=np.float32)}


def enc_golden():
    from stable_diffusion_burn_b200 import topology
    P = O.Params(synth.make_params(0, which=topology.vae_encoder_params()))
    keep = {}
    with torch.no_grad():
        for name, img in enc_images().items():
            y = O.encode_image(P, torch.from_numpy(img))
            keep["img:" + name] = img
            keep["lat:" + name] = y.numpy()
            print("vae_enc", name, tuple(y.shape), "rms", float(y.pow(2).mean().sqrt()), flush=True)
    np.savez_compressed(os.path.join(OUT, "vae_enc.npz"), **keep)


def round2_cases(P):
    """Fixtures for the configurations bench.py actually times (VERDICT r1 item 1b): the CFG batch at L = 77 / Lu = 2, 20 DDIM
    steps, batch 8 at 64x64 (C3/C5), the 96x96 -> 768x768 decode (C4). Select with `make_golden.py r2` (or one of the names)."""
    sel = lambda name: (not ONLY) or ("r2" in ONLY) or (name in ONLY)
    unc = torch.from_numpy(synth.make_context(1, 2, seed=99))[0]
    with torch.no_grad():
        if sel("cfg_L77"):
            # forward_diffuser on the bench's exact shape: n = 1, 64x64, L = 77, Lu = 2, t = 999 and a mid-schedule t
            keep = {}
            x = torch.from_numpy(synth.make_latent(1, 64, 64))
            ctx = torch.from_numpy(synth.make_context(1, 77))
            for t in (999, 449):
                taps = {}
                t1 = time.time()
                pred = O.forward_diffuser(P, x, t, ctx, unc, 7.5, taps=taps)
                keep[f"t{t}:uncond"], keep[f"t{t}:cond"], keep[f"t{t}:pred"] = taps["uncond"].numpy(), taps["cond"].numpy(), pred.numpy()
                print("cfg_L77", t, time.time() - t1, flush=True)
            np.savez_compressed(os.path.join(OUT, "cfg_L77.npz"), **keep)
        if sel("unet_b8_64"):
            x = torch.from_numpy(synth.make_latent(8, 64, 64, seed=808))
            ctx = torch.from_numpy(synth.make_context(8, 77, seed=88))
            t1 = time.time()
            y = torch.cat([O.unet_forward(P, x[i:i + 1], 599, ctx[i:i + 1]) for i in range(8)])
            print("unet_b8_64", time.time() - t1, flush=True)
            np.savez_compressed(os.path.join(OUT, "unet_b8_64.npz"), out=y.numpy())
        if sel("vae_96"):
            lat = torch.from_numpy(synth.make_latent(1, 96, 96, seed=96))
            t1 = time.time()
            img = O.decode_latent(P, lat)
            print("vae_96", time.time() - t1, tuple(img.shape), flush=True)
            np.savez_compressed(os.path.join(OUT, "vae_96.npz"), img_sub=img[:, :, ::8, ::8].numpy().copy(),
                                img_rows=img[:, :, 380:384, :].numpy().copy(), mean=float(img.mean()), std=float(img.std()))
        if sel("sample_20step"):
            # C2 exactly: n = 1, 64x64, 20 steps, cfg 7.5, L = 77, Lu = 2. Taps at steps 0 / 9 / 19: the latent that entered the
            # step and the two UNet outputs on it (per-step parity is judged on the ORACLE's latent), plus the free-running result.
            ctx = torch.from_numpy(synth.make_context(1, 77))
            init = torch.from_numpy(synth.make_latent(1, 64, 64))
            taps = {}
            t1 = time.time()
            lat = O.sample_latent(P, ctx, unc, 7.5, 20, init, taps=taps)
            print("sample_20step latent", time.time() - t1, flush=True)
            imgf = O.latent_to_image_f32(P, lat)
            keep = {"latent": lat.numpy(), "u8_sub": O.to_u8(imgf)[:, ::2, ::2, :].copy()}
            ts, _ = O.ddim_timesteps(20)
            for i in (0, 9, 19):
                keep[f"step{i}:t"] = np.int32(ts[i])
                for k in ("latent_in", "uncond", "cond"):
                    keep[f"step{i}:{k}"] = taps[f"step{i}/{k}"].numpy()
            np.savez_compressed(os.path.join(OUT, "sample_20step.npz"), **keep)


R2_NAMES = {"r2", "cfg_L77", "unet_b8_64", "vae_96", "sample_20step"}


def main():
    torch.set_num_threads(os.cpu_count())
    t0 = time.time()
    if ONLY and ONLY <= R2_NAMES:
        P = O.Params(synth.make_params(0))
        print("params", time.time() - t0, flush=True)
        round2_cases(P)
        print("done", time.time() - t0)
        return
    if not ONLY or "enc" in ONLY:
        enc_golden()
        if ONLY == {"enc"}:
            return
    if not ONLY or "clip" in ONLY:
        clip_golden()
        if ONLY == {"clip"}:
            return
    P = O.Params(synth.make_params(0))
    print("params", time.time() - t0, flush=True)
    with torch.no_grad():
        # --- UNet known-answer inputs
        cases = {}
        # (i) the reference author's eyeball probe: zeros latent, repeat([0.5,1.3],384) context, t=1 (python/dump.py:624-633)
        x = torch.zeros(1, 4, 64, 64)
        cases["kat_zeros"] = (x, 1, torch.from_numpy(synth.kat_context()))
        # (ii) sin ramp latent (python/test_tiny.py:25), L = 13 context, t = 500
        cases["sin_ramp"] = (torch.from_numpy(synth.sin_ramp((1, 4, 64, 64))), 500, torch.from_numpy(synth.make_context(1, 13)))
        # (iii) seeded N(0,1) latent, t = 999 (first DDIM step), README-like L = 13
        cases["randn_t999"] = (torch.from_numpy(synth.make_latent(1, 64, 64)), 999, torch.from_numpy(synth.make_context(1, 13)))
        # (iv) batch 2, small latent (32x32 is the smallest size whose deepest level keeps 16-byte aligned tiles), L = 5
        cases["batch2_32"] = (torch.from_numpy(synth.make_latent(2, 32, 32, seed=7)), 321, torch.from_numpy(synth.make_context(2, 5, seed=5)))
        for name, (x, t, ctx) in cases.items():
            if ONLY and name not in ONLY:
                continue
            t1 = time.time()
            y = O.unet_forward(P, x, t, ctx)
            keep = {"out": y.numpy()}
            np.savez_compressed(os.path.join(OUT, f"unet_{name}.npz"), **keep)
            print(name, time.time() - t1, "rms", float(y.pow(2).mean().sqrt()), flush=True)
        if ONLY and "vae" not in ONLY:
            return finish(P, t0)
        # --- VAE decode
        lat = torch.from_numpy(synth.make_latent(1, 16, 16, seed=21))
        img = O.decode_latent(P, lat)
        np.savez_compressed(os.path.join(OUT, "vae_16.npz"), img=img.numpy())
        lat = torch.from_numpy(synth.make_latent(1, 64, 64, seed=22))
        t1 = time.time()
        img = O.decode_latent(P, lat)
        print("vae64", time.time() - t1, flush=True)
        np.savez_compressed(os.path.join(OUT, "vae_64.npz"), img_sub=img[:, :, ::8, ::8].numpy().copy(),
                            img_rows=img[:, :, 250:254, :].numpy().copy(), mean=float(img.mean()), std=float(img.std()))
        # --- one-step end-to-end (C1 plumbing config): n=1, 64x64, 1 step, cfg 7.5, L = 13, Lu = 2
        ctx = torch.from_numpy(synth.make_context(1, 13))
        unc = torch.from_numpy(synth.make_context(1, 2, seed=99))[0]
        init = torch.from_numpy(synth.make_latent(1, 64, 64))
        t1 = time.time()
        lat1 = O.sample_latent(P, ctx, unc, 7.5, 1, init)
        imgf = O.latent_to_image_f32(P, lat1)
        u8 = O.to_u8(imgf)
        print("e2e 1 step", time.time() - t1, flush=True)
        np.savez_compressed(os.path.join(OUT, "sample_1step.npz"), latent=lat1.numpy(), img_f32_sub=imgf[:, ::4, ::4, :].numpy().copy(),
                            u8=u8)
    round2_cases(P)
    finish(P, t0)


def finish(P, t0):
    with torch.no_grad():
        # --- two DDIM steps on a small latent, batch 2 (exercises alpha_prev lookup and the CFG batch layout)
        unc = torch.from_numpy(synth.make_context(1, 2, seed=99))[0]
        ctx = torch.from_numpy(synth.make_context(2, 7, seed=3))
        init = torch.from_numpy(synth.make_latent(2, 32, 32, seed=31))
        lat2 = O.sample_latent(P, ctx, unc, 5.0, 2, init)
        u8 = O.to_u8(O.latent_to_image_f32(P, lat2))
        np.savez_compressed(os.path.join(OUT, "sample_2step_b2.npz"), latent=lat2.numpy(), u8=u8[:, ::2, ::2, :].copy())
    print("done", time.time() - t0)


if __name__ == "__main__" and ONLY != {"realstats"}:
    main()


def realstats_golden():
    """UNet outputs on the REALISTIC-STATISTICS weights (synth.realistic_stats: log-normal channel gains, wide norm affine,
    sharper attention logits): `python tests/golden/make_golden.py realstats`."""
    from stable_diffusion_burn_b200 import topology
    P = O.Params(synth.realistic_stats(synth.make_params(0, topology.unet_params())))
    keep = {}
    with torch.no_grad():
        y = O.unet_forward(P, torch.from_numpy(synth.make_latent(2, 32, 32, seed=7)), 321, torch.from_numpy(synth.make_context(2, 13, seed=5)))
        keep["b2_32"] = y.numpy()
        y = O.unet_forward(P, torch.from_numpy(synth.make_latent(1, 64, 64)), 999, torch.from_numpy(synth.make_context(1, 77)))
        keep["n1_64_L77"] = y.numpy()
    np.savez_compressed(os.path.join(OUT, "unet_realstats.npz"), **keep)
    print("realstats", {k: float(np.sqrt((v ** 2).mean())) for k, v in keep.items()})


if __name__ == "__main__" and ONLY == {"realstats"}:
    torch.set_num_threads(os.cpu_count())
    realstats_golden()
