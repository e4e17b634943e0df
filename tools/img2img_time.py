"""img2img cost at 512x512, batch 1, 20 DDIM steps, cfg 7.5, L = 77: sample_image, img2img at strength 1.0 and at 0.75,
alternated, three CUDA-event timed runs each after warm-up, on the library's device entry points; then the per-class profile of
one call of each and of the encoder alone, and the card, power limit and SM clock read in the same process.
Usage: python tools/img2img_time.py"""
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from stable_diffusion_burn_b200 import _lib, synth

c = _lib.Context(0)
c.init_synthetic(0)
c.finalize_weights()
dev = torch.device("cuda:0")
n, H, L, STEPS, SCALE = 1, 64, 77, 20, 7.5
ctx = torch.from_numpy(synth.make_context(n, L)).to(dev)
unc = torch.from_numpy(synth.make_context(1, 2, seed=99)[0]).to(dev)
noise = torch.from_numpy(synth.make_latent(n, H, H)).to(dev)
y, x = np.mgrid[0:8 * H, 0:8 * H]
image = torch.from_numpy(np.stack([x / 2, y / 2, 255 - (x + y) / 4], -1).clip(0, 255).astype(np.uint8)[None]).to(dev)
img_f = torch.empty((n, 3, 8 * H, 8 * H), dtype=torch.float32, device=dev)
lat = torch.empty((n, 4, H, H), dtype=torch.float32, device=dev)
rgb = torch.empty((n, 8 * H, 8 * H, 3), dtype=torch.uint8, device=dev)
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
p = lambda t: C.c_void_p(t.data_ptr())


def sample():
    c.check(c.lib.sdb_sample_image_dev(c.h, p(ctx), n, L, p(unc), 2, SCALE, STEPS, p(noise), H, H, p(rgb), st))


def img2img(strength):
    c.check(c.lib.sdb_img2img_dev(c.h, p(image), None, strength, p(ctx), n, L, p(unc), 2, SCALE, STEPS, p(noise), H, H, None,
                                  p(rgb), st))


def encode():
    c.check(c.lib.sdb_encode_image_dev(c.h, p(img_f), n, 8 * H, 8 * H, p(lat), st))


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b)


runs = {"sample_image": sample, "img2img s=1.0": lambda: img2img(1.0), "img2img s=0.75": lambda: img2img(0.75)}
for fn in runs.values():
    fn(), fn()
torch.cuda.synchronize()
ms = {k: [] for k in runs}
for _ in range(3):
    for k, fn in runs.items():
        ms[k].append(timed(fn))
for k, v in ms.items():
    print(f"{k:16s} ms {' '.join(f'{t:8.2f}' for t in v)}   images/s {' '.join(f'{1e3 * n / t:6.3f}' for t in v)}")
for _ in range(2):
    encode()
enc = sorted(timed(encode) for _ in range(5))
print(f"encode_image 512x512: min {enc[0]:.2f} ms, median {enc[2]:.2f} ms")

runs["encode_image"] = encode
for k, fn in runs.items():
    c.profile(True); c.profile_reset()
    fn()
    torch.cuda.synchronize()
    tab = c.profile_table()
    c.profile(False)
    cls = {name: r for name, r in tab.items() if r["launches"]}
    print(f"profile {k}: total {sum(r['ms'] for r in cls.values()):.2f} ms  " +
          "  ".join(f"{name} {r['ms']:.2f} ms/{r['launches']}" for name, r in cls.items()))

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True)
print("card:", q.stdout.strip() or q.stderr.strip())
c.close()
