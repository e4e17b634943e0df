"""Sampler cost at 512x512, batch 1, cfg 7.5, L = 77: DDIM 20 steps, DDIM eta = 1 at 20, DPM-Solver++(2M) at 10, 15 and 20, on
the DDIM grid and on the Karras grid (DESIGN.md §7 f15), alternated, three CUDA-event timed runs each after warm-up, on sdb_sample_image_dev (sampling and decode); the cost of a step and
what the samplers add to it at 20 steps; and the card, power limit and SM clock read in the same process.
Usage: python tools/sampler_time.py"""
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from stable_diffusion_burn_b200 import _lib, synth

c = _lib.Context(0)
c.init_synthetic(0)
c.finalize_weights()
dev = torch.device("cuda:0")
n, H, L, SCALE = 1, 64, 77, 7.5
ctx = torch.from_numpy(synth.make_context(n, L)).to(dev)
unc = torch.from_numpy(synth.make_context(1, 2, seed=99)[0]).to(dev)
noise = torch.from_numpy(synth.make_latent(n, H, H)).to(dev)
rgb = torch.empty((n, 8 * H, 8 * H, 3), dtype=torch.uint8, device=dev)
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
p = lambda t: C.c_void_p(t.data_ptr())


def run(kind, eta, steps, schedule=0):
    c.set_sampler(kind, eta, 1)
    try:
        c.set_schedule(schedule)
        c.check(c.lib.sdb_sample_image_dev(c.h, p(ctx), n, L, p(unc), 2, SCALE, steps, p(noise), H, H, p(rgb), st))
    finally:
        c.set_sampler(0, 0.0, 0)
        c.set_schedule(0)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b)


configs = {}
for name, cfg in {"DDIM 20": (0, 0.0, 20), "DDIM eta=1 20": (0, 1.0, 20), "DPM++(2M) 10": (1, 0.0, 10),
                  "DPM++(2M) 15": (1, 0.0, 15), "DPM++(2M) 20": (1, 0.0, 20)}.items():
    configs[name] = cfg + (0,)
    configs["K " + name] = cfg + (1,)  # the same sampler on the Karras grid
for cfg in configs.values():
    run(*cfg), run(*cfg)
torch.cuda.synchronize()
ms = {k: [] for k in configs}
for _ in range(3):
    for k, cfg in configs.items():
        ms[k].append(timed(lambda: run(*cfg)))
base = sorted(ms["DDIM 20"])[1]
for k, v in ms.items():
    med = sorted(v)[1]
    print(f"{k:17s} ms {' '.join(f'{t:8.2f}' for t in v)}   images/s {' '.join(f'{1e3 * n / t:6.3f}' for t in v)}   "
          f"median speed-up vs DDIM 20 {base / med:5.2f}x")

med = {k: sorted(v)[1] for k, v in ms.items()}
per = (med["DPM++(2M) 20"] - med["DPM++(2M) 10"]) / 10
print(f"per step (DPM++ 20 - 10, median) {per:.2f} ms; at 20 steps DDIM eta=1 - DDIM {med['DDIM eta=1 20'] - base:+.2f} ms, "
      f"DPM++ - DDIM {med['DPM++(2M) 20'] - base:+.2f} ms")
print("Karras - DDIM grid, median: " + ", ".join(f"{k} {med['K ' + k] - med[k]:+.2f} ms" for k in configs if not k.startswith("K ")))

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True)
print("card:", q.stdout.strip() or q.stderr.strip())
c.close()
