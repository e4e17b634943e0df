"""Throughput of a batch of different requests at 512x512, 20 DDIM steps, sampling and decode: 8 requests with prompt lengths 5 to
77, mixed negatives (the empty prompt's 2 tokens, 6 and 11 tokens) and scales 3 to 9, timed with CUDA events
  batch       as one sdb_sample_batch_dev call
  sequential  as 8 sdb_sample_image_dev calls at n = 1, each with its own length, negative and scale
  homogeneous as one sdb_sample_image_dev call at n = 8 (L = 77, the 2-token negative, one scale): the same step and step graph
alternated, three timed runs each after warm-up; images/s, and the card, power limit and SM clock read in the same process.
Usage: python tools/batch_time.py"""
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
n, H, STEPS = 8, 64, 20
LENS = [5, 9, 14, 22, 31, 46, 60, 77]
ULENS = [2, 6, 2, 11, 2, 2, 6, 2]
SCALES = [7.5, 5.0, 3.0, 9.0, 7.5, 6.0, 4.0, 8.0]
ctxs = [synth.make_context(1, L, seed=500 + i)[0] for i, L in enumerate(LENS)]
uncs = [synth.make_context(1, Lu, seed=600 + i)[0] for i, Lu in enumerate(ULENS)]
b = _lib.pack_batch(ctxs, uncs, SCALES, seeds=list(range(1, n + 1)))
t = lambda a: torch.from_numpy(a).to(dev)
d_ctx, d_unc = t(b["context"]), t(b["uncond"])
bs = _lib.batch_struct(b, d_ctx.data_ptr(), d_unc.data_ptr())
d_ctx1 = [t(a) for a in ctxs]
d_unc1 = [t(a) for a in uncs]
d_homo, d_hunc = t(synth.make_context(n, 77)), t(synth.make_context(1, 2, seed=99)[0])
noise = t(synth.make_latent(n, H, H))
rgb = torch.empty((n, 8 * H, 8 * H, 3), dtype=torch.uint8, device=dev)
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
p = lambda x: C.c_void_p(x.data_ptr())


def batch():
    c.check(c.lib.sdb_sample_batch_dev(c.h, C.byref(bs), STEPS, p(noise), H, H, None, p(rgb), st))


def sequential():
    for i in range(n):
        c.check(c.lib.sdb_sample_image_dev(c.h, p(d_ctx1[i]), 1, LENS[i], p(d_unc1[i]), ULENS[i], SCALES[i], STEPS, p(noise[i]),
                                           H, H, p(rgb[i]), st))


def homogeneous():
    c.check(c.lib.sdb_sample_image_dev(c.h, p(d_homo), n, 77, p(d_hunc), 2, 7.5, STEPS, p(noise), H, H, p(rgb), st))


def timed(fn):
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); e.record(); torch.cuda.synchronize()
    return a.elapsed_time(e)


runs = {"batch": batch, "sequential": sequential, "homogeneous": homogeneous}
for fn in runs.values():
    fn(), fn()
torch.cuda.synchronize()
ms = {k: [] for k in runs}
for _ in range(3):
    for k, fn in runs.items():
        ms[k].append(timed(fn))
for k, v in ms.items():
    med = sorted(v)[1]
    print(f"{k:12s} ms {' '.join(f'{x:9.1f}' for x in v)}   images/s {' '.join(f'{1e3 * n / x:6.3f}' for x in v)}   "
          f"median {1e3 * n / med:6.3f}")
med = {k: sorted(v)[1] for k, v in ms.items()}
print(f"batch vs sequential {med['sequential'] / med['batch']:.2f}x images/s; batch vs homogeneous "
      f"{med['homogeneous'] / med['batch']:.3f}x")
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True)
print("card:", q.stdout.strip() or q.stderr.strip())
c.close()
