"""Cost of LoRA adapters (DESIGN.md §7 f8), timed on the device:
  apply     sdb_lora_apply of a seeded adapter (synth.make_lora) onto the base packing: an attention-only adapter (every
            SpatialTransformer Linear / 1x1 conv, 192 UNet modules, and every CLIP attention / MLP Linear, 72) at r = 16, 64, 128,
            and a LoCon adapter on every target (278 + 72 modules) at r = 32; host clock around the synchronous call
  finalize  a full sdb_finalize_weights with the same adapter active
  sampling  sdb_sample_image_dev images/s at 512x512, 20 DDIM steps, n = 1, without and with the r = 64 attention adapter
            (the kernels are the same, so these should match within noise), alternated, CUDA events
Three runs each, median reported; the card, power limit and SM clock are read in the same process.
Usage: python tools/lora_time.py"""
import ctypes as C
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from stable_diffusion_burn_b200 import _lib, lora, synth

c = _lib.Context(0)
c.init_synthetic(0)
c.finalize_weights()
ATTN = sorted(r for r in lora.UNET_MODULES.values() if "/transformer/" in r) + sorted(lora.CLIP_MODULES.values())
ALL = sorted(lora.UNET_MODULES.values()) + sorted(lora.CLIP_MODULES.values())
assert len(ATTN) == 192 + 72 and len(ALL) == 278 + 72


def host_ms(fn):
    t0 = time.perf_counter()
    fn()
    return 1e3 * (time.perf_counter() - t0)


def load(adapter, targets, rank):
    for reg, down, up, a in synth.make_lora(targets, rank, seed=rank):
        c.lora_add(adapter, reg, down, up, a)


for name, targets, rank in [("attention", ATTN, 16), ("attention", ATTN, 64), ("attention", ATTN, 128), ("locon", ALL, 32)]:
    load(0, targets, rank)
    apply_ms, fin_ms = [], []
    for _ in range(3):
        c.lora_scale(0, 1.0)
        apply_ms.append(host_ms(c.lora_apply))  # base packing -> base + adapter: every targeted unit re-packed
        fin_ms.append(host_ms(c.finalize_weights))
        c.lora_scale(0, 0.0)
        c.lora_apply()
    c.lora_remove(0)
    c.lora_apply()
    print(f"{name:9s} r={rank:3d} {len(targets)} modules: lora_apply ms {' '.join(f'{x:8.1f}' for x in apply_ms)} "
          f"(median {sorted(apply_ms)[1]:8.1f}); finalize_weights with the adapter ms {' '.join(f'{x:8.1f}' for x in fin_ms)} "
          f"(median {sorted(fin_ms)[1]:8.1f})")

dev = torch.device("cuda:0")
H, STEPS = 64, 20
d_ctx = torch.from_numpy(synth.make_context(1, 77)).to(dev)
d_unc = torch.from_numpy(synth.make_context(1, 2, seed=99)[0]).to(dev)
noise = torch.from_numpy(synth.make_latent(1, H, H)).to(dev)
rgb = torch.empty((1, 8 * H, 8 * H, 3), dtype=torch.uint8, device=dev)
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
p = lambda x: C.c_void_p(x.data_ptr())


def sample():
    c.check(c.lib.sdb_sample_image_dev(c.h, p(d_ctx), 1, 77, p(d_unc), 2, 7.5, STEPS, p(noise), H, H, p(rgb), st))


def timed(fn):
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); e.record(); torch.cuda.synchronize()
    return a.elapsed_time(e)


load(1, ATTN, 64)
c.lora_scale(1, 0.0)
c.lora_apply()
sample(), sample()
ms = {"base": [], "adapter r=64": []}
for _ in range(3):
    for k, m in (("base", 0.0), ("adapter r=64", 1.0)):
        c.lora_scale(1, m)
        c.lora_apply()
        sample()  # warm after the switch
        torch.cuda.synchronize()
        ms[k].append(timed(sample))
for k, v in ms.items():
    print(f"sample_image_dev 512x512 20 steps, {k:12s}: images/s {' '.join(f'{1e3 / x:6.3f}' for x in v)} "
          f"median {1e3 / sorted(v)[1]:6.3f}")
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True)
print("card:", q.stdout.strip() or q.stderr.strip())
c.close()
