"""InstructPix2Pix cost (DESIGN.md §7 f10) at 512x512, 20 DDIM steps, L = 77, with decode, n = 1 and n = 4: text-to-image
(sdb_sample_image_dev, cfg 7.5) on a 4-channel context against an edit (sdb_edit_image_dev, text 7.5 / image 1.5) on an
8-channel one, one context per process, three alternated CUDA-event timed runs of each after warm-up. Then, in processes of
their own, per-launch device times from torch.profiler: the UNet's conv_in with 4 and 8 input channels at a 64x64 latent (nb = 3
and 12, sdb_unet_forward_dev), and the fused guidance + update step of each call (cfg_step_kernel, two-way <0, false, false, 2>,
three-way <0, false, false, 3>) at n = 1 and 4, graphs off so every launch is traced. The card, power limit and SM clock are read
in the same call.
Usage: python tools/pix2pix_time.py            (the driver; each measurement runs as  python tools/pix2pix_time.py <mode> <cin> <n>)"""
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from stable_diffusion_burn_b200 import _lib, synth

H, L, STEPS, TS, IS = 64, 77, 20, 7.5, 1.5


def context(cin):
    c = _lib.Context(0, pix2pix=cin == 8)
    c.init_synthetic(0)
    c.finalize_weights()
    return c


def setup(cin, n):
    """-> (context, run): one sampling call on the device entry, text-to-image (cin 4) or an edit (cin 8), decoded to u8."""
    c, dev = context(cin), torch.device("cuda:0")
    ctx = torch.from_numpy(synth.make_context(n, L)).to(dev)
    unc = torch.from_numpy(synth.make_context(1, 2, seed=99)[0]).to(dev)
    lat0 = torch.from_numpy(synth.make_latent(n, H, H)).to(dev)
    y, x = np.mgrid[0:8 * H, 0:8 * H]
    img = np.stack([x / 2, y / 2, 255 - (x + y) / 4], -1).clip(0, 255).astype(np.uint8)
    image = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(img, (n, 8 * H, 8 * H, 3)))).to(dev)
    rgb = torch.empty((n, 8 * H, 8 * H, 3), dtype=torch.uint8, device=dev)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())

    def run():
        if cin == 8:
            c.check(c.lib.sdb_edit_image_dev(c.h, p(image), p(ctx), n, L, p(unc), 2, TS, IS, STEPS, p(lat0), H, H, None, p(rgb), st))
        else:
            c.check(c.lib.sdb_sample_image_dev(c.h, p(ctx), n, L, p(unc), 2, TS, STEPS, p(lat0), H, H, p(rgb), st))
    return c, run


def call(cin, n):
    """ms of one call, after two warm-up calls."""
    c, run = setup(cin, n)
    run(), run()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); run(); b.record(); torch.cuda.synchronize()
    print(f"RESULT {a.elapsed_time(b):.3f}")
    c.close()


def step(cin, n):
    """mean device time of the fused guidance + update kernel over one call's 20 steps, from torch.profiler (graphs off)."""
    from torch.profiler import ProfilerActivity, profile
    c, run = setup(cin, n)
    c.set_option("graphs", 0)
    run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    name = f"cfg_step_kernel<0, false, false, {3 if cin == 8 else 2}>"
    us = [e.device_time for e in prof.events() if name in e.name and e.device_time > 0]
    print(f"RESULT {np.mean(us):.3f} {len(us)}")
    c.close()


def conv_in(cin, nb):
    """mean device time of the conv_in kernel over 20 UNet passes (sdb_unet_forward_dev), from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    c, dev = context(cin), torch.device("cuda:0")
    x = torch.randn((nb, cin, H, H), device=dev)
    ctx = torch.from_numpy(synth.make_context(nb, L)).to(dev)
    out = torch.empty((nb, 4, H, H), device=dev)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())
    fwd = lambda: c.check(c.lib.sdb_unet_forward_dev(c.h, p(x), 500, p(ctx), nb, H, H, L, p(out), st))
    fwd(), fwd()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            fwd()
        torch.cuda.synchronize()
    name = "conv3x3_cin4_kernel" if cin == 4 else "conv3x3_cin_cond_kernel"
    us = [e.device_time for e in prof.events() if name in e.name and e.device_time > 0]
    print(f"RESULT {np.mean(us):.3f} {len(us)}")
    c.close()


def sub(*args):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), *map(str, args)], capture_output=True, text=True)
    line = [s for s in r.stdout.splitlines() if s.startswith("RESULT")]
    if r.returncode or not line:
        raise RuntimeError(f"{args}: {r.stdout[-2000:]} {r.stderr[-2000:]}")
    return [float(v) for v in line[0].split()[1:]]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print("card:", q.stdout.strip() or q.stderr.strip(), flush=True)


def main():
    card()
    for n in (1, 4):
        ms = {4: [], 8: []}
        for _ in range(3):
            for cin in (4, 8):
                ms[cin].append(sub("call", cin, n)[0])
        for cin, what in ((4, "txt2img, 4-channel"), (8, "edit, 8-channel")):
            print(f"n={n} {what:20s} ms {' '.join(f'{t:8.2f}' for t in ms[cin])}   images/s "
                  f"{' '.join(f'{1e3 * n / t:6.3f}' for t in ms[cin])}", flush=True)
    for nb in (3, 12):
        for cin in (4, 8):
            us, k = sub("conv_in", cin, nb)
            print(f"conv_in cin={cin} 64x64 nb={nb}: {us:.2f} us per launch ({int(k)} launches)", flush=True)
    for n in (1, 4):
        for cin, what in ((4, "two-way cfg_step_kernel"), (8, "three-way cfg_step_kernel")):
            us, k = sub("step", cin, n)
            print(f"step n={n} {what}: {us:.2f} us per launch ({int(k)} launches)", flush=True)
    card()


if __name__ == "__main__":
    if len(sys.argv) > 1:
        {"call": call, "conv_in": conv_in, "step": step}[sys.argv[1]](int(sys.argv[2]), int(sys.argv[3]))
    else:
        main()
