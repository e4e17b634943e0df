"""Load time of an SD-1.x .safetensors checkpoint (DESIGN.md §7 f13) on the device, against the other ways weights get into a
context. Input: a synthetic 4-channel F16 checkpoint in the LDM layout (synth.make_params(0), read back from the device), about
2.1 GB, written to a temporary directory with the dump-dir of the same weights; the page cache is warmed by one read of each.
Three alternated runs of, host clock around each synchronous call:
  safetensors  sdb_load_safetensors
  pread        the reads alone: os.preadv of the byte ranges the loader reads (runs of back-to-back mapped tensors)
  numpy        lora.read_safetensors + sdb_set_tensor per tensor (Linear weights transposed on the host)
  dump-dir     sdb_load_dump_dir of the same weights
Then one profiled sdb_load_safetensors (torch.profiler, CUDA activities): the convert kernels' and the host-to-device copies'
device time. GB/s are of the checkpoint's file bytes. The card, its power limit and the CPU are read in the same process.
Usage: python tools/checkpoint_time.py"""
import gzip
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

from stable_diffusion_burn_b200 import _lib, dumpdir, lora, synth  # noqa: E402
from test_checkpoint_cpu import ldm_entries, read_header, write_safetensors  # noqa: E402

c = _lib.Context(0)
c.init_synthetic(0)
shapes = dict(c.tensor_list())
tmp = tempfile.mkdtemp(prefix="sdb_ckpt_time_")
path = os.path.join(tmp, "sd14_f16.safetensors")
params, tensors = {}, []
for key, reg, shape, tr in ldm_entries(4):
    a = c.get_tensor(reg, shapes[reg]).astype(np.float16)
    params[reg] = a.astype(np.float32)
    tensors.append((key, "F16", shape, np.ascontiguousarray(a.T if tr else a).astype("<f2").tobytes()))
sched = synth.alpha_cumulative_products()
tensors.append(("alphas_cumprod", "F32", (1000,), sched.astype("<f4").tobytes()))
params["alpha_cumulative_products"] = sched
write_safetensors(path, tensors)
del tensors
root = os.path.join(tmp, "dump")
dumpdir.save_dump_dir(root, params)
del params
size = os.path.getsize(path)
print(f"checkpoint: {size / 1e9:.3f} GB F16, {len(read_header(path))} tensors")

with open(os.path.join(ROOT, "tests", "golden", "ldm_keymap.json.gz"), "rb") as f:
    KEYMAP = json.loads(gzip.decompress(f.read()))


def warm():
    for d, _, fs in os.walk(tmp):
        for name in fs:
            with open(os.path.join(d, name), "rb") as f:
                while f.read(1 << 26):
                    pass


def host_s(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def load_safetensors():
    c.load_safetensors(path)


hdr = read_header(path)
with open(path, "rb") as f:
    body = 8 + int.from_bytes(f.read(8), "little")
ranges = sorted((body + v["data_offsets"][0], body + v["data_offsets"][1]) for v in hdr.values())
runs = []
for b, e in ranges:
    if runs and runs[-1][1] == b:
        runs[-1][1] = e
    else:
        runs.append([b, e])
buf = bytearray(max(64 << 20, max(e - b for b, e in ranges)))


def preads():
    fd = os.open(path, os.O_RDONLY)
    try:
        for b, e in runs:
            o = b
            while o < e:
                n = os.preadv(fd, [memoryview(buf)[:min(len(buf), e - o)]], o)
                o += n
    finally:
        os.close(fd)


def numpy_set_tensor():
    arrays = lora.read_safetensors(path)
    for key, a in arrays.items():
        if key == "alphas_cumprod":
            c.set_tensor("alpha_cumulative_products", a)
            continue
        reg, _, op = KEYMAP[key]
        c.set_tensor(reg, a.T if op == "transpose" else a)


def load_dump_dir():
    c.load_dump_dir(root)


warm()
runs_s = {"safetensors": [], "pread": [], "numpy": [], "dump-dir": []}
for _ in range(3):
    for name, fn in (("safetensors", load_safetensors), ("pread", preads), ("numpy", numpy_set_tensor),
                     ("dump-dir", load_dump_dir)):
        runs_s[name].append(host_s(fn))
for name, v in runs_s.items():
    print(f"{name:12s} s {' '.join(f'{x:7.3f}' for x in v)}  median {sorted(v)[1]:7.3f}  "
          f"{size / 1e9 / sorted(v)[1]:6.2f} GB/s of file bytes")

from torch.profiler import ProfilerActivity, profile  # noqa: E402

with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    t = host_s(load_safetensors)
kern = copy = 0.0  # microseconds
nkern = 0
for e in prof.key_averages():
    us = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
    if "convert_tensors_kernel" in e.key:
        kern += us
        nkern += e.count
    elif "Memcpy HtoD" in e.key:
        copy += us
print(f"profiled load {t:.3f} s: convert_tensors_kernel {nkern} launches {kern / 1e3:.1f} ms "
      f"({100 * kern / 1e6 / t:.1f} % of the call), host-to-device copies {copy / 1e3:.1f} ms")
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True)
print("card:", q.stdout.strip() or q.stderr.strip())
q = subprocess.run(["lscpu"], capture_output=True, text=True)
info = dict(ln.split(":", 1) for ln in q.stdout.splitlines() if ":" in ln)
cpu = " ".join(info.get(k, "").strip() for k in ("Vendor ID", "Model name")).strip() or "unknown"
print(f"cpu: {cpu}, {os.cpu_count()} logical CPUs")
c.close()
shutil.rmtree(tmp)
