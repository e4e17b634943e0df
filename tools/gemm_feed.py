"""Where the gemm_tc time goes, set against how fast the operand tiles have to arrive.

  python tools/gemm_feed.py [--steps 20] [--out DIR]

1. Per-launch table of one sample_image (512x512, batch 1, CFG), from the event-bracketed launches of profile mode
   (SDB_PROFILE_DUMP): for each distinct GEMM label the launch count, time, issued TFLOP/s and the modelled L2 -> shared
   bytes with the bandwidth they imply. Modelled bytes = CTAs x k-chunks per CTA x stage bytes / multicast sharing.
2. Feed probe: the level-0 conv's mainloop (45 k-chunks of a 128 x 160 tile, 3 passes) as a Linear M = 8192, K = 2880,
   N = 320 (128 CTAs), against M = 1024 with split-K off (16 CTAs), and the clock64 stamps of CTA 0 (SDB_GEMM_DBG):
   cycles from the first operands landing to the last product, as FLOP per cycle per SM (data sheet: 4096 fp16 dense).
   Similar per-CTA times at 128 and 16 CTAs mean the mainloop is not limited by L2 bandwidth.

Needs a GPU. With --out DIR the results are also written as DIR/gemm_feed.json.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BM, BK = 128, 64
KINDS = {0: "linear", 2: "conv3", 3: "conv3/s2", 4: "conv3/up2", 5: "conv3/s2p"}
LABEL = re.compile(r"gemm kind=(\d+) n=(\d+) H=(\d+) W=(\d+) P=\d+ C0=(\d+) C1=(\d+) N=(\d+) K=(\d+) xk=(\d+) BN=(\d+) "
                   r"split=(\d+) passes=(\d) geglu=(\d) epi=(\S+) tile=(\d+)x(\d+)x(\d+)(?: cl=(\d)x(\d))?")


def cdiv(a, b):
    return (a + b - 1) // b


def model(label):
    """Shape facts of one gemm launch label: CTAs, k-chunks per CTA, stage bytes, issued FLOPs, modelled L2 -> shared bytes."""
    m = LABEL.search(label)
    if not m:
        return None
    kind, n, H, W, C0, C1, N, K, xk, BN, split, passes, geglu, epi, TN, TH, TW = (
        int(v) if v.lstrip("-").isdigit() else v for v in m.groups()[:17])
    cm, cn = int(m.group(18) or 1), int(m.group(19) or 1)
    ctot = C0 + C1
    taps = K // ctot
    iters = taps * (ctot // BK) + xk // BK
    m_tiles = cdiv(W, TW) * cdiv(H, TH) * cdiv(n, TN)
    n_tiles = cdiv(N, BN)
    z = 4 if kind == 4 else split
    per = cdiv(iters, split)
    chunks = sum(max(0, min(iters, (k + 1) * per) - k * per) for k in range(split)) if kind != 4 else iters * 4
    a_bytes = BM * BK * 2 * (2 if passes >= 2 else 1)
    b_bytes = BN * BK * 2 * (2 if passes >= 3 else 1)
    # each CTA of an N-pair reads half of the shared A tile, each CTA of an M-pair half of the shared B tile
    l2_bytes = m_tiles * n_tiles * chunks * (a_bytes / cn + b_bytes / cm)
    rows = n * H * W * (4 if kind == 4 else 1)
    issued = 2.0 * rows * N * (K + xk) * passes
    return dict(kind=KINDS.get(kind, str(kind)), n=n, H=H, W=W, N=N, K=K + xk, BN=BN, split=split, passes=passes, epi=epi,
                ctas=m_tiles * n_tiles * z, chunks_per_cta=per, stage_bytes=a_bytes + b_bytes, cluster=f"{cm}x{cn}",
                issued_flop=issued, l2_bytes=l2_bytes)


def gpu_facts():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              check=True).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def read_dump(path):
    rows = []
    with open(path) as f:
        for line in f:
            parts = line.rstrip("\n").split("\t")
            if len(parts) == 5 and parts[0] == "gemm_tc":
                rows.append((float(parts[1]), parts[4]))
    return rows


def launch_table(steps):
    """Child process: one sample_image in profile mode, GEMM launches aggregated by label."""
    from stable_diffusion_burn_b200 import _lib, synth
    c = _lib.Context(0)
    c.init_synthetic(0)
    c.finalize_weights()
    ctx, unc = synth.make_context(1, 77), synth.make_context(1, 2, seed=99)[0]
    lat = synth.make_latent(1, 64, 64)
    c.sample_image(ctx, unc, 7.5, steps, init_latent=lat)  # warm: module loads, workspaces
    c.profile(True)
    c.profile_reset()
    c.sample_image(ctx, unc, 7.5, steps, init_latent=lat)
    c.profile(False)  # collects: the dump file is complete
    c.close()


def probe():
    """Child process (SDB_GEMM_DBG set): the feed probe's launches."""
    import numpy as np
    from stable_diffusion_burn_b200 import _lib
    c = _lib.Context(0)
    rng = np.random.default_rng(0)
    K, N = 2880, 320
    w = (rng.standard_normal((K, N)) * K ** -0.5).astype(np.float32)
    for M, splitk in ((8192, 1), (1024, 0)):
        c.set_option("splitk", splitk)
        a = rng.standard_normal((M, K)).astype(np.float32)
        c.test_linear(a, w, None, passes=3)  # warm
        c.profile(True)
        for _ in range(10):
            c.test_linear(a, w, None, passes=3)
        c.profile(False)
    c.close()


def run_child(mode, steps, env_extra):
    fd, dump = tempfile.mkstemp(prefix="gemm_feed_", suffix=".tsv")
    os.close(fd)
    env = dict(os.environ, SDB_PROFILE_DUMP=dump, **env_extra)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", mode, "--steps", str(steps)], env=env,
                       capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise SystemExit(f"{mode} child failed ({r.returncode})")
    rows = read_dump(dump)
    os.unlink(dump)
    return rows, r.stderr


def summarize(rows):
    agg = {}
    for us, label in rows:
        e = agg.setdefault(label, {"count": 0, "us": 0.0})
        e["count"] += 1
        e["us"] += us
    out = []
    for label, e in agg.items():
        f = model(label)
        if f is None:
            continue
        s = e["us"] * 1e-6
        f.update(count=e["count"], us_total=e["us"], us_per_launch=e["us"] / e["count"],
                 issued_tflops=f["issued_flop"] * e["count"] / s / 1e12, l2_tbs=f["l2_bytes"] * e["count"] / s / 1e12, label=label)
        out.append(f)
    out.sort(key=lambda r: -r["us_total"])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child == "table":
        return launch_table(args.steps)
    if args.child == "probe":
        return probe()

    facts = gpu_facts()
    print(f"# gpu: {facts}")
    rows, _ = run_child("table", args.steps, {})
    table = summarize(rows)
    tot = sum(r["us_total"] for r in table)
    print(f"# gemm_tc in one sample_image ({args.steps} steps, profile mode): {tot / 1e3:.2f} ms over "
          f"{sum(r['count'] for r in table)} launches")
    print(f"{'kind':10s} {'n':>2s} {'HxW':>9s} {'N':>5s} {'K':>5s} {'BN':>3s} {'sp':>2s} {'p':>1s} {'cl':>3s} {'ctas':>4s} "
          f"{'ch':>3s} {'cnt':>4s} {'us/launch':>9s} {'ms':>7s} {'TFLOP/s':>7s} {'L2 TB/s':>7s}")
    for r in table:
        print(f"{r['kind']:10s} {r['n']:2d} {r['H']:4d}x{r['W']:<4d} {r['N']:5d} {r['K']:5d} {r['BN']:3d} {r['split']:2d} "
              f"{r['passes']:1d} {r['cluster']:>3s} {r['ctas']:4d} {r['chunks_per_cta']:3d} {r['count']:4d} "
              f"{r['us_per_launch']:9.1f} {r['us_total'] / 1e3:7.2f} {r['issued_tflops']:7.1f} {r['l2_tbs']:7.2f}")

    prow, perr = run_child("probe", args.steps, {"SDB_GEMM_DBG": "1"})
    dbg = re.compile(r"gemm_dbg (gemm .*?) \| cycles since entry: .*?landed (-?\d+) lastmma (-?\d+)")
    probes = []
    for M, ctas in ((8192, 128), (1024, 16)):
        us = sorted(t for t, l in prow if f" W={M} " in l and "passes=3" in l)
        cyc = sorted(int(m.group(3)) - int(m.group(2)) for m in dbg.finditer(perr) if f" W={M} " in m.group(1))
        f = model(next(l for t, l in prow if f" W={M} " in l))
        per_cta_flop = f["issued_flop"] / f["ctas"]
        med_us, med_cyc = us[len(us) // 2], cyc[len(cyc) // 2]
        probes.append(dict(M=M, ctas=f["ctas"], chunks=f["chunks_per_cta"], split=f["split"], us_median=med_us, us_min=us[0],
                           l2_tbs=f["l2_bytes"] / (med_us * 1e-6) / 1e12, mainloop_cycles=med_cyc,
                           flop_per_cycle_per_sm=per_cta_flop / med_cyc))
    print("# feed probe: Linear K=2880 N=320, 3 passes, 45 k-chunks per CTA (kernel time = per-CTA time: one wave)")
    for p in probes:
        print(f"M={p['M']:5d} ctas={p['ctas']:3d} split={p['split']}: {p['us_median']:.1f} us (min {p['us_min']:.1f}), "
              f"modelled L2->smem {p['l2_tbs']:.2f} TB/s; CTA 0 landed->lastmma {p['mainloop_cycles']} cycles = "
              f"{p['flop_per_cycle_per_sm']:.0f} FLOP/cycle/SM ({p['flop_per_cycle_per_sm'] / 4096:.0%} of 4096)")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "gemm_feed.json"), "w") as f:
            json.dump({"gpu": facts, "steps": args.steps, "table": table, "probe": probes}, f, indent=1)


if __name__ == "__main__":
    main()
