"""Generates the stored data of the test_live_* tests (tests/test_ref_pin_cpu.py): what the REFERENCE'S OWN Python model and saver
(python/dump.py and python/stablediffusion.py of the reference checkout, run unmodified on tests/ref_shim/tinygrad) produce on this
repo's synthetic weights (seed 0). Needs the reference checkout: set SDB_REFERENCE_DIR to it.

  python tests/ref_shim/make_live_golden.py

* tests/golden/ref_live_tree.json.gz: the dump-dir tree the reference's saver writes for those weights: every file with its size and
  a digest of the array it holds; and the registry name of every tensor it wrote.
* tests/golden/ref_live.npz: the reference's forwards on those weights (inputs regenerated from seeds by the test; the larger
  outputs as the fixed sample of elements live_sample takes).
"""
import gzip
import json
import os
import shutil
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, HERE]
import run_reference as R  # noqa: E402
from stable_diffusion_burn_b200 import synth, topology  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_ref_pin_cpu import array_digest, live_inputs, live_sample, rel  # noqa: E402

OUT_TREE = os.path.join(ROOT, "tests", "golden", "ref_live_tree.json.gz")
OUT_NPZ = os.path.join(ROOT, "tests", "golden", "ref_live.npz")


def main():
    torch.set_num_threads(os.cpu_count())
    t0 = time.time()
    tmp = ("/dev/shm" if os.path.isdir("/dev/shm") else "/tmp") + "/sdb200_ref_live"
    ref = R.Reference(seed=11)
    shutil.rmtree(tmp, ignore_errors=True)
    ref.save(tmp)
    ref.derive_names(tmp)
    shutil.rmtree(tmp, ignore_errors=True)
    print("reference model built, names derived", f"{time.time() - t0:.0f}s", flush=True)
    params = synth.make_params(0)
    assert ref.assign(params) == len(ref.names)
    ref.set_alphas(params["alpha_cumulative_products"])
    ref.save(tmp)  # the reference's writer, now holding the synthetic weights
    files = {}
    for d, _, fs in os.walk(tmp):
        for f in fs:
            p = os.path.join(d, f)
            size = os.path.getsize(p)
            files[os.path.relpath(p, tmp)] = [size, array_digest(np.load(p))]
    shutil.rmtree(tmp, ignore_errors=True)
    written = sorted("alpha_cumulative_products" if k == "alphas_cumprod" else k for k in ref.names)
    text = json.dumps({"written": written, "files": dict(sorted(files.items()))}, separators=(",", ":"))
    with open(OUT_TREE, "wb") as f:
        f.write(gzip.compress(text.encode(), mtime=0))
    print("tree:", len(files), "files", f"{time.time() - t0:.0f}s", flush=True)

    x, c, lat, img, tok = live_inputs()
    keep = {"unet": ref.unet_forward(x, 321, c), "decode": live_sample(ref.decode_latent(lat)), "encode": ref.encode_image(img),
            "autoencoder": live_sample(ref.autoencoder_forward(img)), "clip": live_sample(ref.clip_forward(tok)),
            "temb": ref.timestep_embedding(321)}
    ref.assign(synth.make_params(0, which=topology.vae_decoder_params()))
    fixture = np.load(os.path.join(ROOT, "tests", "golden", "ref_python.npz"))
    keep["dec16:img"] = live_sample(ref.decode_latent(fixture["dec16:lat"]))
    # the committed fixture is what the reference outputs on the synthetic decoder weights
    assert rel(keep["dec16:img"], live_sample(fixture["dec16:img"])) < 1e-6
    np.savez_compressed(OUT_NPZ, **{k: np.asarray(v, np.float32) for k, v in keep.items()})
    print("forwards stored", f"{time.time() - t0:.0f}s", flush=True)


if __name__ == "__main__":
    main()
