"""Generates tests/golden/ldm_keymap.json.gz: the map from the keys of an SD-1.x single-file checkpoint (the original LDM layout)
to this repo's registry names, as the REFERENCE'S OWN converter applies it. Needs the reference checkout: set SDB_REFERENCE_DIR
to it.

  python tests/ref_shim/make_ckpt_map.py

The reference converts a checkpoint in two steps (python/dump.py, __main__): load_state_dict assigns each checkpoint tensor to
the attribute of dump.py's StableDiffusion() whose state-dict name equals the key, then the reference's savers write every
attribute to the dump-dir tree whose names are the registry names. This script runs both halves on the tinygrad stand-in:

1. builds StableDiffusion() and walks its attribute tree the way tinygrad's get_state_dict names it (lists by index, dicts by
   key, namedtuples by field, objects by attribute): the checkpoint key of every parameter;
2. runs the reference's savers and matches each saved tensor to its parameter (run_reference.derive_names);
3. records, per checkpoint key: the registry name, the checkpoint (LDM) shape, and "copy" or "transpose" (the saver writes a
   Linear weight transposed, python/save.py:19).

The schedule (alphas_cumprod -> alpha_cumulative_products) is not a parameter of a module and is left out.
"""
import gzip
import json
import os
import shutil
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, HERE]
import run_reference as R  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ldm_keymap.json.gz")


def state_dict_names(obj, prefix, out, Tensor):
    """tinygrad.nn.state.get_state_dict: the key load_state_dict matches against each parameter."""
    if isinstance(obj, Tensor):
        out[id(obj)] = (prefix.strip("."), obj)
    elif isinstance(obj, tuple) and hasattr(obj, "_asdict"):
        state_dict_names(obj._asdict(), prefix, out, Tensor)
    elif isinstance(obj, (list, tuple)):
        for i, x in enumerate(obj):
            state_dict_names(x, f"{prefix}{i}.", out, Tensor)
    elif isinstance(obj, dict):
        for k, v in obj.items():
            state_dict_names(v, f"{prefix}{k}.", out, Tensor)
    elif hasattr(obj, "__dict__") and not isinstance(obj, type) and not hasattr(obj, "__code__"):  # not Tensor.silu / lambdas
        state_dict_names(vars(obj), prefix, out, Tensor)


def main():
    if not R.available():
        sys.exit("set SDB_REFERENCE_DIR to the reference checkout")
    t0 = time.time()
    ref = R.Reference(seed=5)
    keys = {}
    state_dict_names(ref.model, "", keys, ref.Tensor)
    tmp = ("/dev/shm" if os.path.isdir("/dev/shm") else "/tmp") + "/sdb200_ckpt_map"
    shutil.rmtree(tmp, ignore_errors=True)
    ref.save(tmp)
    names = ref.derive_names(tmp)
    shutil.rmtree(tmp, ignore_errors=True)
    entries = {}
    for reg, (p, tr) in names.items():
        if reg == "alphas_cumprod":
            continue
        key, _ = keys[id(p)]
        assert key not in entries, key
        entries[key] = [reg, list(p.t.shape), "transpose" if tr else "copy"]
    assert len(entries) == len(keys) - 1, (len(entries), len(keys))  # every parameter but the schedule
    text = json.dumps(dict(sorted(entries.items())), separators=(",", ":"))
    with open(OUT, "wb") as f:
        f.write(gzip.compress(text.encode(), mtime=0))
    print(len(entries), "keys", f"{time.time() - t0:.0f}s")


if __name__ == "__main__":
    main()
