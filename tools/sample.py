"""Stand-in for the reference's `sample` binary with ITS argv (src/bin/sample/main.rs:36-57) on the device path:

  sample <model_type(burn or dump)> <model_name> <unconditional_guidance_scale> <n_diffusion_steps> <prompt> <output_image_name> [device]

  model_type  burn  -> <model_name> is a NamedMpk record file (`SDv1-4.mpk`; stable_diffusion_burn_b200/mpk.py, format unverified)
              dump  -> <model_name> is a dump-dir tree (sdb_load_dump_dir)
              synthetic -> (extension) <model_name> is the seed of the synthetic weight stream: noise images, but end to end
  device      cuda / cudaN (default cuda0). cpu and mps are refused: this library has no CPU fallback (main.rs:61-77 accepts them).
Same messages, same exit codes (1 on a usage / parse / load error), images written as <output_image_name><i>.png like save_images
(main.rs:115-122). The host side of the reference is Rust; with no Rust toolchain in this image the runnable stand-in is Python
over the same C ABI (rust/sdb200_ffi.rs is the source-only Rust binding). Not part of the measured path (bench.py is).
"""
import os
import struct
import sys
import zlib

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402


def write_png(path, rgb):
    """8-bit RGB PNG, no dependency: rgb [H, W, 3] uint8."""
    h, w, _ = rgb.shape
    raw = b"".join(b"\x00" + rgb[y].tobytes() for y in range(h))

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)) +
                chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))


def parse_args(argv):
    """-> (model_type, model_name, scale, n_steps, prompt, output, device index) or raises SystemExit(1) with the reference's text."""
    if len(argv) not in (7, 8):
        print(f"Usage: {argv[0]} <model_type(burn or dump)> <model_name> <unconditional_guidance_scale> <n_diffusion_steps> "
              "<prompt> <output_image_name> [device(cuda, mps, cpu)]", file=sys.stderr)
        raise SystemExit(1)
    try:
        scale = float(argv[3])
    except ValueError:
        print("Error: Invalid unconditional guidance scale.", file=sys.stderr)
        raise SystemExit(1)
    try:
        n_steps = int(argv[4])
        if n_steps < 0:
            raise ValueError
    except ValueError:
        print("Error: Invalid number of diffusion steps.", file=sys.stderr)
        raise SystemExit(1)
    dev = 0
    if len(argv) == 8:
        d = argv[7].lower()
        if d.startswith("cuda"):
            try:
                dev = int(d[4:]) if d[4:] else 0
            except ValueError:
                dev = 0
        elif d in ("cpu", "mps"):
            print(f"Device {d}: this library runs on sm_90a (H100) GPUs only (no CPU fallback)", file=sys.stderr)
            raise SystemExit(1)
        else:
            print(f"Unknown device: {argv[7]}", file=sys.stderr)
            raise SystemExit(1)
    return argv[1], argv[2], scale, n_steps, argv[5], argv[6], dev


def main(argv):
    kind, model, scale, n_steps, prompt, out, dev = parse_args(argv)
    from stable_diffusion_burn_b200 import mpk, pipeline, tokenizer
    print("Loading tokenizer...")
    tok = tokenizer.SimpleTokenizer(tokenizer.find_vocab())
    print("Loading model...")
    sd = pipeline.StableDiffusion(dev)
    try:
        if kind == "burn":
            n = mpk.load_into(sd.ctx, model)
            if n == 0:
                raise RuntimeError("no tensor of the model found in the file")
            sd.ctx.finalize_weights()
        elif kind == "synthetic":
            sd = sd.init_synthetic(int(model))
        else:
            sd = sd.load_dump_dir(model)
    except Exception as err:
        print(f"Error loading model{'' if kind == 'burn' else ' dump'}: {err}", file=sys.stderr)
        return 1
    unconditional_context = sd.unconditional_context(tok)
    context = sd.context(tok, prompt)
    print("Sampling image...")
    images = sd.sample_image(context, unconditional_context, scale, n_steps)
    try:
        for i, img in enumerate(images):
            write_png(f"{out}{i}.png", np.asarray(img, np.uint8).reshape(512, 512, 3))
    except OSError as err:
        print(f"Error saving image: {err}", file=sys.stderr)
        return 1
    sd.close()
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
