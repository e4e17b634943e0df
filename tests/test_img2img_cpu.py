"""Image-to-image / inpainting semantics (DESIGN.md §7 f5) in the CPU oracle: the strength -> schedule rule, the exact
identities the GPU suite relies on, the u8 / mask conversions, and the img2img_b2 fixture re-derived."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sd_oracle as O
from stable_diffusion_burn_b200 import synth

import img2img_oracle as IO
import sampler_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "img2img_b2.npz")


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


@pytest.mark.parametrize("n_steps,strength,ts_run", [
    (20, 0.75, list(range(749, -1, -50))),  # 15 steps from t = 749
    (3, 0.5, [333, 0]),                     # N = 4: 999, 666, 333, 0
    (4, 1.0, [999, 749, 499, 249]),
    (4, 0.5, [499, 249]),
    (4, 0.74, [499, 249]),
    (1, 1.0, [999]),
])
def test_strength_to_schedule(n_steps, strength, ts_run):
    first, ts = SO.img2img_start(strength, n_steps)
    assert ts[first:] == ts_run


@pytest.mark.parametrize("n_steps", [1, 4, 20, 50])
def test_strength_below_one_step_rejected(n_steps):
    N = len(O.ddim_timesteps(n_steps)[0])
    SO.img2img_start(1.0 / N, n_steps)  # the smallest valid strength runs one step
    with pytest.raises(ValueError, match=f"1/{N}"):
        SO.img2img_start(np.nextafter(1.0 / N, 0.0), n_steps)
    for bad in (0.0, -0.5, 1.5, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            SO.img2img_start(bad, n_steps)


def test_image_u8_to_float_formula():
    v = np.arange(256, dtype=np.uint8)
    img = np.stack([v, v[::-1], np.roll(v, 7)], -1).reshape(1, 16, 16, 3)
    x = IO.image_u8_to_float(img)
    assert x.dtype == np.float32 and x.shape == (1, 3, 16, 16)
    # fl(fl(v / 127.5) - 1) restated through float64 (double rounding is innocuous for one division / subtraction)
    q = (img.transpose(0, 3, 1, 2).astype(np.float64) / 127.5).astype(np.float32)
    want = (q.astype(np.float64) - 1.0).astype(np.float32)
    assert np.array_equal(x, want)
    assert x.min() == -1.0 and x.max() == 1.0


def test_mask_to_latent_is_the_area_mean():
    rng = np.random.default_rng(5)
    m = rng.integers(0, 256, (3, 64, 48)).astype(np.uint8)
    m[0] = 0
    m[1, :32] = 255
    w = IO.mask_to_latent(m)
    # the pooled mean in float64, rounded once to float32 (pooling float32 quotients would add up to 64 roundings)
    ref = F.avg_pool2d(torch.from_numpy(m.astype(np.float64) / 255.0)[:, None], 8)[:, 0].numpy().astype(np.float32)
    assert w.shape == (3, 8, 6) and w.dtype == np.float32
    ulp = np.abs(w.view(np.int32).astype(np.int64) - ref.view(np.int32).astype(np.int64))
    assert ulp.max() <= 1
    assert (w[0] == 0).all() and (w[1, :4] == 1).all()


# ------------------------------------------------------------------------------------------------ oracle identities
@pytest.fixture(scope="module")
def small():
    """Full-model oracle at the smallest shapes: a 64x64 px image (8x8 latent), L = 3, Lu = 2."""
    torch.set_num_threads(os.cpu_count() or 1)
    P = O.Params(synth.make_params(0))
    y, x = np.mgrid[0:64, 0:64]
    img = np.stack([4 * x, 4 * y, 255 - 2 * (x + y)], -1).clip(0, 255).astype(np.uint8)[None]
    return dict(P=P, img=img, ctx=torch.from_numpy(synth.make_context(1, 3, seed=8)),
                unc=torch.from_numpy(synth.make_context(1, 2, seed=99))[0], noise=synth.make_latent(1, 8, 8, seed=9))


def _run(s, n_steps, strength, mask=None, taps=None):
    with torch.no_grad():
        return SO.sampler_img2img_latent(s["P"], s["ctx"], s["unc"], 5.0, n_steps, s["img"], strength, s["noise"],
                                         mask_u8=mask, taps=taps).numpy()


def test_strength_one_is_txt2img_from_the_noised_image(small):
    taps = {}
    got = _run(small, 2, 1.0, taps=taps)
    a0 = float(small["P"]("alpha_cumulative_products")[999])
    init = SO.start_latent(a0, taps["z0"], small["noise"])
    with torch.no_grad():
        want = O.sample_latent(small["P"], small["ctx"], small["unc"], 5.0, 2, torch.from_numpy(init)).numpy()
    assert np.array_equal(got, want)


def test_mask_identities(small):
    taps = {}
    none = _run(small, 2, 1.0, taps=taps)
    keep = _run(small, 2, 1.0, mask=np.zeros((1, 64, 64), np.uint8))
    regen = _run(small, 2, 1.0, mask=np.full((1, 64, 64), 255, np.uint8))
    assert np.array_equal(keep, taps["z0"])  # after the last step a_prev = 1: the known region is exactly z0
    assert np.array_equal(regen, none)
    assert not np.array_equal(none, taps["z0"])


# ------------------------------------------------------------------------------------------------ fixture
def test_fixture_inputs_and_z0_w():
    g = np.load(GOLD)
    image, mask = IO.img2img_inputs()
    assert np.array_equal(g["image"], image) and np.array_equal(g["mask"], mask)
    assert np.array_equal(g["noise"], synth.make_latent(2, 32, 32, seed=41))
    assert np.array_equal(g["w"], IO.mask_to_latent(mask))
    assert ((g["w"] > 0) & (g["w"] < 1)).any() and (g["w"] == 0).any() and (g["w"] == 1).any()
    torch.set_num_threads(os.cpu_count() or 1)
    from stable_diffusion_burn_b200 import topology
    P = O.Params(synth.make_params(0, which=topology.vae_encoder_params()))
    with torch.no_grad():
        z = O.encode_image(P, torch.from_numpy(IO.image_u8_to_float(image))).numpy()
    # torch's CPU convolutions may pick other algorithms on another machine: the encoder bar of tests/test_vae_encoder.py
    assert rel(g["z0"], SO.scaled_latent(z)) < 1e-5


def test_fixture_rederived(small):
    """The whole fixture from the oracle (about 15 s on 8 cores)."""
    g = np.load(GOLD)
    P = small["P"]
    with torch.no_grad():
        lat = SO.sampler_img2img_latent(P, torch.from_numpy(synth.make_context(2, 7, seed=3)), small["unc"],
                                        IO.IMG2IMG["scale"], IO.IMG2IMG["n_steps"], g["image"], IO.IMG2IMG["strength"],
                                        g["noise"], mask_u8=g["mask"])
        u8 = O.to_u8(O.latent_to_image_f32(P, lat))
    assert rel(lat.numpy(), g["latent"]) < 1e-4
    d = np.abs(u8[:, ::2, ::2, :].astype(np.int16) - g["u8"].astype(np.int16))
    assert (d <= 1).mean() >= 0.999 and d.max() <= 2
