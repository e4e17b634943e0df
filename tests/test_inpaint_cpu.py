"""Inpainting with a 9-channel UNet (DESIGN.md §7 f9) without a GPU: the 9-channel registry, the mask rules, the masked image,
the oracle's zero-weight identity with image-to-image, argument errors and the inpaint_b2 fixture."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import sd_oracle as O  # noqa: E402
from stable_diffusion_burn_b200 import synth, topology  # noqa: E402

import img2img_oracle as IO  # noqa: E402
import inpaint_oracle as NO  # noqa: E402
import sampler_oracle as SO  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "inpaint_b2.npz")
CONV_IN = "unet/input_blocks/conv/weight"


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def test_topology_differs_in_conv_in_only():
    four, nine = topology.all_params(), topology.all_params(inpaint=True)
    assert [p[0] for p in four] == [p[0] for p in nine]
    diff = [(a, b) for a, b in zip(four, nine) if a != b]
    assert diff == [((CONV_IN, (320, 4, 3, 3), "conv_w", 36), (CONV_IN, (320, 9, 3, 3), "conv_w", 81))]
    with pytest.raises(ValueError):
        topology.unet_params(in_channels=8)


def test_synthetic_tensors_equal_but_conv_in():
    which4 = topology.unet_params()[:8]
    which9 = topology.unet_params(in_channels=9)[:8]
    p4, p9 = synth.make_params(0, which4), synth.make_params(0, which9)
    for n in p4:
        if n != CONV_IN:
            assert np.array_equal(p4[n], p9[n]), n
    assert p9[CONV_IN].shape == (320, 9, 3, 3)
    assert np.abs(p9[CONV_IN]).max() <= np.sqrt(3.0 / 81) + 1e-7  # fan-in 81


def test_mask_binarised_at_128_and_picked_nearest():
    m = np.zeros((1, 16, 24), np.uint8)
    m[0, 0, 0], m[0, 8, 8], m[0, 8, 16] = 127, 128, 255
    m[0, 1:8, 1:8] = 255  # not a pick point: nearest, not an area rule
    lat = NO.latent_mask(m)
    assert lat.dtype == np.float32 and lat.shape == (1, 2, 3)
    assert lat.tolist() == [[[0.0, 0.0, 0.0], [0.0, 1.0, 1.0]]]
    v = np.arange(256, dtype=np.uint8).reshape(1, 16, 16)
    assert np.array_equal(NO.binary_mask(v), v >= 128)
    # F.interpolate's default nearest mode picks the same cells
    t = torch.from_numpy(NO.binary_mask(m).astype(np.float32))[:, None]
    assert np.array_equal(F.interpolate(t, size=(2, 3))[:, 0].numpy(), lat)


def test_masked_image_is_zero_under_the_mask():
    image, mask = IO.img2img_inputs()
    x = IO.image_u8_to_float(image)
    xm = NO.masked_image(image, mask)
    hole = np.broadcast_to(NO.binary_mask(mask)[:, None], x.shape)
    assert xm.dtype == np.float32 and hole.any() and (~hole).any()
    assert (xm[hole] == 0).all() and not np.signbit(xm[hole]).any()
    assert np.array_equal(xm[~hole], x[~hole])
    assert ((mask > 0) & (mask < 128)).any()  # the soft values below 128 are kept


@pytest.fixture(scope="module")
def small():
    """Full-model oracle at the smallest shapes (tests/test_img2img_cpu.py: small) on the 9-channel weights."""
    torch.set_num_threads(os.cpu_count() or 1)
    params = synth.make_params(0, inpaint=True)
    y, x = np.mgrid[0:64, 0:64]
    img = np.stack([4 * x, 4 * y, 255 - 2 * (x + y)], -1).clip(0, 255).astype(np.uint8)[None]
    mask = np.zeros((1, 64, 64), np.uint8)
    mask[0, 16:48, 8:40] = 200
    return dict(params=params, img=img, mask=mask, ctx=torch.from_numpy(synth.make_context(1, 3, seed=8)),
                unc=torch.from_numpy(synth.make_context(1, 2, seed=99))[0], noise=synth.make_latent(1, 8, 8, seed=9))


@pytest.mark.parametrize("kind", [SO.DDIM, SO.DPMPP_2M])
def test_zero_weights_are_img2img_without_mask(small, kind):
    p = dict(small["params"])
    w4 = synth.make_params(0, [(CONV_IN, (320, 4, 3, 3), "conv_w", 36)])[CONV_IN]
    p[CONV_IN] = NO.zero_extension(w4)
    P9 = O.Params(p)
    p4 = dict(small["params"]); p4[CONV_IN] = w4
    P4 = O.Params(p4)
    with torch.no_grad():
        got = NO.inpaint_latent(P9, small["ctx"], small["unc"], 5.0, 2, small["img"], 1.0, small["noise"], small["mask"],
                                kind=kind).numpy()
        want = SO.sampler_img2img_latent(P4, small["ctx"], small["unc"], 5.0, 2, small["img"], 1.0, small["noise"],
                                         kind=kind).numpy()
    assert rel(got, want) < 1e-6


def test_argument_errors(small):
    P = O.Params(small["params"])
    args = (P, small["ctx"], small["unc"], 5.0, 2, small["img"])
    with pytest.raises(ValueError, match="mask"):
        NO.inpaint_latent(*args, 1.0, small["noise"], None)
    for s in (0.0, 1.5, float("nan"), 0.1):
        with pytest.raises(ValueError, match="strength"):
            NO.inpaint_latent(*args, s, small["noise"], small["mask"])
    with pytest.raises(ValueError):
        NO.inpaint_latent(*args, 1.0, small["noise"], small["mask"], kind=SO.DPMPP_2M, eta=0.5)


def test_fixture_inputs_and_mask():
    g = np.load(GOLD)
    image, mask = IO.img2img_inputs()
    assert np.array_equal(g["image"], image) and np.array_equal(g["mask"], mask)
    assert np.array_equal(g["noise"], synth.make_latent(2, 32, 32, seed=41))
    assert np.array_equal(g["m_lat"], NO.latent_mask(mask))
    assert (g["m_lat"] == 0).any() and (g["m_lat"] == 1).any()
    assert g["z_m"].shape == (2, 4, 32, 32)


def test_fixture_rederived():
    """The whole fixture from its script's recipe (both cases; about a minute on 8 cores)."""
    g = np.load(GOLD)
    torch.set_num_threads(os.cpu_count() or 1)
    P = O.Params(synth.make_params(0, inpaint=True))
    ctx = torch.from_numpy(synth.make_context(2, 7, seed=3))
    unc = torch.from_numpy(synth.make_context(1, 2, seed=99))[0]
    for name, c in NO.INPAINT_CASES.items():
        taps = {}
        with torch.no_grad():
            lat = NO.inpaint_latent(P, ctx, unc, NO.INPAINT["scale"], NO.INPAINT["n_steps"], g["image"], c["strength"], g["noise"],
                                    g["mask"], kind=c["kind"], taps=taps)
            u8 = O.to_u8(O.latent_to_image_f32(P, lat))
        assert rel(taps["z_m"], g["z_m"]) < 1e-5
        assert rel(lat.numpy(), g[f"latent_{name}"]) < 1e-4, name
        d = np.abs(u8[:, ::2, ::2, :].astype(np.int16) - g[f"u8_{name}"].astype(np.int16))
        assert (d <= 1).mean() >= 0.999 and d.max() <= 2, name
