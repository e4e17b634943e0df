"""InstructPix2Pix editing with an 8-channel UNet (DESIGN.md §7 f10) without a GPU: the 8-channel registry, the unscaled image
latent, the oracle's zero-weight identity with text-to-image and its image-scale-1 identity with two-way guidance (both in
float64), argument errors and the pix2pix_b2 fixture."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import sd_oracle as O  # noqa: E402
from stable_diffusion_burn_b200 import _lib, pipeline, synth, topology  # noqa: E402

import img2img_oracle as IO  # noqa: E402
import pix2pix_oracle as PO  # noqa: E402
import sampler_oracle as SO  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "pix2pix_b2.npz")
CONV_IN = "unet/input_blocks/conv/weight"
CONV_IN4 = (CONV_IN, (320, 4, 3, 3), "conv_w", 36)


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def test_registry_differs_in_conv_in_only():
    four, eight = topology.all_params(), topology.all_params(pix2pix=True)
    assert [p[0] for p in four] == [p[0] for p in eight]
    diff = [(a, b) for a, b in zip(four, eight) if a != b]
    assert diff == [(CONV_IN4, (CONV_IN, (320, 8, 3, 3), "conv_w", 72))]
    assert topology.all_params(inpaint=True) == topology.conv_in_width_params(9)
    assert eight == topology.conv_in_width_params(8) and four == topology.conv_in_width_params(4)
    with pytest.raises(ValueError):
        topology.all_params(inpaint=True, pix2pix=True)
    with pytest.raises(ValueError):
        topology.unet_params(in_channels=9, pix2pix=True)
    with pytest.raises(ValueError):
        topology.conv_in_width_params(5)


def test_synthetic_tensors_equal_but_conv_in():
    p4 = synth.make_params(0, topology.unet_params()[:8])
    p8 = synth.make_params(0, topology.unet_params(pix2pix=True)[:8])
    for n in p4:
        if n != CONV_IN:
            assert np.array_equal(p4[n], p8[n]), n
    assert p8[CONV_IN].shape == (320, 8, 3, 3)
    assert np.abs(p8[CONV_IN]).max() <= np.sqrt(3.0 / 72) + 1e-7  # fan-in 72


def test_image_latent_is_unscaled():
    """c_I is the encoder's output itself, the posterior mode, with no 0.18215 factor (unlike img2img's z0)."""
    P = O.Params(synth.make_params(0, which=topology.vae_encoder_params()))
    y, x = np.mgrid[0:64, 0:64]
    img = np.stack([4 * x, 4 * y, 255 - 2 * (x + y)], -1).clip(0, 255).astype(np.uint8)[None]
    with torch.no_grad():
        c_i = PO.image_latent(P, img).numpy()
        enc = O.encode_image(P, torch.from_numpy(IO.image_u8_to_float(img))).numpy()
    assert np.array_equal(c_i, enc)
    assert rel(SO.scaled_latent(enc), c_i) > 0.5


@pytest.fixture(scope="module")
def f64():
    """Float64 oracle weights at the smallest shapes: the 8-channel UNet and the encoder (P8), the same with conv_in channels
    4-7 zero (P8z), and the 4-channel UNet with conv_in = P8z's channels 0-3 (P4). The three share every other tensor."""
    torch.set_num_threads(os.cpu_count() or 1)
    which = topology.unet_params(pix2pix=True) + topology.vae_encoder_params()
    P8 = O.Params(synth.make_params(0, which), dtype=torch.float64)
    w4 = synth.make_params(0, [CONV_IN4])[CONV_IN]
    P8z, P4 = copy.copy(P8), copy.copy(P8)
    P8z.t = dict(P8.t, **{CONV_IN: torch.from_numpy(PO.zero_extension(w4)).double()})
    P4.t = dict(P8.t, **{CONV_IN: torch.from_numpy(w4).double()})
    y, x = np.mgrid[0:64, 0:64]
    img = np.stack([4 * x, 4 * y, 255 - 2 * (x + y)], -1).clip(0, 255).astype(np.uint8)[None]
    return dict(P8=P8, P8z=P8z, P4=P4, img=img, ctx=torch.from_numpy(synth.make_context(1, 3, seed=8)),
                unc=torch.from_numpy(synth.make_context(1, 2, seed=99))[0], latent0=synth.make_latent(1, 8, 8, seed=9))


@pytest.mark.parametrize("kind", [SO.DDIM, SO.DPMPP_2M])
def test_zero_weights_are_txt2img(f64, kind):
    """With conv_in channels 4-7 zero, e_I = e_U whatever s_I, and the edit is text-to-image from the same start latent."""
    with torch.no_grad():
        got = PO.pix2pix_latent(f64["P8z"], f64["ctx"], f64["unc"], 5.0, 1.5, 2, f64["img"], f64["latent0"], kind=kind).numpy()
        want = SO.sampler_latent(f64["P4"], f64["ctx"], f64["unc"], 5.0, 2, torch.from_numpy(f64["latent0"]), kind=kind).numpy()
    assert got.dtype == np.float64
    print(f"zero-weight identity, kind {kind}: rel {rel(got, want):.3e}")
    assert rel(got, want) < 1e-12


@pytest.mark.parametrize("kind", [SO.DDIM, SO.DPMPP_2M])
def test_image_scale_one_is_cfg_on_the_image(f64, kind):
    """s_I = 1: pred = e_I + s_T (e_T - e_I), two-way guidance in which both halves see c_I."""
    P = f64["P8"]
    with torch.no_grad():
        got = PO.pix2pix_latent(P, f64["ctx"], f64["unc"], 5.0, 1.0, 2, f64["img"], f64["latent0"], kind=kind).numpy()
        c_i = PO.image_latent(P, f64["img"])
        guide = lambda x, t: O.forward_diffuser(P, torch.cat([x, c_i], 1), t, f64["ctx"], f64["unc"], 5.0)
        want = SO.guided_latent(P, 2, f64["latent0"], guide, kind=kind).numpy()
    print(f"image scale 1, kind {kind}: rel {rel(got, want):.3e}")
    assert rel(got, want) < 1e-12


def test_argument_errors(f64):
    args = (f64["P8"], f64["ctx"], f64["unc"])
    for bad in (float("nan"), float("inf")):
        with pytest.raises(ValueError, match="text_scale"):
            PO.pix2pix_latent(*args, bad, 1.5, 2, f64["img"], f64["latent0"])
        with pytest.raises(ValueError, match="image_scale"):
            PO.pix2pix_latent(*args, 7.5, bad, 2, f64["img"], f64["latent0"])
    with pytest.raises(ValueError):
        PO.pix2pix_latent(*args, 7.5, 1.5, 2, f64["img"], f64["latent0"], kind=SO.DPMPP_2M, eta=0.5)
    # a context is one kind or the other, rejected before any device is touched
    with pytest.raises(ValueError, match="pix2pix"):
        _lib.Context(0, inpaint=True, pix2pix=True)
    with pytest.raises(ValueError, match="pix2pix"):
        pipeline.StableDiffusion(0, inpaint=True, pix2pix=True)
    # Context.edit_image checks its arrays before the call
    c = object.__new__(_lib.Context)
    img, ctx, unc = f64["img"], synth.make_context(1, 3, seed=8), synth.make_context(1, 2, seed=99)[0]
    with pytest.raises(ValueError, match="latent, the image or both"):
        c.edit_image(img, ctx, unc, 7.5, 1.5, 2, latent=False, rgb=False)
    with pytest.raises(ValueError, match="image"):
        c.edit_image(img[:, :60], ctx, unc, 7.5, 1.5, 2)
    with pytest.raises(ValueError, match="context"):
        c.edit_image(img, synth.make_context(2, 3, seed=8), unc, 7.5, 1.5, 2)
    with pytest.raises(ValueError, match="init_latent"):
        c.edit_image(img, ctx, unc, 7.5, 1.5, 2, init_latent=synth.make_latent(1, 16, 16, seed=1))


def test_fixture_inputs():
    g = np.load(GOLD)
    image, _ = IO.img2img_inputs()
    assert np.array_equal(g["image"], image)
    assert np.array_equal(g["latent0"], synth.make_latent(2, 32, 32, seed=43))
    assert g["c_I"].shape == (2, 4, 32, 32)


def test_fixture_rederived():
    """The whole fixture from its script's recipe (both cases; about a minute and a half on 8 cores)."""
    g = np.load(GOLD)
    torch.set_num_threads(os.cpu_count() or 1)
    P = O.Params(synth.make_params(0, pix2pix=True))
    ctx = synth.make_context(2, 7, seed=3)
    unc = synth.make_context(1, 2, seed=99)[0]
    for name, c in PO.PIX2PIX_CASES.items():
        taps = {}
        with torch.no_grad():
            lat = PO.pix2pix_latent(P, ctx, unc, PO.PIX2PIX["text_scale"], PO.PIX2PIX["image_scale"], PO.PIX2PIX["n_steps"],
                                    g["image"], g["latent0"], kind=c["kind"], taps=taps)
            u8 = O.to_u8(O.latent_to_image_f32(P, lat))
        assert rel(taps["c_I"], g["c_I"]) < 1e-5
        assert rel(lat.numpy(), g[f"latent_{name}"]) < 1e-4, name
        d = np.abs(u8[:, ::2, ::2, :].astype(np.int16) - g[f"u8_{name}"].astype(np.int16))
        assert (d <= 1).mean() >= 0.999 and d.max() <= 2, name
