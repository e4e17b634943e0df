"""Image-to-image / masked inpainting on the GPU (DESIGN.md §7 f5) through the C ABI: the img2img_b2 fixture, the bit-exact
identities of the semantics (conversion, final paste, all-255 mask, strength 1 = txt2img), the step-graph cache, the
host / device entries, the launch count, errors and batch independence."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from stable_diffusion_burn_b200 import _lib, synth

import img2img_oracle as IO
import sampler_oracle as SO

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "img2img_b2.npz")
STEPS, STRENGTH, SCALE = 4, 0.5, 5.0  # the fixture's: k = 2, t = 499, 249


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


@pytest.fixture(scope="module")
def sd(ctx):
    ctx.init_synthetic(0)
    ctx.finalize_weights()
    return ctx


@pytest.fixture(scope="module")
def case(sd):
    """The fixture's inputs and the library's results on them: masked (the golden call), all-0 mask (z0), no mask."""
    g = np.load(GOLD)
    d = dict(g=g, image=g["image"], mask=g["mask"], noise=g["noise"], ctx=synth.make_context(2, 7, seed=3),
             unc=synth.make_context(1, 2, seed=99)[0])
    run = lambda **kw: sd.img2img(d["image"], d["ctx"], d["unc"], SCALE, STEPS, kw.pop("strength", STRENGTH),
                                  noise=d["noise"], **kw)
    d["run"] = run
    d["lat"], d["rgb"] = run(mask=d["mask"], latent=True, rgb=True)
    d["z0"] = run(mask=np.zeros_like(d["mask"]), latent=True, rgb=False)
    d["plain"] = run(latent=True, rgb=False)
    return d


def test_golden(case):
    g = case["g"]
    ez = rel(case["z0"], g["z0"])
    e = rel(case["lat"], g["latent"])
    dd = np.abs(case["rgb"][:, ::2, ::2, :].astype(np.int16) - g["u8"].astype(np.int16))
    frac, dmax = float((dd <= 1).mean()), int(dd.max())
    print(f"img2img b2: z0 rel L2 {ez:.3e}, latent rel L2 {e:.3e}, u8 within 1 LSB {frac:.5f}, max {dmax}")
    assert ez < 1e-3  # the encoder bar
    assert e < 2e-3 and frac >= 0.998 and dmax <= 4  # the 2-step bars of test_sample_two_steps_batch2_golden
    assert case["rgb"].shape == (2, 256, 256, 3) and case["rgb"].dtype == np.uint8


def test_conversion_and_final_paste_bit_exact(sd, case):
    x = IO.image_u8_to_float(case["image"])  # numpy float32, the same n (= the same encoder chunking)
    want = SO.scaled_latent(sd.encode_image(x))
    assert np.array_equal(case["z0"], want)
    w = IO.mask_to_latent(case["mask"])
    keep = np.broadcast_to((w == 0)[:, None], case["lat"].shape)
    assert keep.any() and (~keep).any()
    assert np.array_equal(case["lat"][keep], case["z0"][keep])


def test_all_255_mask_is_no_mask(case):
    full = case["run"](mask=np.full_like(case["mask"], 255), latent=True, rgb=False)
    assert np.array_equal(full, case["plain"])
    assert not np.array_equal(case["plain"], case["lat"])


def test_strength_one_is_txt2img(sd, case):
    got = case["run"](strength=1.0, latent=True, rgb=False)
    abar = float(sd.get_tensor("alpha_cumulative_products", (1000,))[999])
    init = SO.start_latent(abar, case["z0"], case["noise"])
    want = sd.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, init_latent=init)
    assert np.array_equal(got, want)


def test_truncation(case):
    a = case["run"](strength=0.5, latent=True, rgb=False)
    b = case["run"](strength=0.74, latent=True, rgb=False)
    assert np.array_equal(a, b) and np.array_equal(a, case["plain"])
    with pytest.raises(_lib.SdbError, match="1/4"):
        case["run"](strength=0.1, latent=True, rgb=False)


def test_step_graph_cache(sd, case):
    """txt2img and img2img of the same shape share the cached step graph; neither may disturb the other."""
    init = synth.make_latent(2, 32, 32, seed=31)
    a1 = sd.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, init_latent=init)
    m1 = case["run"](mask=case["mask"], latent=True, rgb=False)
    a2 = sd.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, init_latent=init)
    m2 = case["run"](mask=case["mask"], latent=True, rgb=False)
    assert np.array_equal(a1, a2)
    assert np.array_equal(m1, m2) and np.array_equal(m1, case["lat"])
    for opt in ("graphs", "emb_hoist"):
        sd.set_option(opt, 0)
        try:
            off = case["run"](mask=case["mask"], latent=True, rgb=False)
        finally:
            sd.set_option(opt, 1)
        assert np.array_equal(off, m1), opt


def test_host_equals_dev(sd, case):
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_img, d_mask, d_ctx, d_unc, d_noise = (t(a) for a in (case["image"], case["mask"], case["ctx"], case["unc"], case["noise"]))
    d_lat = torch.empty((2, 4, 32, 32), dtype=torch.float32, device=dev)
    d_rgb = torch.empty((2, 256, 256, 3), dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    p = lambda x: C.c_void_p(x.data_ptr())
    sd.check(sd.lib.sdb_img2img_dev(sd.h, p(d_img), p(d_mask), STRENGTH, p(d_ctx), 2, 7, p(d_unc), 2, SCALE, STEPS, p(d_noise),
                                    32, 32, p(d_lat), p(d_rgb), C.c_void_p(st)))
    torch.cuda.synchronize()
    assert np.array_equal(d_lat.cpu().numpy(), case["lat"])
    assert np.array_equal(d_rgb.cpu().numpy(), case["rgb"])
    # the device entry needs the noise (the host entry draws it from the seed when it is omitted)
    with pytest.raises(_lib.SdbError):
        sd.check(sd.lib.sdb_img2img_dev(sd.h, p(d_img), None, STRENGTH, p(d_ctx), 2, 7, p(d_unc), 2, SCALE, STEPS, None, 32, 32,
                                        p(d_lat), None, C.c_void_p(st)))


def test_seeded_noise_is_the_txt2img_latent(sd, case):
    """noise = None draws the noise on the device from the seed: the same seed gives the same result, another noise another."""
    a = case["run"](strength=1.0, latent=True, rgb=False)  # explicit noise
    b = sd.img2img(case["image"], case["ctx"], case["unc"], SCALE, STEPS, 1.0, seed=7, latent=True, rgb=False)
    c = sd.img2img(case["image"], case["ctx"], case["unc"], SCALE, STEPS, 1.0, seed=7, latent=True, rgb=False)
    assert np.array_equal(b, c) and not np.array_equal(a, b)


def test_no_extra_launch_per_step(sd, case):
    case["run"](mask=case["mask"], latent=True, rgb=False)  # the step graph of this shape is cached
    n0 = sd.launch_count()
    case["run"](latent=True, rgb=False)
    n1 = sd.launch_count()
    case["run"](mask=case["mask"], latent=True, rgb=False)
    n2 = sd.launch_count()
    assert n2 - n1 == n1 - n0 > 0


def test_errors(sd, case):
    run = case["run"]
    for s in (0.0, 1.5, float("nan")):
        with pytest.raises(_lib.SdbError, match="strength"):
            run(strength=s, latent=True, rgb=False)
    with pytest.raises(_lib.SdbError):
        sd.img2img(case["image"], case["ctx"], case["unc"], SCALE, 2000, 1.0, noise=case["noise"])  # step_by(0)
    unc = case["unc"]
    for px in ((48, 48), (64, 64), (128, 64)):  # 6x6 latent; (H/8)(W/8) = 1, 2: not a multiple of 8
        img = np.zeros((1, *px, 3), np.uint8)
        with pytest.raises(_lib.SdbError):
            sd.img2img(img, case["ctx"][:1], unc, SCALE, STEPS, 0.5)
    img = case["image"]
    u8 = lambda a: a.ctypes.data_as(_lib._u8p)
    with pytest.raises(_lib.SdbError, match="request"):
        sd.check(sd.lib.sdb_img2img(sd.h, u8(img), None, 0.5, _lib.ptr(case["ctx"]), 2, 7, _lib.ptr(unc), 2, SCALE, STEPS, None,
                                    0, 32, 32, None, None))
    # the context is still usable and unchanged
    assert np.array_equal(run(mask=case["mask"], latent=True, rgb=False), case["lat"])


def test_batch_members_independent(sd, case):
    for i in (0, 1):
        one = sd.img2img(case["image"][i:i + 1], case["ctx"][i:i + 1], case["unc"], SCALE, STEPS, STRENGTH,
                         mask=case["mask"][i:i + 1], noise=case["noise"][i:i + 1], latent=True, rgb=False)
        e = rel(one, case["lat"][i:i + 1])
        print(f"img2img batch member {i}: rel L2 {e:.3e}")
        assert e < 1e-3  # not bit-exact: split-K factors change with the batch (test_batch_invariance)
