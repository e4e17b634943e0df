"""The samplers on the GPU (DESIGN.md §7 f6) through the C ABI: the sampler_b2 fixture, the sampler arithmetic isolated from the
UNet (a host loop of sdb_forward_diffuser), the bit-exact identities (default = DDIM eta 0, img2img at strength 1 = txt2img,
all-255 mask = no mask, seeded noise), the step-graph cache, host / device entries, launch counts, the noise stream and errors."""
import contextlib
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from stable_diffusion_burn_b200 import _lib, pipeline, synth

import sampler_oracle as SO

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sampler_b2.npz")
CFG = SO.SAMPLER_CASES
STEPS, SCALE, ETA, NSEED, STRENGTH = CFG["n_steps"], CFG["scale"], CFG["eta"], CFG["noise_seed"], CFG["strength"]
SAMPLERS = {"ddim": (SO.DDIM, 0.0), "eta": (SO.DDIM, ETA), "dpmpp": (SO.DPMPP_2M, 0.0)}


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


@contextlib.contextmanager
def sampler(sd, kind, eta=0.0, noise_seed=NSEED):
    sd.set_sampler(kind, eta, noise_seed)
    try:
        yield
    finally:
        sd.set_sampler(0, 0.0, 0)  # the session's context is shared with every other GPU test


@pytest.fixture(scope="module")
def sd(ctx):
    ctx.init_synthetic(0)
    ctx.finalize_weights()
    return ctx


@pytest.fixture(scope="module")
def case(sd):
    from img2img_oracle import img2img_inputs
    g = np.load(GOLD)
    image, mask = img2img_inputs()
    d = dict(g=g, noise=g["noise"], image=image, mask=mask, ctx=synth.make_context(2, 7, seed=3),
             unc=synth.make_context(1, 2, seed=99)[0])

    def txt(name, **kw):
        with sampler(sd, *SAMPLERS[name], **kw):
            return sd.sample_latent(d["ctx"], d["unc"], SCALE, STEPS, init_latent=d["noise"])

    def i2i(name, strength=STRENGTH, mask=None, **kw):
        with sampler(sd, *SAMPLERS[name], **kw):
            return sd.img2img(image, d["ctx"], d["unc"], SCALE, STEPS, strength, mask=mask, noise=d["noise"], latent=True, rgb=False)

    d["txt"], d["i2i"] = txt, i2i
    d["res"] = {k: txt(k) for k in SAMPLERS}
    d["res"]["inpaint"] = i2i("dpmpp", mask=mask)
    return d


def test_golden(sd, case):
    """Against the fixture at the bars of test_sample_two_steps_batch2_golden (free-running oracle, all 4 / 3 steps)."""
    g = case["g"]
    for name, key in (("dpmpp", "dpmpp"), ("eta", "eta"), ("inpaint", "inpaint")):
        lat = case["res"][name]
        e = rel(lat, g[f"{key}_latent"])
        u8 = sd.latent_to_image(lat)[:, ::2, ::2, :]
        dd = np.abs(u8.astype(np.int16) - g[f"{key}_u8"].astype(np.int16))
        frac, dmax = float((dd <= 1).mean()), int(dd.max())
        print(f"sampler {name}: latent rel L2 {e:.3e}, u8 within 1 LSB {frac:.5f}, max {dmax}")
        assert e < 2e-3 and frac >= 0.998 and dmax <= 4, name


def _host_loop(sd, case, kind, eta):
    """sample_latent restated on the host around sdb_forward_diffuser: the two UNet outputs of each step from the library, the
    guidance combine as the fused step's SASS computes it (pred = fma(c - u, scale, u)), then the oracle's step_loop with its
    KERNEL arithmetic (x0 = fma(-pred, sqrt(1 - a_t), x) / sqrt(a_t), the eta = 0 update fma(pred, sqrt(1 - a'),
    fl(x0 sqrt(a')))), the new updates from the oracle (numpy float32, no contraction, as the kernel's __f*_rn) and eta's noise
    from sdb_test_step_noise. So only the sampler arithmetic is compared."""
    def guide(x, t):
        _, u, c = sd.forward_diffuser(x, t, case["ctx"], case["unc"], SCALE)
        return SO.fma(np.subtract(c, u), np.float32(SCALE), u)

    return SO.step_loop(case["noise"], guide, sd.get_tensor("alpha_cumulative_products", (1000,)), STEPS, SO.KERNEL, kind, eta,
                        lambda t, shape: sd.test_step_noise(NSEED, t, math.prod(shape)).reshape(shape))


@pytest.mark.parametrize("name", list(SAMPLERS))
def test_step_exact(sd, case, name):
    """The library against its own UNet outputs and the oracle's update, 4 steps: the UNet pass of sdb_forward_diffuser and the
    cached step graph's are bit-identical, and so is the sampler arithmetic once the fused step's contractions are restated."""
    want = _host_loop(sd, case, *SAMPLERS[name])
    print(f"sampler {name}: sample_latent vs host loop of forward_diffuser + oracle update, rel L2 "
          f"{rel(case['res'][name], want):.3e}")
    assert np.array_equal(case["res"][name], want)


def test_default_is_ddim_eta0(sd, case):
    plain = sd.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, init_latent=case["noise"])
    assert np.array_equal(plain, case["res"]["ddim"])
    for s in (0, 5, 2 ** 40):
        with sampler(sd, 0, 0.0, s):
            assert np.array_equal(sd.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, init_latent=case["noise"]), plain)
    assert not np.array_equal(plain, case["res"]["dpmpp"]) and not np.array_equal(plain, case["res"]["eta"])


@pytest.mark.parametrize("name", list(SAMPLERS))
def test_img2img_identities(sd, case, name):
    """strength 1 = txt2img from the same start latent; an all-255 mask = no mask; for every sampler."""
    abar = float(sd.get_tensor("alpha_cumulative_products", (1000,))[999])
    from img2img_oracle import image_u8_to_float
    init = SO.start_latent(abar, SO.scaled_latent(sd.encode_image(image_u8_to_float(case["image"]))), case["noise"])
    got = case["i2i"](name, strength=1.0)
    with sampler(sd, *SAMPLERS[name]):
        want = sd.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, init_latent=init)
    assert np.array_equal(got, want)
    plain = case["i2i"](name)
    full = case["i2i"](name, mask=np.full_like(case["mask"], 255))
    assert np.array_equal(full, plain)
    assert not np.array_equal(plain, case["i2i"](name, mask=case["mask"]))


def test_noise_seed(sd, case):
    a = case["txt"]("eta", noise_seed=NSEED)
    b = case["txt"]("eta", noise_seed=NSEED + 1)
    assert np.array_equal(a, case["res"]["eta"]) and not np.array_equal(a, b)
    # DPM++ draws no noise: the seed does not matter
    assert np.array_equal(case["txt"]("dpmpp", noise_seed=123), case["res"]["dpmpp"])


def test_step_graph_cache_and_options(sd, case):
    """Samplers alternating on one shape reuse the cached step graph and reproduce each result; graphs / emb_hoist off agree."""
    for name in ("ddim", "dpmpp", "eta", "ddim", "dpmpp"):
        assert np.array_equal(case["txt"](name), case["res"][name]), name
    assert np.array_equal(case["i2i"]("dpmpp", mask=case["mask"]), case["res"]["inpaint"])
    for opt in ("graphs", "emb_hoist"):
        sd.set_option(opt, 0)
        try:
            for name in SAMPLERS:
                assert np.array_equal(case["txt"](name), case["res"][name]), (opt, name)
            assert np.array_equal(case["i2i"]("dpmpp", mask=case["mask"]), case["res"]["inpaint"]), opt
        finally:
            sd.set_option(opt, 1)


def test_host_equals_dev(sd, case):
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_ctx, d_unc, d_noise, d_img, d_mask = (t(a) for a in (case["ctx"], case["unc"], case["noise"], case["image"], case["mask"]))
    d_rgb = torch.empty((2, 256, 256, 3), dtype=torch.uint8, device=dev)
    d_lat = torch.empty((2, 4, 32, 32), dtype=torch.float32, device=dev)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda x: C.c_void_p(x.data_ptr())
    for name in ("eta", "dpmpp"):
        with sampler(sd, *SAMPLERS[name]):
            host = sd.sample_image(case["ctx"], case["unc"], SCALE, STEPS, init_latent=case["noise"])
            sd.check(sd.lib.sdb_sample_image_dev(sd.h, p(d_ctx), 2, 7, p(d_unc), 2, SCALE, STEPS, p(d_noise), 32, 32, p(d_rgb), st))
            torch.cuda.synchronize()
            assert np.array_equal(d_rgb.cpu().numpy(), host), name
            assert np.array_equal(host, sd.latent_to_image(case["res"][name])), name
            sd.check(sd.lib.sdb_img2img_dev(sd.h, p(d_img), p(d_mask), STRENGTH, p(d_ctx), 2, 7, p(d_unc), 2, SCALE, STEPS,
                                            p(d_noise), 32, 32, p(d_lat), None, st))
            torch.cuda.synchronize()
            host_i2i = sd.img2img(case["image"], case["ctx"], case["unc"], SCALE, STEPS, STRENGTH, mask=case["mask"],
                                  noise=case["noise"], latent=True, rgb=False)
            assert np.array_equal(d_lat.cpu().numpy(), host_i2i), name
    assert np.array_equal(host_i2i, case["res"]["inpaint"])


def test_launch_count_is_the_same_for_every_sampler(sd, case):
    case["txt"]("ddim")  # the step graph of this shape is cached
    counts = {}
    for name in ("ddim", "eta", "dpmpp", "ddim"):
        n0 = sd.launch_count()
        case["txt"](name)
        counts.setdefault(name, []).append(sd.launch_count() - n0)
    print("launches per call:", counts)
    assert len({c for v in counts.values() for c in v}) == 1


def test_step_noise_matches_the_numpy_mirror(sd):
    for seed, t, n in ((0, 999, 4096), (NSEED, 249, 2 * 4 * 32 * 32), (2 ** 40 + 3, 0, 1 << 18)):
        got = sd.test_step_noise(seed, t, n)
        want = synth.step_noise(seed, t, (n,))
        d = float(np.abs(got - want).max())
        print(f"step noise seed {seed} t {t}: max |device - numpy| {d:.2e}")
        assert d <= 1e-5
    assert not np.array_equal(sd.test_step_noise(1, 999, 4096), sd.test_step_noise(2, 999, 4096))


def test_errors_leave_the_context_usable(sd, case):
    for kind, eta, what in ((0, 1.5, "eta"), (0, -0.1, "eta"), (0, float("nan"), "eta"), (1, 0.5, "deterministic"),
                            (2, 0.0, "unknown kind 2"), (-1, 0.0, "unknown kind -1")):
        with pytest.raises(_lib.SdbError, match=what):
            sd.set_sampler(kind, eta, 0)
    with pytest.raises(_lib.SdbError):
        sd.check(sd.lib.sdb_test_step_noise(sd.h, 0, 1000, 16, _lib.ptr(np.empty(16, np.float32))))
    # the failed calls changed nothing: still the default sampler
    assert np.array_equal(sd.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, init_latent=case["noise"]), case["res"]["ddim"])
    with sampler(sd, *SAMPLERS["dpmpp"]):
        with pytest.raises(_lib.SdbError):
            sd.set_sampler(1, 0.25, 0)
        assert np.array_equal(sd.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, init_latent=case["noise"]),
                              case["res"]["dpmpp"])


def test_pipeline_arguments(sd, case):
    """StableDiffusion's sampler / eta / noise_seed hold for the one call; the default sampler is restored after it."""
    p = pipeline.StableDiffusion.__new__(pipeline.StableDiffusion)
    p.ctx = sd  # the session's context (a second one would hold another copy of the weights)
    kw = dict(init_latent=case["noise"], height=256, width=256)
    got = p.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, sampler="ddim", eta=ETA, noise_seed=NSEED, **kw)
    assert np.array_equal(got, case["res"]["eta"])
    assert np.array_equal(p.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, **kw), case["res"]["ddim"])
    rgb = p.sample_image(case["ctx"], case["unc"], SCALE, STEPS, sampler="dpmpp_2m", **kw)
    assert np.array_equal(np.stack(rgb), sd.latent_to_image(case["res"]["dpmpp"]).reshape(2, -1))
    with pytest.raises(_lib.SdbError):
        p.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, sampler="dpmpp_2m", eta=0.5, **kw)
    out = p.img2img(case["image"], case["ctx"], case["unc"], SCALE, STEPS, STRENGTH, mask=case["mask"], noise=case["noise"],
                    sampler="dpmpp_2m")
    assert np.array_equal(np.stack(out), sd.latent_to_image(case["res"]["inpaint"]).reshape(2, -1))
    assert np.array_equal(p.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, **kw), case["res"]["ddim"])
