"""The Karras schedule on the GPU (DESIGN.md §7 f15) through the C ABI: sdb_unet_forward_at against sdb_unet_forward and the oracle,
the schedule_b2 fixture, every sampling entry step-exact against a host loop of sdb_unet_forward_at, the identities (strength 1 =
txt2img, all-255 mask = no mask, Karras != DDIM, defaults restored, the DDIM grid untouched), graphs and emb_hoist off, the launch
count, batches and errors."""
import contextlib
import math
import os

import numpy as np
import pytest
import torch

from oracle import sd_oracle as O
from stable_diffusion_burn_b200 import _lib, pipeline, synth

import img2img_oracle as IO
import inpaint_oracle as NO
import sampler_oracle as SO
import schedule_oracle as KO

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "schedule_b2.npz")
CFG = SO.SAMPLER_CASES
STEPS, SCALE, ETA, NSEED, STRENGTH = CFG["n_steps"], CFG["scale"], CFG["eta"], CFG["noise_seed"], CFG["strength"]
SAMPLERS = {"ddim": (SO.DDIM, 0.0), "eta": (SO.DDIM, ETA), "dpmpp": (SO.DPMPP_2M, 0.0)}
KARRAS = KO.KARRAS
IS = 1.5  # image guidance scale of the edits


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


@contextlib.contextmanager
def sampler(sd, name, schedule="karras", noise_seed=NSEED):
    kind, eta = SAMPLERS[name]
    sd.set_sampler(kind, eta, noise_seed)
    try:
        sd.set_schedule(schedule)
        yield
    finally:
        sd.set_sampler(0, 0.0, 0)  # the session's context is shared with every other GPU test
        sd.set_schedule(0)


@contextlib.contextmanager
def side_context(**kind):
    """A 9- or 8-channel context beside the session's, with a small work arena; synthetic seed 0, so every tensor but conv_in
    equals the session context's."""
    old = os.environ.get("SDB_WORK_GB")
    os.environ["SDB_WORK_GB"] = "8"
    try:
        c = _lib.Context(0, **kind)
    finally:
        if old is None:
            del os.environ["SDB_WORK_GB"]
        else:
            os.environ["SDB_WORK_GB"] = old
    try:
        c.init_synthetic(0)
        c.finalize_weights()
        yield c
    finally:
        c.close()


@pytest.fixture(scope="module")
def sd(ctx):
    ctx.init_synthetic(0)
    ctx.finalize_weights()
    return ctx


@pytest.fixture(scope="module")
def case(sd):
    g = np.load(GOLD)
    image, mask = IO.img2img_inputs()
    d = dict(g=g, noise=g["noise"], image=image, mask=mask, ctx=synth.make_context(2, 7, seed=3),
             unc=synth.make_context(1, 2, seed=99)[0], unc7=synth.make_context(1, 7, seed=99)[0])

    def txt(name, schedule="karras", unc=d["unc"], **kw):
        with sampler(sd, name, schedule, **kw):
            return sd.sample_latent(d["ctx"], unc, SCALE, STEPS, init_latent=d["noise"])

    def i2i(name, strength=STRENGTH, mask=None, schedule="karras", unc=d["unc"]):
        with sampler(sd, name, schedule):
            return sd.img2img(image, d["ctx"], unc, SCALE, STEPS, strength, mask=mask, noise=d["noise"], latent=True, rgb=False)

    d["txt"], d["i2i"] = txt, i2i
    # the DDIM grid's results before any Karras call on this context
    d["ddim_grid"] = {k: txt(k, "ddim") for k in SAMPLERS}
    d["ddim_grid"]["inpaint"] = i2i("dpmpp", mask=mask, schedule="ddim")
    d["res"] = {k: txt(k) for k in SAMPLERS}
    d["res"]["inpaint"] = i2i("dpmpp", mask=mask)
    return d


# ------------------------------------------------------------------------------------------------ sdb_unet_forward_at
def test_unet_forward_at_integer_t_is_unet_forward(sd, case):
    x = synth.make_latent(2, 32, 32, seed=5)
    for t in (0, 1, 500, 687, 999):
        assert np.array_equal(sd.unet_forward_at(x, float(t), case["ctx"]), sd.unet_forward(x, t, case["ctx"])), t
    assert not np.array_equal(sd.unet_forward_at(x, 687.1533, case["ctx"]), sd.unet_forward(x, 687, case["ctx"]))


def test_unet_forward_at_conditioned_contexts(sd, case):
    """The 9- and 8-channel UNets at integer t: sdb_unet_forward_at = sdb_unet_forward bit for bit."""
    for kind, cin in (({"inpaint": True}, 9), ({"pix2pix": True}, 8)):
        with side_context(**kind) as c:
            x = np.concatenate([synth.make_latent(2, 32, 32, seed=5 + j) for j in range(3)], 1)[:, :cin]
            for t in (0, 500, 999):
                assert np.array_equal(c.unet_forward_at(x, float(t), case["ctx"]), c.unet_forward(x, t, case["ctx"])), (cin, t)


def test_unet_forward_at_oracle(sd):
    """At t = 687.1533 (step 1 of the 4-step Karras grid) against the oracle's UNet with the float32 embedding."""
    x = synth.make_latent(1, 32, 32, seed=3)
    ctx = synth.make_context(1, 5, seed=4)
    t = float(KO.grid(sd.get_tensor("alpha_cumulative_products", (1000,)), 4, KARRAS)[0][1])
    assert abs(t - 687.1533) < 1e-4
    out = sd.unet_forward_at(x, t, ctx)
    torch.set_num_threads(os.cpu_count() or 1)
    P = O.Params({n: sd.get_tensor(n, s) for n, s in sd.tensor_list() if n.startswith("unet/")})
    with torch.no_grad():
        ref = KO.unet_forward_at(P, torch.from_numpy(x), t, torch.from_numpy(ctx)).numpy()
    e = rel(out, ref)
    print(f"unet_forward_at t = {t}: rel L2 vs oracle {e:.3e}")
    assert e < 1e-3


# ------------------------------------------------------------------------------------------------ fixture
def test_golden(sd, case):
    """Against the fixture at the bars of test_sampler_gpu.py::test_golden."""
    g = case["g"]
    for name in ("ddim", "eta", "dpmpp", "inpaint"):
        lat = case["res"][name]
        e = rel(lat, g[f"{name}_latent"])
        u8 = sd.latent_to_image(lat)[:, ::2, ::2, :]
        dd = np.abs(u8.astype(np.int16) - g[f"{name}_u8"].astype(np.int16))
        frac, dmax = float((dd <= 1).mean()), int(dd.max())
        print(f"karras {name}: latent rel L2 {e:.3e}, u8 within 1 LSB {frac:.5f}, max {dmax}")
        assert e < 2e-3 and frac >= 0.998 and dmax <= 4, name


# ------------------------------------------------------------------------------------------------ step-exact
def _loop(sd, name, start, guide, first=0, blend=None):
    """step_loop's KERNEL arithmetic on the Karras grid, eta noise from sdb_test_step_noise keyed by the grid index."""
    kind, eta = SAMPLERS[name]
    return KO.step_loop(start, guide, sd.get_tensor("alpha_cumulative_products", (1000,)), STEPS, SO.KERNEL, kind, eta,
                        lambda i, shape: sd.test_step_noise(NSEED, i, math.prod(shape)).reshape(shape), first, blend, KARRAS)


def _two_way(sd, ctx, unc, cond=None):
    """The guidance of one step from ONE sdb_unet_forward_at at batch 2n, (negative | prompt), L = Lu, with the fused step's
    combine fma(c - u, scale, u); cond [n,c,H,W] is appended to the latent's channels (9-channel inpainting)."""
    n = ctx.shape[0]
    ctx2 = np.concatenate([np.repeat(unc[None], n, 0), ctx], 0)

    def guide(x, t):
        xi = x if cond is None else np.concatenate([x, cond], 1)
        e = sd.unet_forward_at(np.concatenate([xi, xi], 0), float(t), ctx2)
        u, c = e[:n], e[n:]
        return SO.fma(np.subtract(c, u), np.float32(SCALE), u)
    return guide


def _z0(sd, image):
    return SO.scaled_latent(sd.encode_image(IO.image_u8_to_float(image)))


@pytest.mark.parametrize("name", list(SAMPLERS))
def test_step_exact_txt2img_and_img2img(sd, case, name):
    unc7 = case["unc7"]
    guide = _two_way(sd, case["ctx"], unc7)
    got = case["txt"](name, unc=unc7)
    want = _loop(sd, name, case["noise"], guide)
    print(f"karras {name}: sample_latent vs host loop of unet_forward_at, rel L2 {rel(got, want):.3e}")
    assert np.array_equal(got, want)
    first = KO.img2img_first(STRENGTH, STEPS)
    _, abars, _ = KO.grid(sd.get_tensor("alpha_cumulative_products", (1000,)), STEPS, KARRAS)
    z0, eps = _z0(sd, case["image"]), case["noise"]
    start = SO.start_latent(abars[first], z0, eps)
    assert np.array_equal(case["i2i"](name, unc=unc7), _loop(sd, name, start, guide, first))
    blend = (IO.mask_to_latent(case["mask"])[:, None], z0, eps)
    assert np.array_equal(case["i2i"](name, mask=case["mask"], unc=unc7), _loop(sd, name, start, guide, first, blend))


def test_step_exact_inpaint_and_edit(sd, case):
    """9-channel inpainting at strength 0.75 and an 8-channel InstructPix2Pix edit, every sampler."""
    unc7, image, mask = case["unc7"], case["image"], case["mask"]
    first = KO.img2img_first(STRENGTH, STEPS)
    with side_context(inpaint=True) as c:
        _, abars, _ = KO.grid(c.get_tensor("alpha_cumulative_products", (1000,)), STEPS, KARRAS)
        z_m = SO.scaled_latent(c.encode_image(NO.masked_image(image, mask)))
        cond = np.concatenate([NO.latent_mask(mask)[:, None], z_m], 1)
        start = SO.start_latent(abars[first], _z0(c, image), case["noise"])
        for name in SAMPLERS:
            with sampler(c, name):
                got = c.img2img(image, case["ctx"], unc7, SCALE, STEPS, STRENGTH, mask=mask, noise=case["noise"], latent=True,
                                rgb=False)
            assert np.array_equal(got, _loop(c, name, start, _two_way(c, case["ctx"], unc7, cond), first)), ("inpaint", name)
    with side_context(pix2pix=True) as c:
        c_i = c.encode_image(IO.image_u8_to_float(image))
        n = c_i.shape[0]
        ctx3 = np.concatenate([np.repeat(unc7[None], 2 * n, 0), case["ctx"]], 0)
        f = np.float32

        def guide(x, t):
            x3 = np.concatenate([np.concatenate([x, np.zeros_like(c_i)], 1), np.concatenate([x, c_i], 1),
                                 np.concatenate([x, c_i], 1)], 0)
            e = c.unet_forward_at(x3, float(t), ctx3)
            u, i, tx = e[:n], e[n:2 * n], e[2 * n:]
            return np.add(np.add(u, np.multiply(f(SCALE), np.subtract(tx, i))), np.multiply(f(IS), np.subtract(i, u)))

        for name in SAMPLERS:
            with sampler(c, name):
                got = c.edit_image(image, case["ctx"], unc7, SCALE, IS, STEPS, init_latent=case["noise"], latent=True, rgb=False)
            assert np.array_equal(got, _loop(c, name, case["noise"], guide)), ("edit", name)


# ------------------------------------------------------------------------------------------------ identities
@pytest.mark.parametrize("name", list(SAMPLERS))
def test_identities(sd, case, name):
    """strength 1 = txt2img from the same start latent; an all-255 mask = no mask; Karras != DDIM."""
    _, abars, _ = KO.grid(sd.get_tensor("alpha_cumulative_products", (1000,)), STEPS, KARRAS)
    init = SO.start_latent(abars[0], _z0(sd, case["image"]), case["noise"])
    got = case["i2i"](name, strength=1.0)
    with sampler(sd, name):
        want = sd.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, init_latent=init)
    assert np.array_equal(got, want)
    plain = case["i2i"](name)
    assert np.array_equal(case["i2i"](name, mask=np.full_like(case["mask"], 255)), plain)
    assert not np.array_equal(plain, case["i2i"](name, mask=case["mask"]))
    assert not np.array_equal(case["res"][name], case["ddim_grid"][name])
    assert not np.array_equal(plain, case["i2i"](name, schedule="ddim"))


def test_ddim_grid_unchanged_by_karras_calls(sd, case):
    """The DDIM grid's results on this context are the same bits before and after Karras calls, and the default is the DDIM
    grid; the pipeline's schedule argument holds for one call."""
    for k in SAMPLERS:
        assert np.array_equal(case["txt"](k, "ddim"), case["ddim_grid"][k]), k
    assert np.array_equal(case["i2i"]("dpmpp", mask=case["mask"], schedule="ddim"), case["ddim_grid"]["inpaint"])
    plain = sd.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, init_latent=case["noise"])
    assert np.array_equal(plain, case["ddim_grid"]["ddim"])
    p = pipeline.StableDiffusion.__new__(pipeline.StableDiffusion)
    p.ctx = sd
    kw = dict(init_latent=case["noise"], height=256, width=256)
    got = p.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, sampler="dpmpp_2m", schedule="karras", **kw)
    assert np.array_equal(got, case["res"]["dpmpp"])
    assert np.array_equal(p.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, **kw), plain)
    out = p.img2img(case["image"], case["ctx"], case["unc"], SCALE, STEPS, STRENGTH, mask=case["mask"], noise=case["noise"],
                    sampler="dpmpp_2m", schedule="karras")
    assert np.array_equal(np.stack(out), sd.latent_to_image(case["res"]["inpaint"]).reshape(2, -1))
    with pytest.raises(ValueError, match="unknown schedule"):
        p.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, schedule="exponential", **kw)
    assert np.array_equal(p.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, **kw), plain)


def test_graphs_and_emb_hoist_off(sd, case):
    for opt in ("graphs", "emb_hoist"):
        sd.set_option(opt, 0)
        try:
            for name in SAMPLERS:
                assert np.array_equal(case["txt"](name), case["res"][name]), (opt, name)
            assert np.array_equal(case["i2i"]("dpmpp", mask=case["mask"]), case["res"]["inpaint"]), opt
            assert np.array_equal(case["txt"]("eta", "ddim"), case["ddim_grid"]["eta"]), opt
        finally:
            sd.set_option(opt, 1)
    # emb_hoist off again after both kinds of per-step graph exist: neither replays the other
    sd.set_option("emb_hoist", 0)
    try:
        for sch in ("ddim", "karras", "ddim"):
            want = case["ddim_grid"]["dpmpp"] if sch == "ddim" else case["res"]["dpmpp"]
            assert np.array_equal(case["txt"]("dpmpp", sch), want), sch
    finally:
        sd.set_option("emb_hoist", 1)


def test_launch_count_matches_the_ddim_grid(sd, case):
    """A Karras call replays the DDIM step graph of its shape: as many launches as a second DDIM call, and no capture."""
    case["txt"]("ddim", "ddim")  # the step graph of this shape is cached
    counts = []
    for sch in ("ddim", "karras", "karras", "ddim"):
        n0 = sd.launch_count()
        case["txt"]("dpmpp", sch)
        counts.append(sd.launch_count() - n0)
    print("launches per call (ddim, karras, karras, ddim):", counts)
    assert len(set(counts)) == 1


# ------------------------------------------------------------------------------------------------ batches
@pytest.mark.parametrize("name", list(SAMPLERS))
def test_batches(sd, case, name):
    """A uniform batch is the single call; at n = 1 a seeded batch call is the seeded single call."""
    ctx, unc, noise = case["ctx"], case["unc"], case["noise"]
    rows = [ctx[0], ctx[1]]
    with sampler(sd, name):
        lat = sd.sample_batch(rows, unc, SCALE, STEPS, init_latent=noise, H=32, W=32, latent=True, rgb=False,
                              noise_seeds=[NSEED, NSEED])
        got_i2i = sd.img2img_batch(case["image"], rows, [unc, unc], [SCALE, SCALE], STEPS, STRENGTH, mask=case["mask"], noise=noise,
                                   latent=True, rgb=False)
    if name != "eta":  # at n > 1 the batch keys eta noise per sample, the single call over the flat latent
        assert np.array_equal(lat, case["res"][name])
        assert np.array_equal(got_i2i, case["i2i"](name, mask=case["mask"]))
    s, q = 2 ** 35 + 17, 29
    with sampler(sd, name, noise_seed=q):
        want = sd.sample_latent(ctx[:1], unc, SCALE, STEPS, seed=s, H=32, W=32)
    with sampler(sd, name):
        got = sd.sample_batch([ctx[0]], unc, SCALE, STEPS, seeds=[s], noise_seeds=[q], H=32, W=32, latent=True, rgb=False)
    assert np.array_equal(got, want)


# ------------------------------------------------------------------------------------------------ errors
def test_errors_leave_the_context_usable(sd, case):
    for kind in (2, -1, 7):
        with pytest.raises(_lib.SdbError, match=f"unknown kind {kind}"):
            sd.set_schedule(kind)
    assert np.array_equal(sd.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, init_latent=case["noise"]),
                          case["ddim_grid"]["ddim"])
    with sampler(sd, "dpmpp"):
        with pytest.raises(_lib.SdbError):
            sd.set_schedule(3)
        assert np.array_equal(case["txt"]("dpmpp"), case["res"]["dpmpp"])  # still Karras
    x = synth.make_latent(1, 32, 32, seed=5)
    for t in (-0.5, 999.5, float("nan"), float("inf")):
        with pytest.raises(_lib.SdbError, match="unet_forward_at"):
            sd.unet_forward_at(x, t, case["ctx"][:1])
    # a schedule the Karras grid cannot take: the call fails before anything is staged, naming the first bad index; the DDIM grid
    # still runs on it
    good = sd.get_tensor("alpha_cumulative_products", (1000,))
    bad = good.copy()
    bad[300] = bad[299]
    try:
        sd.set_tensor("alpha_cumulative_products", bad)
        sd.finalize_weights()
        with pytest.raises(_lib.SdbError, match=r"alpha_cumulative_products\[300\]"):
            case["txt"]("ddim")
        with pytest.raises(_lib.SdbError, match=r"alpha_cumulative_products\[300\]"):
            case["i2i"]("dpmpp", mask=case["mask"])
        assert np.isfinite(case["txt"]("ddim", "ddim")).all()
    finally:
        sd.set_tensor("alpha_cumulative_products", good)
        sd.finalize_weights()
    assert np.array_equal(case["txt"]("dpmpp"), case["res"]["dpmpp"])
    assert np.array_equal(case["txt"]("ddim", "ddim"), case["ddim_grid"]["ddim"])
