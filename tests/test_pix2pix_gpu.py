"""InstructPix2Pix editing with an 8-channel UNet on the GPU (DESIGN.md §7 f10) through the C ABI: the registry of
sdb_create_pix2pix, the pix2pix_b2 fixture, the step-exact three-way guidance against a host loop of sdb_unet_forward, the
zero-weight identity with the 4-channel model, the unscaled image latent, the step-graph cache, host / device entries, launch
counts and errors across 4-, 8- and 9-channel contexts."""
import contextlib
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from stable_diffusion_burn_b200 import _lib, dumpdir, pipeline, synth, topology

import img2img_oracle as IO
import pix2pix_oracle as PO
import sampler_oracle as SO

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pix2pix_b2.npz")
STEPS, TS, IS, NSEED, ETA = PO.PIX2PIX["n_steps"], PO.PIX2PIX["text_scale"], PO.PIX2PIX["image_scale"], 11, 0.7
SAMPLERS = {"ddim": (SO.DDIM, 0.0), "eta": (SO.DDIM, ETA), "dpmpp": (SO.DPMPP_2M, 0.0)}
CONV_IN = "unet/input_blocks/conv/weight"


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


@contextlib.contextmanager
def sampler(sd, name):
    kind, eta = SAMPLERS[name]
    sd.set_sampler(kind, eta, NSEED)
    try:
        yield
    finally:
        sd.set_sampler(0, 0.0, 0)


@contextlib.contextmanager
def work_gb(gb):
    """A small work arena for a context beside the session's: the default one of each would take most of the card."""
    old = os.environ.get("SDB_WORK_GB")
    os.environ["SDB_WORK_GB"] = str(gb)
    try:
        yield
    finally:
        if old is None:
            del os.environ["SDB_WORK_GB"]
        else:
            os.environ["SDB_WORK_GB"] = old


@pytest.fixture(scope="module")
def sd4(ctx):
    ctx.init_synthetic(0)
    ctx.finalize_weights()
    return ctx


@pytest.fixture(scope="module")
def sd8(sd4):
    """A second context, 8-channel. Synthetic seed 0, so every tensor but conv_in equals the session context's."""
    with work_gb(8):
        c = _lib.Context(0, pix2pix=True)
    c.init_synthetic(0)
    c.finalize_weights()
    yield c
    c.close()


@pytest.fixture(scope="module")
def case(sd8):
    g = np.load(GOLD)
    d = dict(g=g, image=g["image"], latent0=g["latent0"], ctx=synth.make_context(2, 7, seed=3),
             unc=synth.make_context(1, 2, seed=99)[0])

    def run(sd, name="ddim", image=d["image"], latent0=d["latent0"], ctx=d["ctx"], unc=d["unc"], s_i=IS, n_steps=STEPS):
        with sampler(sd, name):
            return sd.edit_image(image, ctx, unc, TS, s_i, n_steps, init_latent=latent0, latent=True, rgb=False)

    d["run"] = run
    d["lat"] = run(sd8)
    return d


def test_registry_is_the_pix2pix_topology(sd8, sd4):
    got = sd8.tensor_list()
    want = [(n, tuple(s)) for (n, s, _, _) in topology.all_params(pix2pix=True)] + [("alpha_cumulative_products", (1000,))]
    assert got == want
    assert sd8.unet_in_channels() == 8 and sd4.unet_in_channels() == 4
    four = sd4.tensor_list()
    assert [n for n, _ in four] == [n for n, _ in got]
    assert [i for i, (a, b) in enumerate(zip(four, got)) if a != b] == [[n for n, _ in got].index(CONV_IN)]


def test_golden(sd8, case):
    g = case["g"]
    for name, c in PO.PIX2PIX_CASES.items():
        smp = "dpmpp" if c["kind"] == SO.DPMPP_2M else "ddim"
        with sampler(sd8, smp):
            lat, rgb = sd8.edit_image(case["image"], case["ctx"], case["unc"], TS, IS, STEPS, init_latent=case["latent0"],
                                      latent=True, rgb=True)
        e = rel(lat, g[f"latent_{name}"])
        dd = np.abs(rgb[:, ::2, ::2, :].astype(np.int16) - g[f"u8_{name}"].astype(np.int16))
        frac, dmax = float((dd <= 1).mean()), int(dd.max())
        print(f"pix2pix {name}: latent rel L2 {e:.3e}, u8 within 1 LSB {frac:.5f}, max {dmax}")
        assert e < 2e-3 and frac >= 0.998 and dmax <= 4, name


def _host_loop(sd, case, name, unc, c_i=None):
    """sdb_edit_image restated on the host: c_I from sdb_encode_image (unscaled), each step's three UNet outputs from ONE
    sdb_unet_forward at batch 3n on [3n,8,H,W] = (x | 0), (x | c_I), (x | c_I) under (negative, negative, prompt) — the call's
    group order — then the kernel's combine and update in float32 (tests/test_inpaint_gpu.py: _host_loop)."""
    kind, eta = SAMPLERS[name]
    f = np.float32
    if c_i is None:
        c_i = sd.encode_image(IO.image_u8_to_float(case["image"]))
    n = c_i.shape[0]
    ctx3 = np.concatenate([np.repeat(unc[None], 2 * n, 0), case["ctx"]], 0)

    def guide(x, t):
        x3 = np.concatenate([np.concatenate([x, np.zeros_like(c_i)], 1), np.concatenate([x, c_i], 1),
                             np.concatenate([x, c_i], 1)], 0)
        e = sd.unet_forward(x3, t, ctx3)
        u, i, tx = e[:n], e[n:2 * n], e[2 * n:]
        return np.add(np.add(u, np.multiply(f(TS), np.subtract(tx, i))), np.multiply(f(IS), np.subtract(i, u)))

    return SO.step_loop(case["latent0"], guide, sd.get_tensor("alpha_cumulative_products", (1000,)), STEPS, SO.KERNEL, kind, eta,
                        lambda t, shape: sd.test_step_noise(NSEED, t, math.prod(shape)).reshape(shape))


@pytest.mark.parametrize("name", list(SAMPLERS))
def test_step_exact_three_way_guidance(sd8, case, name):
    unc7 = synth.make_context(1, 7, seed=99)[0]  # L = Lu: sdb_unet_forward takes one length
    got = case["run"](sd8, name, unc=unc7)
    want = _host_loop(sd8, case, name, unc7)
    print(f"pix2pix {name}: sdb_edit_image vs host loop of unet_forward, rel L2 {rel(got, want):.3e}")
    assert np.array_equal(got, want)


def test_image_latent_is_unscaled(sd8, case):
    """The call conditions on encode_image(x) itself: the host loop on that input equals the call, on 0.18215 of it not."""
    unc7 = synth.make_context(1, 7, seed=99)[0]
    got = case["run"](sd8, unc=unc7)
    c_i = sd8.encode_image(IO.image_u8_to_float(case["image"]))
    print(f"c_I rel to the fixture's {rel(c_i, case['g']['c_I']):.3e}")
    assert rel(c_i, case["g"]["c_I"]) < 1e-3
    assert np.array_equal(got, _host_loop(sd8, case, "ddim", unc7, c_i))
    scaled = _host_loop(sd8, case, "ddim", unc7, SO.scaled_latent(c_i))
    print(f"pix2pix: result with a scaled image latent differs by rel L2 {rel(scaled, got):.3e}")
    assert rel(scaled, got) > 1e-3


@pytest.fixture
def zero_ext(sd8, sd4):
    """conv_in of the 8-channel context = the session context's conv_in, extended by zero weights on channels 4-7."""
    keep = sd8.get_tensor(CONV_IN, (320, 8, 3, 3))
    sd8.set_tensor(CONV_IN, PO.zero_extension(sd4.get_tensor(CONV_IN, (320, 4, 3, 3))))
    sd8.finalize_weights()
    yield
    sd8.set_tensor(CONV_IN, keep)
    sd8.finalize_weights()


@pytest.mark.parametrize("name", ["ddim", "dpmpp"])
def test_zero_weight_identity(sd8, sd4, case, zero_ext, name):
    x = case["latent0"]
    c_i = sd8.encode_image(IO.image_u8_to_float(case["image"]))
    unc2 = np.repeat(case["unc"][None], 2, 0)
    e = sd8.unet_forward(np.concatenate([np.concatenate([x, c_i], 1), np.concatenate([x, np.zeros_like(c_i)], 1)], 0), 500,
                         np.concatenate([unc2, unc2], 0))
    assert np.array_equal(e[:2], e[2:])  # e_I == e_U
    assert np.array_equal(sd8.unet_forward(np.concatenate([x, c_i], 1), 500, case["ctx"]), sd4.unet_forward(x, 500, case["ctx"]))
    got = case["run"](sd8, name, s_i=2.5)
    with sampler(sd4, name):
        want = sd4.sample_latent(case["ctx"], case["unc"], TS, STEPS, init_latent=x)
    print(f"pix2pix {name}: zero-weight edit vs 4-channel txt2img, rel L2 {rel(got, want):.3e}")
    assert rel(got, want) < 1e-3


def test_step_graph_cache(sd8, sd4, case):
    """Two latent sizes in turn make the conditioning slot regrow (and move); the first size again must still be right. A
    text-to-image call on the 4-channel context between edits leaves both contexts' cached graphs right."""
    img64 = np.ascontiguousarray(np.tile(case["image"][:1], (1, 2, 2, 1)))
    l64 = synth.make_latent(1, 64, 64, seed=12)
    big = case["run"](sd8, image=img64, latent0=l64, ctx=case["ctx"][:1])
    assert np.array_equal(case["run"](sd8), case["lat"])
    sd8.set_option("graphs", 0)
    try:
        off = case["run"](sd8)
        big_off = case["run"](sd8, image=img64, latent0=l64, ctx=case["ctx"][:1])
    finally:
        sd8.set_option("graphs", 1)
    assert np.array_equal(off, case["lat"]) and np.array_equal(big_off, big)
    sd8.set_option("emb_hoist", 0)
    try:
        assert np.array_equal(case["run"](sd8), case["lat"])
    finally:
        sd8.set_option("emb_hoist", 1)
    t2i = lambda: sd4.sample_latent(case["ctx"], case["unc"], TS, STEPS, init_latent=case["latent0"])
    first = t2i()
    assert np.array_equal(case["run"](sd8), case["lat"])
    assert np.array_equal(t2i(), first)
    assert np.array_equal(case["run"](sd8), case["lat"])


def test_host_equals_dev(sd8, case):
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_img, d_ctx, d_unc, d_l0 = (t(a) for a in (case["image"], case["ctx"], case["unc"], case["latent0"]))
    d_lat = torch.empty((2, 4, 32, 32), dtype=torch.float32, device=dev)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda x: C.c_void_p(x.data_ptr())
    sd8.check(sd8.lib.sdb_edit_image_dev(sd8.h, p(d_img), p(d_ctx), 2, 7, p(d_unc), 2, TS, IS, STEPS, p(d_l0), 32, 32, p(d_lat),
                                         None, st))
    torch.cuda.synchronize()
    assert np.array_equal(d_lat.cpu().numpy(), case["lat"])
    x8 = np.concatenate([case["latent0"], synth.make_latent(2, 32, 32, seed=7)], 1)
    d_x, d_out = t(x8), torch.empty((2, 4, 32, 32), dtype=torch.float32, device=dev)
    sd8.check(sd8.lib.sdb_unet_forward_dev(sd8.h, p(d_x), 500, p(d_ctx), 2, 32, 32, 7, p(d_out), st))
    torch.cuda.synchronize()
    assert np.array_equal(d_out.cpu().numpy(), sd8.unet_forward(x8, 500, case["ctx"]))
    # the pipeline call returns the decoded image of the same edit; NULL init latent = sample_image's seeded stream
    sd = object.__new__(pipeline.StableDiffusion)
    sd.ctx = sd8
    imgs = sd.edit_image(case["image"], case["ctx"], case["unc"], TS, IS, STEPS, init_latent=case["latent0"])
    rgb = sd8.edit_image(case["image"], case["ctx"], case["unc"], TS, IS, STEPS, init_latent=case["latent0"])
    assert len(imgs) == 2 and all(np.array_equal(imgs[i], rgb[i].reshape(-1)) for i in range(2))
    seeded = sd8.edit_image(case["image"][:1], case["ctx"][:1], case["unc"], TS, IS, STEPS, seed=5, latent=True, rgb=False)
    with_init = case["run"](sd8, image=case["image"][:1], latent0=synth.seeded_latents([5], 32, 32), ctx=case["ctx"][:1])
    print(f"pix2pix: NULL init latent vs its host restatement (a few ulp apart), rel L2 {rel(seeded, with_init):.3e}")
    assert rel(seeded, with_init) < 1e-3


def test_launch_counts(sd8, sd4, case):
    """Per step: as many launches as text-to-image (one UNet pass, one fused guidance + update). Per call: the image staging
    and one encoder pass more."""
    def edit(k):
        return sd8.edit_image(case["image"], case["ctx"], case["unc"], TS, IS, k, init_latent=case["latent0"], latent=True,
                              rgb=False)

    def t2i(k):
        return sd4.sample_latent(case["ctx"], case["unc"], TS, k, init_latent=case["latent0"])

    def launches(sd, fn, k):
        fn(k)  # the step graph of this shape is cached
        n0 = sd.launch_count()
        fn(k)
        return sd.launch_count() - n0

    c8 = {k: launches(sd8, edit, k) for k in (2, 4)}
    c4 = {k: launches(sd4, t2i, k) for k in (2, 4)}
    n0 = sd4.launch_count()
    sd4.encode_image(IO.image_u8_to_float(case["image"]))
    enc = sd4.launch_count() - n0
    print(f"launches per call at 4 steps: edit {c8[4]}, txt2img {c4[4]}, encoder pass {enc}; per step {(c8[4] - c8[2]) // 2}")
    assert c8[4] - c8[2] == c4[4] - c4[2] > 0
    assert c8[4] - c4[4] == 1 + enc


def _conv_tree(root, cin):
    """The smallest dump-dir that reaches the conv_in check: the schedule length and a [320,cin,3,3] conv_in."""
    os.makedirs(os.path.join(root, "unet/input_blocks/conv"), exist_ok=True)
    dumpdir.save_scalar(1000, "n_steps", root)
    dumpdir.save_tensor(np.zeros((320, cin, 3, 3), np.float32), "weight", os.path.join(root, "unet/input_blocks/conv"))
    return root


def test_errors(sd8, sd4, case, tmp_path):
    u8, ptr, f32 = (lambda a: a.ctypes.data_as(_lib._u8p)), _lib.ptr, np.float32
    img, ctx, unc, l0 = case["image"], case["ctx"], case["unc"], case["latent0"]
    mask = np.full(img.shape[:3], 255, np.uint8)
    lat = np.empty((2, 4, 32, 32), f32)
    # every sampling entry but sdb_edit_image refuses the 8-channel context and names it
    edit = "sdb_edit_image"
    calls = {
        "sample_latent": lambda: sd8.sample_latent(ctx, unc, TS, STEPS, init_latent=l0),
        "sample_image": lambda: sd8.sample_image(ctx, unc, TS, STEPS, seed=1, H=32, W=32),
        "sample_image_dev": lambda: sd8.check(sd8.lib.sdb_sample_image_dev(sd8.h, None, 2, 7, None, 2, TS, STEPS, None, 32, 32,
                                                                          None, None)),
        "img2img": lambda: sd8.img2img(img, ctx, unc, TS, STEPS, 1.0, noise=l0),
        "img2img masked": lambda: sd8.img2img(img, ctx, unc, TS, STEPS, 1.0, mask=mask, noise=l0),
        "img2img_dev": lambda: sd8.check(sd8.lib.sdb_img2img_dev(sd8.h, None, None, 1.0, None, 2, 7, None, 2, TS, STEPS, None, 32,
                                                                 32, None, None, None)),
        "sample_batch": lambda: sd8.sample_batch(list(ctx[:, None]), unc, TS, STEPS, seeds=[1, 2], H=32, W=32),
        "img2img_batch": lambda: sd8.img2img_batch(img, list(ctx[:, None]), unc, TS, STEPS, 1.0, noise=l0),
        "forward_diffuser": lambda: sd8.forward_diffuser(np.concatenate([l0, l0], 1), 500, ctx, unc, TS),
        "forward_diffuser_dev": lambda: sd8.check(sd8.lib.sdb_forward_diffuser_dev(sd8.h, None, 500, None, 2, 7, None, 2, TS, 32,
                                                                                   32, None, None)),
    }
    for what, call in calls.items():
        with pytest.raises(_lib.SdbError, match=edit):
            call()
        print(f"{what}: refused")
    with work_gb(2):
        sd9 = _lib.Context(0, inpaint=True)
    try:
        sd9.init_synthetic(0)
        sd9.finalize_weights()
        # sdb_edit_image refuses the 4- and 9-channel contexts and names sdb_create_pix2pix
        for sd in (sd4, sd9):
            with pytest.raises(_lib.SdbError, match="sdb_create_pix2pix"):
                sd.edit_image(img, ctx, unc, TS, IS, STEPS, init_latent=l0)
            with pytest.raises(_lib.SdbError, match="sdb_create_pix2pix"):
                sd.check(sd.lib.sdb_edit_image_dev(sd.h, None, None, 2, 7, None, 2, TS, IS, STEPS, None, 32, 32, None, None, None))
        # a conv_in of the wrong width, between all three widths, names both shapes and the right create entry
        w = {c: np.zeros((320, c, 3, 3), f32) for c in (4, 8, 9)}
        entry = {4: r"sdb_create\b", 8: "sdb_create_pix2pix", 9: "sdb_create_inpaint"}
        for sd, cin in ((sd4, 4), (sd8, 8), (sd9, 9)):
            for other in (4, 8, 9):
                if other == cin:
                    continue
                pat = rf"\[320,{other},3,3\].*\[320,{cin},3,3\].*{entry[other]}"
                with pytest.raises(_lib.SdbError, match=pat):
                    sd.set_tensor(CONV_IN, w[other])
                with pytest.raises(_lib.SdbError, match=pat):
                    sd.load_dump_dir(_conv_tree(str(tmp_path / f"c{cin}_{other}"), other))
        assert np.isfinite(sd9.unet_forward(synth.make_latent(1, 32, 32, seed=5).repeat(3, 1)[:, :9], 500, ctx[:1])).all()
    finally:
        sd9.close()
    # argument rules of the edit entries
    for bad in (float("nan"), float("inf")):
        with pytest.raises(_lib.SdbError, match=r"text_scale = (nan|inf)"):
            sd8.edit_image(img, ctx, unc, bad, IS, STEPS, init_latent=l0)
        with pytest.raises(_lib.SdbError, match=r"image_scale = (nan|inf)"):
            sd8.edit_image(img, ctx, unc, TS, bad, STEPS, init_latent=l0)
    with pytest.raises(_lib.SdbError, match="latent, the image or both"):
        sd8.check(sd8.lib.sdb_edit_image(sd8.h, u8(img), ptr(ctx), 2, 7, ptr(unc), 2, TS, IS, STEPS, ptr(l0), 0, 32, 32, None, None))
    with pytest.raises(_lib.SdbError, match="null image"):
        sd8.check(sd8.lib.sdb_edit_image(sd8.h, None, ptr(ctx), 2, 7, ptr(unc), 2, TS, IS, STEPS, ptr(l0), 0, 32, 32, ptr(lat), None))
    with pytest.raises(_lib.SdbError, match="n_steps"):
        sd8.edit_image(img, ctx, unc, TS, IS, 0, init_latent=l0)
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_img, d_ctx, d_unc, d_lat = t(img), t(ctx), t(unc), torch.empty((2, 4, 32, 32), dtype=torch.float32, device=dev)
    p = lambda x: C.c_void_p(x.data_ptr())
    with pytest.raises(_lib.SdbError, match="start latent"):
        sd8.check(sd8.lib.sdb_edit_image_dev(sd8.h, p(d_img), p(d_ctx), 2, 7, p(d_unc), 2, TS, IS, STEPS, None, 32, 32, p(d_lat),
                                             None, None))
    # both contexts still work and are unchanged
    assert np.array_equal(case["run"](sd8), case["lat"])
    y = sd4.unet_forward(synth.make_latent(1, 32, 32, seed=5), 500, ctx[:1])
    assert np.isfinite(y).all()
