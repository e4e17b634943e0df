"""Inpainting with a 9-channel UNet on the GPU (DESIGN.md §7 f9) through the C ABI: the registry of sdb_create_inpaint, the
inpaint_b2 fixture, the step-exact conditioning against a host loop of sdb_forward_diffuser, the zero-weight identity with the
4-channel model, the step-graph cache, host / device entries, batches, launch counts and errors."""
import contextlib
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from stable_diffusion_burn_b200 import _lib, dumpdir, synth, topology

import img2img_oracle as IO
import inpaint_oracle as NO
import sampler_oracle as SO

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inpaint_b2.npz")
STEPS, SCALE, NSEED, ETA = NO.INPAINT["n_steps"], NO.INPAINT["scale"], 11, 0.7
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


@pytest.fixture(scope="module")
def sd4(ctx):
    ctx.init_synthetic(0)
    ctx.finalize_weights()
    return ctx


@pytest.fixture(scope="module")
def sd9(sd4):
    """A second context, 9-channel, beside the session's: a small work arena, since the default one of each would take most of
    the card. Synthetic seed 0, so every tensor but conv_in equals the session context's."""
    old = os.environ.get("SDB_WORK_GB")
    os.environ["SDB_WORK_GB"] = "8"
    try:
        c = _lib.Context(0, inpaint=True)
    finally:
        if old is None:
            del os.environ["SDB_WORK_GB"]
        else:
            os.environ["SDB_WORK_GB"] = old
    c.init_synthetic(0)
    c.finalize_weights()
    yield c
    c.close()


@pytest.fixture(scope="module")
def case(sd9):
    g = np.load(GOLD)
    d = dict(g=g, image=g["image"], mask=g["mask"], noise=g["noise"], ctx=synth.make_context(2, 7, seed=3),
             unc=synth.make_context(1, 2, seed=99)[0])

    def run(sd, name="ddim", strength=1.0, mask=d["mask"], image=d["image"], noise=d["noise"], ctx=d["ctx"]):
        with sampler(sd, name):
            return sd.img2img(image, ctx, d["unc"], SCALE, STEPS, strength, mask=mask, noise=noise, latent=True, rgb=False)

    d["run"] = run
    d["lat"] = run(sd9)
    return d


def test_registry_is_the_inpaint_topology(sd9, sd4):
    got = sd9.tensor_list()
    want = [(n, tuple(s)) for (n, s, _, _) in topology.all_params(inpaint=True)] + [("alpha_cumulative_products", (1000,))]
    assert got == want
    assert sd9.unet_in_channels() == 9 and sd4.unet_in_channels() == 4
    four = sd4.tensor_list()
    assert [n for n, _ in four] == [n for n, _ in got]
    assert [i for i, (a, b) in enumerate(zip(four, got)) if a != b] == [[n for n, _ in got].index(CONV_IN)]


def test_golden(sd9, case):
    g = case["g"]
    for name, c in NO.INPAINT_CASES.items():
        smp = "dpmpp" if c["kind"] == SO.DPMPP_2M else "ddim"
        with sampler(sd9, smp):
            lat, rgb = sd9.img2img(case["image"], case["ctx"], case["unc"], SCALE, STEPS, c["strength"], mask=case["mask"],
                                   noise=case["noise"], latent=True, rgb=True)
        e = rel(lat, g[f"latent_{name}"])
        dd = np.abs(rgb[:, ::2, ::2, :].astype(np.int16) - g[f"u8_{name}"].astype(np.int16))
        frac, dmax = float((dd <= 1).mean()), int(dd.max())
        print(f"inpaint {name}: latent rel L2 {e:.3e}, u8 within 1 LSB {frac:.5f}, max {dmax}")
        assert e < 2e-3 and frac >= 0.998 and dmax <= 4, name


def _host_loop(sd, case, name, strength):
    """sdb_img2img on a 9-channel context restated on the host: z0 and z_m from sdb_encode_image, the latent mask and the start
    latent in numpy, each step's two UNet outputs from sdb_forward_diffuser on [n,9,H,W] = x | m_lat | z_m, and the update with
    the fused step's contractions (tests/test_sampler_gpu.py: _host_loop)."""
    kind, eta = SAMPLERS[name]
    z0 = SO.scaled_latent(sd.encode_image(IO.image_u8_to_float(case["image"])))
    z_m = SO.scaled_latent(sd.encode_image(NO.masked_image(case["image"], case["mask"])))
    cond = np.concatenate([NO.latent_mask(case["mask"])[:, None], z_m], 1)
    alphas = sd.get_tensor("alpha_cumulative_products", (1000,))
    first, ts = SO.img2img_start(strength, STEPS)

    def guide(x, t):
        _, u, c = sd.forward_diffuser(np.concatenate([x, cond], 1), t, case["ctx"], case["unc"], SCALE)
        return SO.fma(np.subtract(c, u), np.float32(SCALE), u)

    return SO.step_loop(SO.start_latent(float(alphas[ts[first]]), z0, case["noise"]), guide, alphas, STEPS, SO.KERNEL, kind, eta,
                        lambda t, shape: sd.test_step_noise(NSEED, t, math.prod(shape)).reshape(shape), first)


@pytest.mark.parametrize("name", list(SAMPLERS))
def test_step_exact_conditioning(sd9, case, name):
    got = case["run"](sd9, name, strength=0.75)
    want = _host_loop(sd9, case, name, 0.75)
    print(f"inpaint {name}: sdb_img2img vs host loop of forward_diffuser, rel L2 {rel(got, want):.3e}")
    assert np.array_equal(got, want)


@pytest.fixture
def zero_ext(sd9, sd4):
    """conv_in of the 9-channel context = the session context's conv_in, extended by zero weights on channels 4-8."""
    keep = sd9.get_tensor(CONV_IN, (320, 9, 3, 3))
    sd9.set_tensor(CONV_IN, NO.zero_extension(sd4.get_tensor(CONV_IN, (320, 4, 3, 3))))
    sd9.finalize_weights()
    yield
    sd9.set_tensor(CONV_IN, keep)
    sd9.finalize_weights()


@pytest.mark.parametrize("name", list(SAMPLERS))
def test_zero_weight_identity(sd9, sd4, case, zero_ext, name):
    for mask in (case["mask"], np.full_like(case["mask"], 255)):
        got = case["run"](sd9, name, strength=0.75, mask=mask)
        want = case["run"](sd4, name, strength=0.75, mask=None)
        assert np.array_equal(got, want)
    x = synth.make_latent(2, 32, 32, seed=5)
    junk = synth.make_latent(2, 32, 32, seed=6)[:, :4].repeat(2, 1)[:, :5]
    got = sd9.unet_forward(np.concatenate([x, junk], 1), 500, case["ctx"])
    assert np.array_equal(got, sd4.unet_forward(x, 500, case["ctx"]))


def test_mask_changes_the_result(sd9, case):
    other = case["mask"].copy()
    other[:, :, :64] = 255
    got = case["run"](sd9, mask=other)
    assert not np.array_equal(got, case["lat"])
    assert np.array_equal(case["run"](sd9), case["lat"])


def test_step_graph_cache(sd9, case):
    """Two latent sizes in turn make the conditioning slot regrow (and move); the first size again must still be right."""
    img64 = np.ascontiguousarray(np.tile(case["image"][:1], (1, 2, 2, 1)))
    m64 = np.ascontiguousarray(np.tile(case["mask"][:1], (1, 2, 2)))
    n64 = synth.make_latent(1, 64, 64, seed=12)
    big = case["run"](sd9, image=img64, mask=m64, noise=n64, ctx=case["ctx"][:1])
    again = case["run"](sd9)
    assert np.array_equal(again, case["lat"])
    sd9.set_option("graphs", 0)
    try:
        off = case["run"](sd9)
        big_off = case["run"](sd9, image=img64, mask=m64, noise=n64, ctx=case["ctx"][:1])
    finally:
        sd9.set_option("graphs", 1)
    assert np.array_equal(off, case["lat"]) and np.array_equal(big_off, big)
    sd9.set_option("emb_hoist", 0)
    try:
        assert np.array_equal(case["run"](sd9), case["lat"])
    finally:
        sd9.set_option("emb_hoist", 1)


def test_host_equals_dev(sd9, case):
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_img, d_mask, d_ctx, d_unc, d_noise = (t(a) for a in (case["image"], case["mask"], case["ctx"], case["unc"], case["noise"]))
    d_lat = torch.empty((2, 4, 32, 32), dtype=torch.float32, device=dev)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda x: C.c_void_p(x.data_ptr())
    sd9.check(sd9.lib.sdb_img2img_dev(sd9.h, p(d_img), p(d_mask), 1.0, p(d_ctx), 2, 7, p(d_unc), 2, SCALE, STEPS, p(d_noise), 32,
                                      32, p(d_lat), None, st))
    torch.cuda.synchronize()
    assert np.array_equal(d_lat.cpu().numpy(), case["lat"])
    x9 = np.concatenate([case["noise"], synth.make_latent(2, 32, 32, seed=7)[:, :4], case["noise"][:, :1]], 1)
    d_x, d_out = t(x9), torch.empty((2, 4, 32, 32), dtype=torch.float32, device=dev)
    sd9.check(sd9.lib.sdb_unet_forward_dev(sd9.h, p(d_x), 500, p(d_ctx), 2, 32, 32, 7, p(d_out), st))
    torch.cuda.synchronize()
    assert np.array_equal(d_out.cpu().numpy(), sd9.unet_forward(x9, 500, case["ctx"]))


def test_batches(sd9, case):
    uni = sd9.img2img_batch(case["image"], list(case["ctx"][:, None]), case["unc"], SCALE, STEPS, 1.0, mask=case["mask"],
                            noise=case["noise"], latent=True, rgb=False)
    assert np.array_equal(uni, case["lat"])
    for i in (0, 1):
        one = case["run"](sd9, image=case["image"][i:i + 1], mask=case["mask"][i:i + 1], noise=case["noise"][i:i + 1],
                          ctx=case["ctx"][i:i + 1])
        e = rel(one, case["lat"][i:i + 1])
        print(f"inpaint batch member {i}: rel L2 {e:.3e}")
        assert e < 1e-3


def test_launch_counts(sd9, sd4, case):
    """Per step: as many launches as masked 4-channel img2img. Per call: inpaint_prep and one encoder pass more."""
    def count(sd, n_steps, mask):
        sd.img2img(case["image"], case["ctx"], case["unc"], SCALE, n_steps, 1.0, mask=mask, noise=case["noise"], latent=True,
                   rgb=False)  # the step graph of this shape is cached
        n0 = sd.launch_count()
        sd.img2img(case["image"], case["ctx"], case["unc"], SCALE, n_steps, 1.0, mask=mask, noise=case["noise"], latent=True,
                   rgb=False)
        return sd.launch_count() - n0
    c9 = {k: count(sd9, k, case["mask"]) for k in (2, 4)}
    c4 = {k: count(sd4, k, case["mask"]) for k in (2, 4)}
    assert c9[4] - c9[2] == c4[4] - c4[2] > 0
    n0 = sd4.launch_count()
    sd4.encode_image(IO.image_u8_to_float(case["image"]))
    enc = sd4.launch_count() - n0
    print(f"launches per call: 9-channel {c9[4]}, 4-channel {c4[4]}, encoder pass {enc}")
    assert c9[4] - c4[4] == 1 + enc


def _conv_tree(root, cin):
    """The smallest dump-dir that reaches the conv_in check: the schedule length and a [320,cin,3,3] conv_in."""
    os.makedirs(os.path.join(root, "unet/input_blocks/conv"), exist_ok=True)
    dumpdir.save_scalar(1000, "n_steps", root)
    dumpdir.save_tensor(np.zeros((320, cin, 3, 3), np.float32), "weight", os.path.join(root, "unet/input_blocks/conv"))
    return root


def test_errors(sd9, sd4, case, tmp_path):
    u8, ptr = (lambda a: a.ctypes.data_as(_lib._u8p)), _lib.ptr
    with pytest.raises(_lib.SdbError, match="mask"):
        sd9.check(sd9.lib.sdb_img2img(sd9.h, u8(case["image"]), None, 1.0, ptr(case["ctx"]), 2, 7, ptr(case["unc"]), 2, SCALE,
                                      STEPS, ptr(case["noise"]), 0, 32, 32, ptr(np.empty((2, 4, 32, 32), np.float32)), None))
    with pytest.raises(_lib.SdbError, match="mask"):
        sd9.img2img_batch(case["image"], list(case["ctx"][:, None]), case["unc"], SCALE, STEPS, 1.0, noise=case["noise"])
    with pytest.raises(_lib.SdbError, match="sdb_img2img"):
        sd9.sample_latent(case["ctx"], case["unc"], SCALE, STEPS, init_latent=case["noise"])
    with pytest.raises(_lib.SdbError, match="sdb_img2img"):
        sd9.sample_image(case["ctx"], case["unc"], SCALE, STEPS, seed=1, H=32, W=32)
    with pytest.raises(_lib.SdbError, match="sdb_img2img"):
        sd9.sample_batch(list(case["ctx"][:, None]), case["unc"], SCALE, STEPS, seeds=[1, 2], H=32, W=32)
    with pytest.raises(_lib.SdbError, match=r"\[320,4,3,3\].*\[320,9,3,3\].*sdb_create\b"):
        sd9.set_tensor(CONV_IN, np.zeros((320, 4, 3, 3), np.float32))
    with pytest.raises(_lib.SdbError, match=r"\[320,9,3,3\].*\[320,4,3,3\].*sdb_create_inpaint"):
        sd4.set_tensor(CONV_IN, np.zeros((320, 9, 3, 3), np.float32))
    with pytest.raises(_lib.SdbError, match=r"\[320,4,3,3\].*sdb_create\b"):
        sd9.load_dump_dir(_conv_tree(str(tmp_path / "four"), 4))
    with pytest.raises(_lib.SdbError, match=r"\[320,9,3,3\].*sdb_create_inpaint"):
        sd4.load_dump_dir(_conv_tree(str(tmp_path / "nine"), 9))
    # both contexts are still usable and unchanged
    assert np.array_equal(case["run"](sd9), case["lat"])
    x = synth.make_latent(1, 32, 32, seed=5)
    y = sd4.unet_forward(x, 500, case["ctx"][:1])
    assert np.isfinite(y).all()
