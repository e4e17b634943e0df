"""Batches of different requests on the GPU (DESIGN.md §7 f7) through the C ABI: the batch_hetero fixture, the uniform batch and
the n = 1 seeded batch against the single-request entries bit for bit, pad rows never read, batch independence, the step-graph
cache and options, host / device entries, the launch budget and errors."""
import contextlib
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from stable_diffusion_burn_b200 import _lib, pipeline, synth

import sampler_oracle as SO

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "batch_hetero.npz")
STEPS, SCALE = 4, 5.0
SAMPLERS = {"ddim": (SO.DDIM, 0.0), "eta": (SO.DDIM, 0.7), "dpmpp": (SO.DPMPP_2M, 0.0)}


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


@contextlib.contextmanager
def sampler(sd, name, noise_seed=0):
    sd.set_sampler(*SAMPLERS[name], noise_seed)
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
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import make_batch_golden as MB
    from img2img_oracle import img2img_inputs
    cfg = MB.BATCH_CASES
    ctxs, uncs, _ = MB.requests()
    g = np.load(GOLD)
    image, mask = img2img_inputs()
    d = dict(g=g, cfg=cfg, ctxs=ctxs, uncs=uncs, noise=g["noise"], image=image[list(cfg["images"])],
             mask=mask[list(cfg["masks"])], ctx2=synth.make_context(2, 7, seed=3), unc=synth.make_context(1, 2, seed=99)[0],
             noise2=synth.make_latent(2, 32, 32, seed=41), image2=image, mask2=mask)

    def txt(name, idx=(0, 1, 2), **kw):
        idx = list(idx)
        with sampler(sd, name):
            return sd.sample_batch([ctxs[i] for i in idx], [uncs[i] for i in idx], [cfg["scales"][i] for i in idx], STEPS,
                                   noise_seeds=[cfg["noise_seeds"][i] for i in idx], init_latent=d["noise"][idx], latent=True,
                                   rgb=False, **kw)

    def inpaint(idx=(0, 1, 2)):
        idx = list(idx)
        with sampler(sd, "dpmpp"):
            return sd.img2img_batch(d["image"][idx], [ctxs[i] for i in idx], [uncs[i] for i in idx],
                                    [cfg["scales"][i] for i in idx], STEPS, cfg["strength"], mask=d["mask"][idx],
                                    noise=d["noise"][idx], latent=True, rgb=False)

    d["txt"], d["inpaint"] = txt, inpaint
    d["res"] = {k: txt(k) for k in SAMPLERS}
    d["res"]["inpaint"] = inpaint()
    return d


def test_golden(sd, case):
    """Each request of the heterogeneous batch against the oracle run of that request alone, at the bars of
    test_sample_two_steps_batch2_golden."""
    g = case["g"]
    for name in ("ddim", "dpmpp", "eta", "inpaint"):
        lat = case["res"][name]
        e = rel(lat, g[f"{name}_latent"])
        u8 = sd.latent_to_image(lat)[:, ::2, ::2, :]
        dd = np.abs(u8.astype(np.int16) - g[f"{name}_u8"].astype(np.int16))
        frac, dmax = float((dd <= 1).mean()), int(dd.max())
        per = [rel(lat[i], g[f"{name}_latent"][i]) for i in range(3)]
        print(f"batch {name}: latent rel L2 {e:.3e} (per request {', '.join(f'{v:.2e}' for v in per)}), u8 within 1 LSB "
              f"{frac:.5f}, max {dmax}")
        assert e < 2e-3 and max(per) < 2e-3 and frac >= 0.998, name


@pytest.mark.parametrize("name", ["ddim", "dpmpp"])
def test_uniform_batch_is_the_single_request_call(sd, case, name):
    """Equal lengths, one negative, one scale, an explicit start latent / noise: sdb_sample_batch and sdb_img2img_batch give
    exactly what sdb_sample_latent, sdb_sample_image and sdb_img2img (with and without a mask) give."""
    ctx2, unc, noise = case["ctx2"], case["unc"], case["noise2"]
    rows = [ctx2[0], ctx2[1]]
    with sampler(sd, name):
        lat, rgb = sd.sample_batch(rows, unc, SCALE, STEPS, init_latent=noise, latent=True, rgb=True)
        assert np.array_equal(lat, sd.sample_latent(ctx2, unc, SCALE, STEPS, init_latent=noise))
        assert np.array_equal(rgb, sd.sample_image(ctx2, unc, SCALE, STEPS, init_latent=noise))
        for mask in (None, case["mask2"]):
            want = sd.img2img(case["image2"], ctx2, unc, SCALE, STEPS, 0.75, mask=mask, noise=noise, latent=True, rgb=False)
            got = sd.img2img_batch(case["image2"], rows, [unc, unc], [SCALE, SCALE], STEPS, 0.75, mask=mask, noise=noise,
                                   latent=True, rgb=False)
            assert np.array_equal(got, want), mask is not None


@pytest.mark.parametrize("name", list(SAMPLERS))
def test_one_seeded_request_is_the_seeded_call(sd, case, name):
    """n = 1: seed = s and noise_seed = q give exactly sdb_sample_latent(seed = s) / sdb_img2img(seed = s) under
    sdb_set_sampler(..., q). (At n > 1 the batch keys eta noise per sample, the single-request call over the flat latent.)"""
    ctx1, unc = case["ctx2"][:1], case["unc"]
    s, q = 2 ** 35 + 17, 29
    with sampler(sd, name, q):
        want = sd.sample_latent(ctx1, unc, SCALE, STEPS, seed=s, H=32, W=32)
        want_i2i = sd.img2img(case["image2"][:1], ctx1, unc, SCALE, STEPS, 0.75, mask=case["mask2"][:1], seed=s, latent=True,
                              rgb=False)
    with sampler(sd, name):
        got = sd.sample_batch([ctx1[0]], unc, SCALE, STEPS, seeds=[s], noise_seeds=[q], H=32, W=32, latent=True, rgb=False)
        got_i2i = sd.img2img_batch(case["image2"][:1], [ctx1[0]], unc, SCALE, STEPS, 0.75, mask=case["mask2"][:1], seeds=[s],
                                   noise_seeds=[q], latent=True, rgb=False)
    assert np.array_equal(got, want) and np.array_equal(got_i2i, want_i2i)
    with sampler(sd, name, q):  # noise_seed NULL: the context's noise seed
        assert np.array_equal(sd.sample_batch([ctx1[0]], unc, SCALE, STEPS, seeds=[s], H=32, W=32, latent=True, rgb=False), want)


def _raw_batch(sd, b, init):
    lat = np.empty((b["context"].shape[0], 4, 32, 32), np.float32)
    sd.check(sd.lib.sdb_sample_batch(sd.h, C.byref(_lib.batch_struct(b)), STEPS, _lib.ptr(np.ascontiguousarray(init)), 32, 32,
                                     _lib.ptr(lat), None))
    return lat


def test_pad_rows_are_never_read(sd, case):
    """Caller pad rows full of NaN give the zero-padded result bit for bit; lengths 5 at stride 13 give the L = 5 call."""
    cfg = case["cfg"]
    b = _lib.pack_batch(case["ctxs"], case["uncs"], cfg["scales"], noise_seeds=cfg["noise_seeds"])
    for key, lens in (("context", b["context_len"]), ("uncond", b["uncond_len"])):
        for i, l in enumerate(lens):
            b[key][i, l:] = np.nan
    with sampler(sd, "eta"):
        assert np.array_equal(_raw_batch(sd, b, case["noise"]), case["res"]["eta"])
    ctx5 = synth.make_context(2, 5, seed=8)
    wide = np.full((2, 13, 768), np.nan, np.float32)
    wide[:, :5] = ctx5
    b = _lib.pack_batch([ctx5[0], ctx5[1]], case["unc"], SCALE)
    b["context"], b["context_len"] = wide, np.array([5, 5], np.int32)
    for name in ("ddim", "dpmpp"):
        with sampler(sd, name):
            want = sd.sample_latent(ctx5, case["unc"], SCALE, STEPS, init_latent=case["noise2"])
            assert np.array_equal(_raw_batch(sd, b, case["noise2"]), want), name


def test_batch_independence(sd, case):
    """Request i of the heterogeneous batch is within 1e-3 of request i run alone, and a permutation of the requests permutes
    the outputs (split-K factors change with the batch size: the test_batch_invariance bar)."""
    for name in ("ddim", "eta"):
        full = case["res"][name]
        alone = [case["txt"](name, idx=(i,))[0] for i in range(3)]
        e = [rel(full[i], alone[i]) for i in range(3)]
        perm = (2, 0, 1)
        got = case["txt"](name, idx=perm)
        ep = [rel(got[j], full[i]) for j, i in enumerate(perm)]
        print(f"batch {name}: member vs alone rel L2 {', '.join(f'{v:.2e}' for v in e)}; permuted {', '.join(f'{v:.2e}' for v in ep)}")
        assert max(e) < 1e-3 and max(ep) < 1e-3, name


def test_step_graph_cache_and_options(sd, case):
    """A single-request call, a batch call of the same (nb, H, W, Lpad), the single-request call again: the same result. The
    graphs-off and emb_hoist-off paths give the default path's result."""
    cfg = case["cfg"]
    ctx3 = synth.make_context(3, 77, seed=5)
    a = sd.sample_latent(ctx3, case["unc"], SCALE, STEPS, init_latent=case["noise"])  # Lpad 96, as the batch
    assert np.array_equal(case["txt"]("ddim"), case["res"]["ddim"])
    assert np.array_equal(sd.sample_latent(ctx3, case["unc"], SCALE, STEPS, init_latent=case["noise"]), a)
    for opt in ("graphs", "emb_hoist"):
        sd.set_option(opt, 0)
        try:
            for name in SAMPLERS:
                assert np.array_equal(case["txt"](name), case["res"][name]), (opt, name)
            assert np.array_equal(case["inpaint"](), case["res"]["inpaint"]), opt
        finally:
            sd.set_option(opt, 1)


def test_host_equals_dev(sd, case):
    cfg = case["cfg"]
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    p = lambda x: C.c_void_p(x.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    b = _lib.pack_batch(case["ctxs"], case["uncs"], cfg["scales"], seeds=cfg["seeds"], noise_seeds=cfg["noise_seeds"])
    d_ctx, d_unc, d_noise, d_img, d_mask = (t(a) for a in (b["context"], b["uncond"], case["noise"], case["image"], case["mask"]))
    bs = _lib.batch_struct(b, d_ctx.data_ptr(), d_unc.data_ptr())
    d_lat = torch.empty((3, 4, 32, 32), dtype=torch.float32, device=dev)
    d_rgb = torch.empty((3, 256, 256, 3), dtype=torch.uint8, device=dev)
    for name in ("eta", "dpmpp"):
        with sampler(sd, name):
            sd.check(sd.lib.sdb_sample_batch_dev(sd.h, C.byref(bs), STEPS, p(d_noise), 32, 32, p(d_lat), p(d_rgb), st))
            torch.cuda.synchronize()
            assert np.array_equal(d_lat.cpu().numpy(), case["res"][name]), name
            assert np.array_equal(d_rgb.cpu().numpy(), sd.latent_to_image(case["res"][name])), name
            # seeds: the device draws the start latents
            sd.check(sd.lib.sdb_sample_batch_dev(sd.h, C.byref(bs), STEPS, None, 32, 32, p(d_lat), None, st))
            torch.cuda.synchronize()
            host = sd.sample_batch(case["ctxs"], case["uncs"], cfg["scales"], STEPS, seeds=cfg["seeds"],
                                   noise_seeds=cfg["noise_seeds"], H=32, W=32, latent=True, rgb=False)
            assert np.array_equal(d_lat.cpu().numpy(), host), name
            sd.check(sd.lib.sdb_img2img_batch_dev(sd.h, C.byref(bs), p(d_img), p(d_mask), cfg["strength"], STEPS, None, 32, 32,
                                                  p(d_lat), None, st))
            torch.cuda.synchronize()
            host = sd.img2img_batch(case["image"], case["ctxs"], case["uncs"], cfg["scales"], STEPS, cfg["strength"],
                                    mask=case["mask"], seeds=cfg["seeds"], noise_seeds=cfg["noise_seeds"], latent=True, rgb=False)
            assert np.array_equal(d_lat.cpu().numpy(), host), name
    with sampler(sd, "dpmpp"):
        sd.check(sd.lib.sdb_img2img_batch_dev(sd.h, C.byref(bs), p(d_img), p(d_mask), cfg["strength"], STEPS, p(d_noise), 32, 32,
                                              p(d_lat), None, st))
        torch.cuda.synchronize()
    assert np.array_equal(d_lat.cpu().numpy(), case["res"]["inpaint"])


def test_seeds_are_per_request(sd, case):
    """Each request's start latent comes from its own seed at the index within the request: member i of a seeded batch is within
    the batch-invariance bar of request i run alone from seeds[i], and of the batch started from the numpy mirror's latents
    (synth.seeded_latents, a few ulp from the device's logf / cosf)."""
    cfg = case["cfg"]
    with sampler(sd, "ddim"):
        got = sd.sample_batch(case["ctxs"], case["uncs"], cfg["scales"], STEPS, seeds=cfg["seeds"], H=32, W=32, latent=True,
                              rgb=False)
        alone = [sd.sample_batch([case["ctxs"][i]], [case["uncs"][i]], [cfg["scales"][i]], STEPS, seeds=[cfg["seeds"][i]], H=32,
                                 W=32, latent=True, rgb=False)[0] for i in range(3)]
    e = [rel(got[i], alone[i]) for i in range(3)]
    em = rel(got, case["res"]["ddim"])
    print(f"seeded batch: member vs alone rel L2 {', '.join(f'{v:.2e}' for v in e)}; vs mirror start latents {em:.2e}")
    assert max(e) < 1e-3 and em < 1e-3


@pytest.mark.parametrize("steps", [4, 8])
def test_launch_budget(sd, case, steps):
    """A batch call launches at most 2 more kernels than sdb_sample_latent at the same (nb, H, W, Lpad), and none per step."""
    cfg = case["cfg"]
    ctx3 = synth.make_context(3, 77, seed=5)
    run_a = lambda: sd.sample_latent(ctx3, case["unc"], SCALE, steps, seed=3, H=32, W=32)
    run_b = lambda: sd.sample_batch(case["ctxs"], case["uncs"], cfg["scales"], steps, seeds=cfg["seeds"], H=32, W=32,
                                    latent=True, rgb=False)
    run_a(), run_b()  # the step graph of this shape is cached
    counts = []
    for fn in (run_a, run_b):
        n0 = sd.launch_count()
        fn()
        counts.append(sd.launch_count() - n0)
    print(f"{steps} steps: launches sample_latent {counts[0]}, sample_batch {counts[1]}")
    assert counts[1] <= counts[0] + 2


def test_errors_leave_the_context_usable(sd, case):
    cfg = case["cfg"]
    good = lambda: _lib.pack_batch(case["ctxs"], case["uncs"], cfg["scales"], seeds=cfg["seeds"])
    lat = np.empty((3, 4, 32, 32), np.float32)

    def call(b, bs=None, init=None):
        bs = bs if bs is not None else _lib.batch_struct(b)
        sd.check(sd.lib.sdb_sample_batch(sd.h, C.byref(bs), STEPS, init, 32, 32, _lib.ptr(lat), None))

    cases = []
    b = good(); b["context_len"][1] = 0; cases.append((b, None, r"context_len\[1\] = 0"))
    b = good(); b["context_len"][2] = 78; cases.append((b, None, r"context_len\[2\] = 78 is outside \[1, L = 77\]"))
    b = good(); b["uncond_len"][0] = 10; cases.append((b, None, r"uncond_len\[0\] = 10"))
    b = good(); b["uncond_len"][2] = -1; cases.append((b, None, r"uncond_len\[2\] = -1"))
    b = good(); b["scale"][1] = np.inf; cases.append((b, None, r"guidance_scale\[1\] = inf"))
    b = good(); b["scale"][0] = np.nan; cases.append((b, None, r"guidance_scale\[0\] = nan"))
    b = good(); bs = _lib.batch_struct(b); bs.n = 0; cases.append((b, bs, "n = 0"))
    b = good(); bs = _lib.batch_struct(b); bs.seed = None; cases.append((b, bs, "seed is NULL"))
    b = good(); bs = _lib.batch_struct(b); bs.guidance_scale = None; cases.append((b, bs, "guidance_scale is NULL"))
    b = good(); bs = _lib.batch_struct(b); bs.context = None; cases.append((b, bs, "context is NULL"))
    b = good(); bs = _lib.batch_struct(b); bs.uncond = None; cases.append((b, bs, "uncond is NULL"))
    for b, bs, what in cases:
        with pytest.raises(_lib.SdbError, match=what):
            call(b, bs)
    with pytest.raises(_lib.SdbError, match="batch: null descriptor"):
        sd.check(sd.lib.sdb_sample_batch(sd.h, None, STEPS, None, 32, 32, _lib.ptr(lat), None))
    b = good()
    with pytest.raises(_lib.SdbError, match=r"context_len\[1\]"):
        b["context_len"][1] = 0
        sd.check(sd.lib.sdb_img2img_batch(sd.h, C.byref(_lib.batch_struct(b)), case["image"].ctypes.data_as(_lib._u8p), None,
                                          0.75, STEPS, None, 32, 32, _lib.ptr(lat), None))
    # a seed is not needed when the start latent is given
    b = good(); bs = _lib.batch_struct(b); bs.seed = None
    call(b, bs, _lib.ptr(np.ascontiguousarray(case["noise"])))
    # the context still works
    assert np.array_equal(case["txt"]("dpmpp"), case["res"]["dpmpp"])


def test_pipeline(sd, case):
    """StableDiffusion.sample_batch / img2img_batch: lists of flat u8 images, the sampler set for the call and restored."""
    cfg = case["cfg"]
    p = pipeline.StableDiffusion.__new__(pipeline.StableDiffusion)
    p.ctx = sd  # the session's context (a second one would hold another copy of the weights)
    ctxs = [c[None] for c in case["ctxs"]]  # [1, L, 768] as StableDiffusion.context returns
    out = p.sample_batch(ctxs, case["uncs"], list(cfg["scales"]), STEPS, list(cfg["seeds"]), height=256, width=256,
                         sampler="ddim", eta=0.7, noise_seeds=list(cfg["noise_seeds"]))
    with sampler(sd, "eta"):
        want = sd.sample_batch(case["ctxs"], case["uncs"], cfg["scales"], STEPS, seeds=cfg["seeds"],
                               noise_seeds=cfg["noise_seeds"], H=32, W=32)
    assert len(out) == 3 and np.array_equal(np.stack(out), want.reshape(3, -1))
    out = p.img2img_batch(case["image"], ctxs, case["uncs"], list(cfg["scales"]), STEPS, cfg["strength"], masks=case["mask"],
                          noise=case["noise"], sampler="dpmpp_2m")
    assert np.array_equal(np.stack(out), sd.latent_to_image(case["res"]["inpaint"]).reshape(3, -1))
    # the default sampler is back
    assert np.array_equal(sd.sample_batch(case["ctxs"], case["uncs"], cfg["scales"], STEPS, init_latent=case["noise"],
                                          noise_seeds=cfg["noise_seeds"], latent=True, rgb=False), case["res"]["ddim"])
