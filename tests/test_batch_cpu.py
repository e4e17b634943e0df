"""Batches of different requests (DESIGN.md §7 f7) without a GPU: the padding helper behind Context.sample_batch /
img2img_batch, the numpy mirror of the per-request start latents, and the batch_hetero fixture re-derived from the oracle."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import sd_oracle as O
from stable_diffusion_burn_b200 import _lib, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "batch_hetero.npz")


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def _maker():
    spec = importlib.util.spec_from_file_location("make_batch_golden", os.path.join(ROOT, "tests", "golden", "make_batch_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    return mk


# ------------------------------------------------------------------------------------------------ padding helper
def test_pack_ragged_with_a_shared_negative():
    ctxs = [synth.make_context(1, L, seed=L)[0] for L in (5, 13)] + [synth.make_context(1, 77, seed=1)]  # [L,768] or [1,L,768]
    unc = synth.make_context(1, 2, seed=99)[0]
    b = _lib.pack_batch(ctxs, unc, 7.5, seeds=[1, 2, 2 ** 40])
    assert b["context"].shape == (3, 77, 768) and b["context"].dtype == np.float32
    assert b["context_len"].tolist() == [5, 13, 77] and b["context_len"].dtype == np.int32
    for i, L in enumerate((5, 13, 77)):
        assert np.array_equal(b["context"][i, :L], np.asarray(ctxs[i]).reshape(L, 768))
        assert not b["context"][i, L:].any()
    assert b["uncond"].shape == (3, 2, 768) and b["uncond_len"].tolist() == [2, 2, 2]
    assert all(np.array_equal(b["uncond"][i], unc) for i in range(3))
    assert b["scale"].tolist() == [7.5] * 3 and b["scale"].dtype == np.float64
    assert b["seed"].tolist() == [1, 2, 2 ** 40] and b["seed"].dtype == np.uint64
    assert b["noise_seed"] is None


def test_pack_per_request_negatives_and_the_struct():
    ctxs = [synth.make_context(1, L, seed=L)[0] for L in (5, 13)]
    uncs = [synth.make_context(1, 2, seed=99), synth.make_context(1, 9, seed=4)[0]]
    b = _lib.pack_batch(ctxs, uncs, [7.5, 1.0], noise_seeds=[3, 4])
    assert b["uncond"].shape == (2, 9, 768) and b["uncond_len"].tolist() == [2, 9]
    assert np.array_equal(b["uncond"][0, :2], uncs[0][0]) and not b["uncond"][0, 2:].any()
    assert np.array_equal(b["uncond"][1], uncs[1])
    assert b["scale"].tolist() == [7.5, 1.0] and b["seed"] is None and b["noise_seed"].tolist() == [3, 4]
    s = _lib.batch_struct(b)
    assert (s.n, s.L, s.Lu) == (2, 13, 9)
    assert s.context == b["context"].ctypes.data and s.uncond == b["uncond"].ctypes.data
    assert [s.context_len[i] for i in range(2)] == [5, 13] and [s.uncond_len[i] for i in range(2)] == [2, 9]
    assert [s.guidance_scale[i] for i in range(2)] == [7.5, 1.0] and not s.seed and [s.noise_seed[i] for i in range(2)] == [3, 4]
    d = _lib.batch_struct(b, 0x1000, 0x2000)  # the _dev entries: device context / uncond
    assert (d.context, d.uncond) == (0x1000, 0x2000)
    assert C.sizeof(_lib.SdbBatch) == 72  # the C layout of sdb_batch on LP64


@pytest.mark.parametrize("args,what", [
    (([], np.zeros((2, 768)), 1.0), "non-empty"),
    ((np.zeros((1, 5, 768), np.float32), np.zeros((2, 768)), 1.0), "non-empty"),
    (([np.zeros((5, 700))], np.zeros((2, 768)), 1.0), r"contexts\[0\]"),
    (([np.zeros((0, 768))], np.zeros((2, 768)), 1.0), r"contexts\[0\]"),
    (([np.zeros((2, 5, 768))], np.zeros((2, 768)), 1.0), r"contexts\[0\]"),
    (([np.zeros((5, 768))], [np.zeros((2, 768))] * 2, 1.0), "2 unconditional contexts for 1"),
    (([np.zeros((5, 768))], [np.zeros((2, 7))], 1.0), r"unconds\[0\]"),
    (([np.zeros((5, 768))] * 2, np.zeros((2, 768)), [1.0]), "scales"),
    (([np.zeros((5, 768))], np.zeros((2, 768)), float("nan")), "finite"),
    (([np.zeros((5, 768))], np.zeros((2, 768)), [float("inf")]), "finite"),
])
def test_pack_errors(args, what):
    with pytest.raises(ValueError, match=what):
        _lib.pack_batch(*args)


def test_pack_seed_counts():
    with pytest.raises(ValueError, match="seeds"):
        _lib.pack_batch([np.zeros((5, 768))] * 2, np.zeros((2, 768)), 1.0, seeds=[1])
    with pytest.raises(ValueError, match="noise_seeds"):
        _lib.pack_batch([np.zeros((5, 768))] * 2, np.zeros((2, 768)), 1.0, noise_seeds=[1, 2, 3])


# ------------------------------------------------------------------------------------------------ start latents
def test_seeded_latents_are_the_init_stream_per_request():
    """Request i is the stream the single-request entries draw for seeds[i] at n = 1 (randn_launch: randn_stream under the
    seed's init keys), at the index within the request; the eta-noise keys are the same init keys mixed with the timestep."""
    seeds = [0, 7, 2 ** 33 + 5]
    x = synth.seeded_latents(seeds, 8, 16)
    assert x.shape == (3, 4, 8, 16) and x.dtype == np.float32
    for i, s in enumerate(seeds):
        assert np.array_equal(x[i].ravel(), synth.randn_stream(4 * 8 * 16, *synth.init_noise_keys(s)))
        assert np.array_equal(synth.seeded_latents([s], 8, 16)[0], x[i])
        k0, k1 = synth.step_noise_keys(s, 999)
        assert k0 ^ synth._mix32_scalar(0x3C6EF372 + 999) == synth.init_noise_keys(s)[0]
        assert k1 ^ synth._mix32_scalar(k0 ^ 0xA54FF53A) == synth.init_noise_keys(s)[1]
    assert not np.array_equal(x[0], x[1]) and abs(float(x.mean())) < 0.1 and abs(float(x.std()) - 1.0) < 0.1


# ------------------------------------------------------------------------------------------------ fixture
def test_fixture_inputs():
    mk = _maker()
    cfg = mk.BATCH_CASES
    g = np.load(GOLD)
    ctxs, uncs, noise = mk.requests()
    assert [c.shape[0] for c in ctxs] == [5, 13, 77] and [u.shape[0] for u in uncs] == [2, 9, 2]
    assert np.array_equal(uncs[0], uncs[2]) and cfg["scales"] == (7.5, 1.0, 3.0) and len(set(cfg["seeds"])) == 3
    assert np.array_equal(g["noise"], noise) and np.array_equal(noise, synth.seeded_latents(cfg["seeds"], 32, 32))
    for k in ("ddim", "dpmpp", "eta", "inpaint"):
        assert g[f"{k}_latent"].shape == (3, 4, 32, 32) and g[f"{k}_u8"].shape == (3, 128, 128, 3)


def test_fixture_rederived():
    """The whole fixture from the oracle, each request on its own (about two minutes on 8 cores)."""
    torch.set_num_threads(os.cpu_count() or 1)
    out = _maker().compute(O.Params(synth.make_params(0)))
    g = np.load(GOLD)
    for k in ("ddim", "dpmpp", "eta", "inpaint"):
        assert rel(out[f"{k}_latent"], g[f"{k}_latent"]) < 1e-4, k
        d = np.abs(out[f"{k}_u8"].astype(np.int16) - g[f"{k}_u8"].astype(np.int16))
        assert (d <= 1).mean() >= 0.999 and d.max() <= 2, k
