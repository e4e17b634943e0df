"""The samplers (DESIGN.md §7 f6) in the CPU oracle: DPM-Solver++(2M) converges at second order and DDIM at first on a problem with
an exact solution, the identities the GPU suite relies on, the argument rules, the per-step noise mirror, and the sampler_b2
fixture re-derived."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import sd_oracle as O
from stable_diffusion_burn_b200 import synth

import sampler_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "sampler_b2.npz")


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


# ------------------------------------------------------------------------------------------------ convergence order
@pytest.mark.parametrize("kind,lo,hi", [(SO.DDIM, 0.8, 1.2), (SO.DPMPP_2M, 1.8, None)])
def test_convergence_order_on_gaussian_data(kind, lo, hi):
    """Gaussian data N(0.7, 0.3^2) under the SD-v1 schedule: the exact probability-flow map from t = 999 to t = 99 against the
    solver on nested grids of 9 ... 144 steps, max error over x_T in [-3, 3]. The fixed endpoint matters: on the library's own
    schedule the last timestep moves with n_steps and a fitted order means nothing."""
    ab = synth.alpha_cumulative_products().astype(np.float64)
    mu, s = 0.7, 0.3
    x = np.linspace(-3.0, 3.0, 61)
    errs = []
    for n in (9, 18, 36, 72, 144):
        g = SO.nested_grid(n)
        assert g[0] == 999 and g[-1] == 99 and len(set(g)) == n + 1
        abars = [float(ab[t]) for t in g]
        got = SO.gaussian_solve(kind, x.copy(), abars, mu, s)
        errs.append(float(np.abs(got - SO.gaussian_flow(x, abars[0], abars[-1], mu, s)).max()))
    orders = [math.log2(errs[i] / errs[i + 1]) for i in range(len(errs) - 1)]
    print(f"kind {kind}: max error {errs[0]:.2e} -> {errs[-1]:.2e}, observed orders " + " ".join(f"{o:.2f}" for o in orders))
    assert all(o >= lo for o in orders)
    if hi is not None:
        assert all(o <= hi for o in orders)


def test_first_order_dpmpp_step_is_ddim():
    """A first-order DPM++ step is DDIM with eta = 0: sigma'/sigma x - alpha' expm1(-h) x0 = alpha' x0 + sigma' eps."""
    ab = synth.alpha_cumulative_products().astype(np.float64)
    x, x0 = np.linspace(-2, 2, 9), np.linspace(1, -1, 9)
    for t, tn in ((999, 749), (500, 450), (60, 10)):
        a, an = float(ab[t]), float(ab[tn])
        cx, cd, c2, _ = SO.dpmpp_coefs(a, an, None)
        assert c2 is None
        eps = (x - math.sqrt(a) * x0) / math.sqrt(1.0 - a)
        np.testing.assert_allclose(cx * x + cd * x0, math.sqrt(an) * x0 + math.sqrt(1.0 - an) * eps, rtol=1e-12, atol=1e-12)
    assert SO.dpmpp_coefs(float(ab[49]), 1.0, 0.3) == (0.0, 1.0, None, None)  # the final step returns x0
    assert SO.ddim_coefs(float(ab[49]), 1.0, 1.0) == (0.0, 0.0)  # and so does eta-DDIM's: s = 0


@pytest.mark.parametrize("eta", [0.0, 0.3, 1.0])
def test_eta_keeps_the_direction_real(eta):
    ab = synth.alpha_cumulative_products().astype(np.float64)
    for n_steps in (1, 4, 20, 50, 1000):
        ts, step = O.ddim_timesteps(n_steps)
        for t in ts:
            a, an = float(ab[t]), (float(ab[t - step]) if t >= step else 1.0)
            s, d = SO.ddim_coefs(a, an, eta)
            assert 0.0 <= s and 1.0 - an - s * s >= -1e-15 and np.isfinite(d)


# ------------------------------------------------------------------------------------------------ argument rules
def test_argument_rules():
    for kind, eta in ((0, 0.0), (0, 0.5), (0, 1.0), (1, 0.0)):
        SO.check_sampler(kind, eta)
    for eta in (-0.1, 1.01, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="eta"):
            SO.check_sampler(SO.DDIM, eta)
    with pytest.raises(ValueError, match="deterministic"):
        SO.check_sampler(SO.DPMPP_2M, 0.5)
    for kind in (-1, 2, 7):
        with pytest.raises(ValueError, match="unknown"):
            SO.check_sampler(kind, 0.0)


# ------------------------------------------------------------------------------------------------ noise mirror
def test_step_noise_moments_and_keys():
    z = synth.step_noise(5, 999, (4, 4, 64, 64))
    assert z.dtype == np.float32 and z.shape == (4, 4, 64, 64) and np.isfinite(z).all()
    assert abs(float(z.mean())) < 0.01 and abs(float(z.std()) - 1.0) < 0.01
    assert abs(float((z.astype(np.float64) ** 4).mean()) - 3.0) < 0.1
    others = [synth.step_noise(6, 999, z.shape), synth.step_noise(5, 949, z.shape), synth.step_noise(5 + (1 << 32), 999, z.shape)]
    for o in others:
        assert abs(np.corrcoef(z.ravel(), o.ravel())[0, 1]) < 0.01
    assert np.array_equal(synth.step_noise(5, 999, z.shape), z)
    # a prefix of the stream does not depend on the call's size (the key is the flat element index)
    assert np.array_equal(synth.step_noise(5, 999, (2, 4, 64, 64)), z[:2])


# ------------------------------------------------------------------------------------------------ full-model identities
@pytest.fixture(scope="module")
def small():
    """Full-model oracle at the smallest shapes: an 8x8 latent, L = 3, Lu = 2."""
    torch.set_num_threads(os.cpu_count() or 1)
    P = O.Params(synth.make_params(0))
    return dict(P=P, ctx=torch.from_numpy(synth.make_context(1, 3, seed=8)),
                unc=torch.from_numpy(synth.make_context(1, 2, seed=99))[0], init=torch.from_numpy(synth.make_latent(1, 8, 8, seed=9)))


def test_eta_zero_is_sample_latent(small):
    with torch.no_grad():
        want = O.sample_latent(small["P"], small["ctx"], small["unc"], 5.0, 2, small["init"]).numpy()
        got = SO.sampler_latent(small["P"], small["ctx"], small["unc"], 5.0, 2, small["init"], SO.DDIM, 0.0).numpy()
    assert np.array_equal(got, want)


@pytest.mark.parametrize("n_steps", [1, 2])
def test_all_first_order_dpmpp_is_ddim(small, n_steps):
    """n_steps = 1, 2: the first step has no history and the last returns x0, so DPM++ takes first-order steps only."""
    with torch.no_grad():
        ddim = O.sample_latent(small["P"], small["ctx"], small["unc"], 5.0, n_steps, small["init"]).numpy()
        dpm = SO.sampler_latent(small["P"], small["ctx"], small["unc"], 5.0, n_steps, small["init"], SO.DPMPP_2M).numpy()
    e = rel(dpm, ddim)
    print(f"n_steps {n_steps}: DPM++ vs DDIM rel L2 {e:.2e}")
    assert e < 1e-5


# ------------------------------------------------------------------------------------------------ fixture
def test_fixture_inputs():
    g = np.load(GOLD)
    assert np.array_equal(g["noise"], synth.make_latent(2, 32, 32, seed=41))
    for k in ("dpmpp", "eta", "inpaint"):
        assert g[f"{k}_latent"].shape == (2, 4, 32, 32) and g[f"{k}_u8"].shape == (2, 128, 128, 3)
    first, ts = SO.img2img_start(SO.SAMPLER_CASES["strength"], SO.SAMPLER_CASES["n_steps"])
    assert ts[first:] == [749, 499, 249]


def test_fixture_rederived(small):
    """The whole fixture from the oracle (about a minute on 8 cores)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_sampler_golden", os.path.join(ROOT, "tests", "golden",
                                                                                      "make_sampler_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    g = np.load(GOLD)
    out = mk.compute(small["P"])
    for k in ("dpmpp", "eta", "inpaint"):
        assert rel(out[f"{k}_latent"], g[f"{k}_latent"]) < 1e-4, k
        d = np.abs(out[f"{k}_u8"].astype(np.int16) - g[f"{k}_u8"].astype(np.int16))
        assert (d <= 1).mean() >= 0.999 and d.max() <= 2, k
