"""The Karras schedule (DESIGN.md §7 f15) in the CPU oracle: the grid and sigma_to_t against k-diffusion's numbers, the schedule
check and the argument rules, the library's VP step loop against the published VE samplers, the convergence orders on a problem
with an exact solution, and the schedule_b2 fixture re-derived."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import sd_oracle as O
from stable_diffusion_burn_b200 import synth

import sampler_oracle as SO
import schedule_oracle as KO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "schedule_b2.npz")
AB = synth.alpha_cumulative_products()


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


# ------------------------------------------------------------------------------------------------ the grid
def test_grid_values():
    sig = KO.karras_sigma_table(AB)
    assert abs(sig[999] - 14.614641) < 5e-7 and abs(sig[0] - 0.029168) < 5e-7
    s4 = KO.karras_sigmas(AB, 4)
    np.testing.assert_allclose(s4, [14.6146, 3.1686, 0.44692, 0.029168], rtol=2e-5)
    ts, abars, keys = KO.grid(AB, 4, KO.KARRAS)
    assert all(isinstance(t, np.float32) for t in ts)
    np.testing.assert_allclose([float(t) for t in ts], [999, 687.1533, 145.9392, 0], atol=1e-4)
    assert abars[-1] == 1.0 and keys == [0, 1, 2, 3]
    np.testing.assert_allclose(abars[:-1], [1 / (1 + s * s) for s in s4], rtol=0)
    ts20 = [float(t) for t in KO.grid(AB, 20, KO.KARRAS)[0]]
    np.testing.assert_allclose(ts20[:3], [999, 961.733, 921.042], atol=1e-3)
    np.testing.assert_allclose(ts20[-3:], [5.9918, 1.7829, 0], atol=1e-4)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 20, 50, 999, 1000])
def test_grid_is_monotone_between_the_table_ends(n):
    sig = KO.karras_sigma_table(AB)
    s = KO.karras_sigmas(AB, n)
    assert len(s) == n and s[0] == sig[999]
    if n > 1:
        assert s[-1] == sig[0]
    assert all(a > b for a, b in zip(s, s[1:]))
    ts, abars, _ = KO.grid(AB, n, KO.KARRAS)
    assert float(ts[0]) == 999.0 and (n == 1 or float(ts[-1]) == 0.0)
    assert all(a >= b for a, b in zip(ts, ts[1:])) and all(a < b for a, b in zip(abars, abars[1:]))
    assert all(0.0 <= float(t) <= 999.0 for t in ts)


def test_ddim_grid_is_the_reference_schedule():
    for n in (1, 4, 20, 50, 1000):
        ts, abars, keys = KO.grid(AB, n)
        want, _ = O.ddim_timesteps(n)
        assert ts == want and keys == want and abars == [float(AB[t]) for t in want] + [1.0]


def test_sigma_to_t():
    sig = KO.karras_sigma_table(AB)
    ls = [math.log(v) for v in sig]
    for j in (0, 1, 7, 500, 998, 999):
        assert KO.sigma_to_t(ls, sig[j]) == j
    assert KO.sigma_to_t(ls, sig[999]) == 999.0 and KO.sigma_to_t(ls, sig[0]) == 0.0
    # outside the table: clamped to the ends
    assert KO.sigma_to_t(ls, sig[999] * 2) == 999.0 and KO.sigma_to_t(ls, sig[0] / 2) == 0.0
    # t -> sigma (log-linear between neighbours) -> t
    for t in np.linspace(0.0, 999.0, 173):
        lo = min(int(t), 998)
        w = t - lo
        s = math.exp((1 - w) * ls[lo] + w * ls[lo + 1])
        assert abs(KO.sigma_to_t(ls, s) - t) < 1e-9


def test_step_loop_on_the_ddim_grid_is_the_sampler_oracle_loop():
    """schedule_oracle.step_loop on the DDIM grid is sampler_oracle.step_loop bit for bit (KERNEL arithmetic, every sampler, with
    and without the blend), so the Karras loop differs from it in the grid alone."""
    rng = np.random.default_rng(7)
    x = rng.standard_normal((2, 4, 8, 8)).astype(np.float32)
    w = rng.uniform(0, 1, (2, 1, 8, 8)).astype(np.float32)
    z0, eps = (rng.standard_normal((2, 4, 8, 8)).astype(np.float32) for _ in range(2))
    guide = lambda v, t: (np.asarray(v, np.float32) * np.float32(0.5 + t / 2000.0)).astype(np.float32)
    noise = lambda k, shape: synth.step_noise(11, k, shape)
    for kind, eta in ((SO.DDIM, 0.0), (SO.DDIM, 0.7), (SO.DPMPP_2M, 0.0)):
        for first, blend in ((0, None), (1, (w, z0, eps))):
            want = SO.step_loop(x, guide, AB, 4, SO.KERNEL, kind, eta, noise, first, blend)
            got = KO.step_loop(x, guide, AB, 4, SO.KERNEL, kind, eta, noise, first, blend, KO.SCHEDULE_DDIM)
            assert np.array_equal(got, want), (kind, eta, first)


# ------------------------------------------------------------------------------------------------ check and argument rules
def test_schedule_check_names_the_first_bad_index():
    KO.karras_sigma_table(AB)
    for j, v in ((0, 1.0), (0, 0.0), (5, float("nan")), (400, float("inf")), (999, -0.1)):
        a = AB.copy()
        a[j] = v
        with pytest.raises(ValueError, match=rf"alpha_cumulative_products\[{j}\]"):
            KO.karras_sigma_table(a)
    a = AB.copy()
    a[300] = a[299]  # not strictly decreasing
    with pytest.raises(ValueError, match=r"alpha_cumulative_products\[300\]"):
        KO.karras_sigma_table(a)
    # the DDIM grid takes any schedule the library accepts
    KO.grid(a, 4)


def test_argument_rules():
    for n in (1, 4, 20):
        assert KO.img2img_first(1.0, n) == 0
        with pytest.raises(ValueError, match=f"1/{n}"):
            KO.img2img_first(0.99 / n, n)
    assert KO.img2img_first(0.75, 4) == 1 and KO.img2img_first(0.5, 20) == 10
    for s in (0.0, -0.5, 1.01, float("nan")):
        with pytest.raises(ValueError, match="strength"):
            KO.img2img_first(s, 4)


# ------------------------------------------------------------------------------------------------ VP = VE
def _vp_guide(den, grid_ts, grid_abars):
    """step_loop's guide from a VE denoiser: x_VE = x / sqrt(a), x0 = den(x_VE, sigma), eps = (x - sqrt(a) x0) / sqrt(1 - a)."""
    a_of = {float(t): a for t, a in zip(grid_ts, grid_abars)}

    def guide(x, t):
        a = a_of[float(t)]
        x = np.asarray(x, np.float64)
        x0 = den(x / math.sqrt(a), math.sqrt((1.0 - a) / a))
        return torch.from_numpy((x - math.sqrt(a) * x0) / math.sqrt(1.0 - a))
    return guide


@pytest.mark.parametrize("n", [1, 4, 20, 50])
@pytest.mark.parametrize("sampler", [(SO.DDIM, 0.0), (SO.DDIM, 0.5), (SO.DDIM, 1.0), (SO.DPMPP_2M, 0.0)])
def test_vp_loop_is_the_ve_sampler(n, sampler):
    """step_loop's arithmetic on the Karras grid in float64 against Euler, Euler-ancestral(eta) and DPM++ 2M restated in VE
    variables, from x_VE = sqrt(1 + sigma_0^2) z with the same z_i, under the Gaussian problem's exact E[x0 | x] and under a
    random affine denoiser."""
    kind, eta = sampler
    rng = np.random.default_rng(n * 10 + int(eta * 4) + kind)
    z = rng.standard_normal(64)
    Z = rng.standard_normal((n, 64))
    sig = KO.karras_sigmas(AB, n)
    ts, abars, _ = KO.grid(AB, n, KO.KARRAS)
    g, c = rng.uniform(0.5, 1.5, 64), rng.standard_normal(64)
    dens = {"gaussian": lambda x, s: SO.gaussian_x0(x / math.sqrt(1 + s * s), 1 / (1 + s * s), 0.7, 0.3),
            "affine": lambda x, s: g * x / (1 + s) + c}
    arith = SO.oracle(torch.float64)
    for name, den in dens.items():
        vp = KO.step_loop(torch.from_numpy(z), _vp_guide(den, ts, abars), AB, n, arith, kind, eta, lambda k, shape: Z[k],
                          schedule=KO.KARRAS, dt=np.float64)
        ve = KO.ve_sample(kind, eta, math.sqrt(1 + sig[0] ** 2) * z, sig + [0.0], den, lambda i: Z[i])
        e = rel(np.asarray(vp), ve)
        assert e < 1e-12, (name, e)


# ------------------------------------------------------------------------------------------------ convergence order
def _solve_error(kind, abars, mu=0.7, s=0.3):
    x = np.linspace(-3.0, 3.0, 61)
    got = SO.gaussian_solve(kind, x.copy(), abars, mu, s)
    return float(np.abs(got - SO.gaussian_flow(x, abars[0], abars[-1], mu, s)).max())


@pytest.mark.parametrize("kind,lo,hi", [(SO.DDIM, 0.8, 1.2), (SO.DPMPP_2M, 1.8, None)])
def test_convergence_order_on_the_karras_grid(kind, lo, hi):
    """Gaussian data N(0.7, 0.3^2) from sigma_max to sigma_min (the same ends for every N): N + 1 Karras points, N steps, N = 8
    ... 256. The pair 8 -> 16 is printed, not gated: at N = 8 the grid's last step spans h = 1.15 in log-SNR (0.60 at N = 16),
    outside the asymptotic range, and DPM++'s observed order there is 1.07."""
    errs = []
    for n in (8, 16, 32, 64, 128, 256):
        abars = [1 / (1 + v * v) for v in KO.karras_sigmas(AB, n + 1)]
        errs.append(_solve_error(kind, abars))
    orders = [math.log2(errs[i] / errs[i + 1]) for i in range(len(errs) - 1)]
    print(f"kind {kind}: max error {errs[0]:.2e} -> {errs[-1]:.2e}, observed orders " + " ".join(f"{o:.2f}" for o in orders))
    assert all(o >= lo for o in orders[1:])
    if hi is not None:
        assert all(o <= hi for o in orders)


def test_dpmpp_error_on_both_grids():
    """Not a gate: DPM++(2M)'s global error over a whole run (to abar = 1) at N = 10, 15, 20, DDIM grid vs Karras grid."""
    for n in (10, 15, 20):
        e = {sch: _solve_error(SO.DPMPP_2M, KO.grid(AB, n, sch)[1]) for sch in (KO.SCHEDULE_DDIM, KO.KARRAS)}
        print(f"DPM++(2M) N = {n}: max error DDIM grid {e['ddim']:.3e}, Karras grid {e['karras']:.3e}")
        assert all(np.isfinite(v) for v in e.values())


# ------------------------------------------------------------------------------------------------ fixture
def test_fixture_inputs():
    g = np.load(GOLD)
    assert np.array_equal(g["noise"], synth.make_latent(2, 32, 32, seed=41))
    for k in ("ddim", "eta", "dpmpp", "inpaint"):
        assert g[f"{k}_latent"].shape == (2, 4, 32, 32) and g[f"{k}_u8"].shape == (2, 128, 128, 3)


def test_fixture_rederived():
    """The whole fixture from the oracle (a few minutes on 8 cores)."""
    import importlib.util
    torch.set_num_threads(os.cpu_count() or 1)
    spec = importlib.util.spec_from_file_location("make_schedule_golden", os.path.join(ROOT, "tests", "golden",
                                                                                       "make_schedule_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    g = np.load(GOLD)
    out = mk.compute(O.Params(synth.make_params(0)))
    for k in ("ddim", "eta", "dpmpp", "inpaint"):
        assert rel(out[f"{k}_latent"], g[f"{k}_latent"]) < 1e-4, k
        d = np.abs(out[f"{k}_u8"].astype(np.int16) - g[f"{k}_u8"].astype(np.int16))
        assert (d <= 1).mean() >= 0.999 and d.max() <= 2, k
