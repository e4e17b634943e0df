"""CPU oracle of the samplers (DESIGN.md §7 f6): stochastic DDIM (eta) and DPM-Solver++(2M) — TEST INFRASTRUCTURE ONLY.

The reference samples with DDIM at eta = 0 (oracle/sd_oracle.py: sample_latent). The per-step coefficients below are computed in
double exactly as the library's host loop computes them (csrc/model.cu: step_scalars) and rounded once to float32; the new
updates are evaluated in numpy float32, one rounding per operation, which is what the fused step's __f*_rn intrinsics compute.
The solvers take an explicit list of schedule values, so the same step functions drive the full model (sampler_latent) and
the closed-form Gaussian problem the convergence-order test integrates (gaussian_*).
The fixture tests/golden/sampler_b2.npz is written by tests/golden/make_sampler_golden.py from SAMPLER_CASES.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle.sd_oracle import ddim_timesteps, encode_image, forward_diffuser
from stable_diffusion_burn_b200 import synth

import img2img_oracle as IO

DDIM, DPMPP_2M = 0, 1  # SDB_SAMPLER_DDIM, SDB_SAMPLER_DPMPP_2M


def check_sampler(kind, eta):
    """The argument rules of sdb_set_sampler."""
    if kind not in (DDIM, DPMPP_2M):
        raise ValueError(f"unknown sampler kind {kind}")
    if not (math.isfinite(eta) and 0.0 <= eta <= 1.0):
        raise ValueError(f"eta {eta} must be finite and in [0, 1]")
    if kind == DPMPP_2M and eta != 0.0:
        raise ValueError(f"DPM-Solver++(2M) is deterministic; eta {eta} must be 0")


# ------------------------------------------------------------------------------------------------ per-step coefficients
def ddim_coefs(a_t, a_next, eta):
    """-> (s, dir): x' = sqrt(a') x0 + dir eps + s z with s = eta sqrt((1-a')/(1-a)) sqrt(1 - a/a') (Song et al. 2021, eq. 16),
    dir = sqrt(1 - a' - s^2) (clamped at 0 against rounding). a' = 1 (the final step) gives s = 0."""
    s = eta * math.sqrt((1.0 - a_next) / (1.0 - a_t)) * math.sqrt(1.0 - a_t / a_next)
    return s, math.sqrt(max(0.0, 1.0 - a_next - s * s))


def dpmpp_coefs(a_t, a_next, h_prev):
    """DPM-Solver++(2M) (Lu et al. 2022), data prediction: x' = cx x + cd D, D = x0 (first order) or (1 + c2) x0 - c2 x0_prev
    with c2 = 1/(2r), r = h_prev / h (second order, when h_prev is not None). -> (cx, cd, c2 or None, h). lambda = ln(alpha /
    sigma), h = lambda' - lambda, cx = sigma'/sigma, cd = -alpha' expm1(-h). a' = 1 (sigma' = 0, h = inf): x' = x0, h None."""
    if a_next == 1.0:
        return 0.0, 1.0, None, None
    lam = math.log(math.sqrt(a_t) / math.sqrt(1.0 - a_t))
    lam_next = math.log(math.sqrt(a_next) / math.sqrt(1.0 - a_next))
    h = lam_next - lam
    cx = math.sqrt(1.0 - a_next) / math.sqrt(1.0 - a_t)
    cd = -math.sqrt(a_next) * math.expm1(-h)
    c2 = None if h_prev is None else 1.0 / (2.0 * (h_prev / h))
    return cx, cd, c2, h


def ddim_eta_update(x0, pred, a_next, s, dir_, z, dt=np.float32):
    """fl(fl(fl(sqrt(a') x0) + fl(dir pred)) + fl(s z))"""
    c = lambda v: dt(v)
    return np.add(np.add(np.multiply(c(math.sqrt(a_next)), x0), np.multiply(c(dir_), pred)), np.multiply(c(s), z))


def dpmpp_update(x, x0, x0_prev, cx, cd, c2, dt=np.float32):
    """D = x0 or fl(fl(c1 x0) - fl(c2 x0_prev)), c1 = fl(1 + c2); x' = fl(fl(cx x) + fl(cd D))"""
    c = lambda v: dt(v)
    d = x0 if c2 is None else np.subtract(np.multiply(c(1.0 + c2), x0), np.multiply(c(c2), x0_prev))
    return np.add(np.multiply(c(cx), x), np.multiply(c(cd), d))


# ------------------------------------------------------------------------------------------------ the full model
def sampler_latent(P, context, uncond, scale, n_steps, init_latent, kind=DDIM, eta=0.0, noise_seed=0, first=0, blend=None):
    """sample_latent (oracle/sd_oracle.py) under any sampler, from schedule index `first` on (img2img). With kind = DDIM and
    eta = 0 every operation is sample_latent's own. blend = (w [n,1,H,W], z0, eps0) applies the img2img keep-mask after every
    step, x = fl(fl(w nl) + fl(fl(1 - w) known)), known = fl(fl(sqrt(a') z0) + fl(sqrt(1 - a') eps0)). -> latent (torch)."""
    check_sampler(kind, eta)
    alphas = P("alpha_cumulative_products").to(torch.float32)
    ts, step = ddim_timesteps(n_steps)
    latent = init_latent.to(P.dtype)
    x0_prev, h_prev = None, None
    for t in ts[first:]:
        a_t = float(alphas[t])
        a_prev = float(alphas[t - step]) if t >= step else 1.0
        sqrt_noise = math.sqrt(1.0 - a_t)
        pred = forward_diffuser(P, latent, t, context, uncond, scale)
        predx0 = (latent - pred * sqrt_noise) / math.sqrt(a_t)
        if kind == DDIM and eta == 0.0:
            dir_latent = pred * math.sqrt(1.0 - a_prev - 0.0 * 0.0)
            latent = predx0 * math.sqrt(a_prev) + dir_latent
        elif kind == DDIM:
            s, dir_ = ddim_coefs(a_t, a_prev, eta)
            z = synth.step_noise(noise_seed, t, tuple(latent.shape))
            latent = torch.from_numpy(ddim_eta_update(predx0.numpy(), pred.numpy(), a_prev, s, dir_, z))
        else:
            cx, cd, c2, h = dpmpp_coefs(a_t, a_prev, h_prev)
            x0 = predx0.numpy()
            latent = torch.from_numpy(dpmpp_update(latent.numpy(), x0, x0_prev, cx, cd, c2))
            x0_prev, h_prev = x0, h
        if blend is not None:
            w, z0, eps = blend
            ka, kb = np.float32(math.sqrt(a_prev)), np.float32(math.sqrt(1.0 - a_prev))
            known = np.add(np.multiply(ka, z0), np.multiply(kb, eps))
            nl = latent.to(torch.float32).numpy()
            latent = torch.from_numpy(np.add(np.multiply(w, nl), np.multiply(np.subtract(np.float32(1.0), w), known))).to(P.dtype)
    return latent


def sampler_img2img_latent(P, context, uncond, scale, n_steps, image_u8, strength, noise, mask_u8=None, kind=DDIM, eta=0.0,
                           noise_seed=0):
    """img2img / masked inpainting (tests/img2img_oracle.py: img2img_latent) under any sampler: the same start latent and blend."""
    alphas = P("alpha_cumulative_products").to(torch.float32)
    first, ts = IO.img2img_start(strength, n_steps)
    z0 = np.multiply(encode_image(P, torch.from_numpy(IO.image_u8_to_float(image_u8))).to(torch.float32).numpy(),
                     np.float32(0.18215))
    eps = np.asarray(noise, np.float32)
    a0 = float(alphas[ts[first]])
    start = np.add(np.multiply(np.float32(math.sqrt(a0)), z0), np.multiply(np.float32(math.sqrt(1.0 - a0)), eps))
    blend = None if mask_u8 is None else (IO.mask_to_latent(mask_u8)[:, None], z0, eps)
    return sampler_latent(P, context, uncond, scale, n_steps, torch.from_numpy(start), kind, eta, noise_seed, first, blend)


# ------------------------------------------------------------------------------------------------ closed-form Gaussian problem
# Data x0 ~ N(mu, s^2) under VP noising x = alpha x0 + sigma eps: E[x0 | x] and the probability-flow ODE map between two noise
# levels are affine, so a solver's global error can be measured exactly (float64).
def gaussian_x0(x, a, mu, s):
    """E[x0 | x] at abar = a: mu + alpha s^2 / (alpha^2 s^2 + sigma^2) (x - alpha mu)."""
    al = math.sqrt(a)
    return mu + al * s * s / (a * s * s + (1.0 - a)) * (x - al * mu)


def gaussian_flow(x, a_from, a_to, mu, s):
    """The exact probability-flow ODE map: (x - alpha mu) / sqrt(alpha^2 s^2 + sigma^2) is constant along a trajectory."""
    sd = lambda a: math.sqrt(a * s * s + (1.0 - a))
    return math.sqrt(a_to) * mu + sd(a_to) / sd(a_from) * (x - math.sqrt(a_from) * mu)


def gaussian_solve(kind, x, abars, mu, s):
    """Integrate from abars[0] to abars[-1] (ascending abar, i.e. descending t) with the deterministic sampler `kind` in float64,
    the denoiser being the exact E[x0 | x]."""
    x0_prev, h_prev = None, None
    for a_t, a_next in zip(abars[:-1], abars[1:]):
        x0 = gaussian_x0(x, a_t, mu, s)
        if kind == DDIM:
            eps = (x - math.sqrt(a_t) * x0) / math.sqrt(1.0 - a_t)
            _, dir_ = ddim_coefs(a_t, a_next, 0.0)
            x = math.sqrt(a_next) * x0 + dir_ * eps
        else:
            cx, cd, c2, h = dpmpp_coefs(a_t, a_next, h_prev)
            x = dpmpp_update(x, x0, x0_prev, cx, cd, c2, dt=np.float64)
            x0_prev, h_prev = x0, h
    return x


def nested_grid(n):
    """t = round(linspace(999, 99, n + 1)): the same endpoints for every n (nested for n = 9, 18, 36, ...)."""
    return [int(v) for v in np.rint(np.linspace(999, 99, n + 1))]


# ------------------------------------------------------------------------------------------------ fixture
SAMPLER_CASES = dict(n_steps=4, scale=5.0, eta=0.7, noise_seed=11, strength=0.75)
