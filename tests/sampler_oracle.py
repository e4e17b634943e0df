"""CPU oracle of the samplers (DESIGN.md §7 f6): stochastic DDIM (eta) and DPM-Solver++(2M), and the one step loop of every
sampling oracle and step-exact host loop — TEST INFRASTRUCTURE ONLY.

The reference samples with DDIM at eta = 0 (oracle/sd_oracle.py: sample_latent). The per-step coefficients below are computed in
double exactly as the library's host loop computes them (csrc/model.cu: step_scalars) and rounded once to float32; the new
updates are evaluated in numpy float32, one rounding per operation, which is what the fused step's __f*_rn intrinsics compute.
step_loop walks the schedule for txt2img, img2img, 9-channel inpainting and editing alike: the caller's guide(x, t) gives each
step's prediction, and one of two arithmetics computes x0 and the eta = 0 update, oracle(dtype) (sample_latent's torch ops) or
KERNEL (the fused step's contractions). The update functions take explicit schedule values, so they also drive the closed-form
Gaussian problem the convergence-order test integrates (gaussian_*).
The fixture tests/golden/sampler_b2.npz is written by tests/golden/make_sampler_golden.py from SAMPLER_CASES.
"""
from __future__ import annotations

import collections
import functools
import math

import numpy as np
import torch

from oracle.sd_oracle import ddim_timesteps, encode_image, forward_diffuser
from stable_diffusion_burn_b200 import synth

import img2img_oracle as IO

DDIM, DPMPP_2M = 0, 1  # SDB_SAMPLER_DDIM, SDB_SAMPLER_DPMPP_2M


# ------------------------------------------------------------------------------------------------ request rules
def check_sampler(kind, eta):
    """The argument rules of sdb_set_sampler."""
    if kind not in (DDIM, DPMPP_2M):
        raise ValueError(f"unknown sampler kind {kind}")
    if not (math.isfinite(eta) and 0.0 <= eta <= 1.0):
        raise ValueError(f"eta {eta} must be finite and in [0, 1]")
    if kind == DPMPP_2M and eta != 0.0:
        raise ValueError(f"DPM-Solver++(2M) is deterministic; eta {eta} must be 0")


def img2img_start(strength, n_steps):
    """-> (first schedule index, ts): of the N timesteps of ddim_timesteps(n_steps), the last k = floor(strength * N) run.
    Rejects a strength that is not finite or not in (0, 1], and one that runs no step (below 1/N)."""
    ts, _ = ddim_timesteps(n_steps)
    N = len(ts)
    if not (math.isfinite(strength) and 0.0 < strength <= 1.0):
        raise ValueError("strength must be finite and in (0, 1]")
    k = int(math.floor(strength * N))
    if k == 0:
        raise ValueError(f"strength {strength} runs none of the {N} timesteps; the smallest valid strength is 1/{N}")
    return N - k, ts


def scaled_latent(enc):
    """fl(enc * 0.18215) in float32 (the latent scale of latent_to_image, stablediffusion/mod.rs:71): z0 of img2img and z_m of
    inpainting. enc is the encoder's output, the oracle's tensor or the library's array."""
    return np.multiply(np.asarray(enc, np.float32), np.float32(0.18215))


def start_latent(abar, z0, eps):
    """fl(fl(sqrt(abar) z0) + fl(sqrt(1 - abar) eps)) in float32, each factor rounded once to float32: img2img's start latent at
    abar[t0], and the known latent the blend pastes at abar'."""
    return np.add(np.multiply(np.float32(math.sqrt(abar)), z0), np.multiply(np.float32(math.sqrt(1.0 - abar)), eps))


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


# ------------------------------------------------------------------------------------------------ the step loop
# How a loop computes x0 and the eta = 0 update, and the latent type it keeps: latent(a) converts the start latent and the numpy
# results of the eta / DPM++ updates and of the blend.
Arithmetic = collections.namedtuple("Arithmetic", "x0 ddim latent")


def oracle(dtype):
    """sample_latent's arithmetic: torch ops on latents of `dtype`, one rounding per operation. x0 = (x - pred sqrt(1 - a)) /
    sqrt(a) and x' = x0 sqrt(a') + pred sqrt(1 - a') (sample_latent's sqrt(1 - a' - sigma^2) at sigma = 0: subtracting 0.0
    leaves every double as it is). Every other result is cast back to `dtype`."""
    return Arithmetic(lambda x, pred, a: (x - pred * math.sqrt(1.0 - a)) / math.sqrt(a),
                      lambda x0, pred, a: x0 * math.sqrt(a) + pred * math.sqrt(1.0 - a),
                      lambda v: torch.as_tensor(v).to(dtype))


def fma(a, b, c):
    """fl32(a b + c) with one rounding (the product of two float32 values is exact in float64)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


# The fused step's arithmetic (csrc/kernels.cu: cfg_step) on float32 numpy latents, with the contractions its SASS makes:
# x0 = fl(fma(-pred, sqrt(1 - a), x) / sqrt(a)) and the eta = 0 update fma(pred, sqrt(1 - a'), fl(x0 sqrt(a'))).
KERNEL = Arithmetic(lambda x, pred, a: np.divide(fma(-pred, np.float32(math.sqrt(1.0 - a)), x), np.float32(math.sqrt(a))),
                    lambda x0, pred, a: fma(pred, np.float32(math.sqrt(1.0 - a)), np.multiply(x0, np.float32(math.sqrt(a)))),
                    lambda v: np.asarray(v, np.float32))


def step_loop(x, guide, alphas, n_steps, arith, kind=DDIM, eta=0.0, noise=None, first=0, blend=None):
    """Sample from the latent x at ts[first] of ddim_timesteps(n_steps) -> the final latent. Per step t (a = abar[t], a' the
    next step's, 1 after the last step): pred = guide(x, t), x0 = arith.x0, then kind's update: arith.ddim at eta = 0,
    ddim_eta_update with z = noise(t, shape), or dpmpp_update with the history of the steps this call ran; the last two work on
    numpy arrays of the latents. alphas: abar per timestep, float32 values. blend = (w [n,1,H,W], z0, eps) keeps the known
    region after every step: x = fl(fl(w nl) + fl(fl(1 - w) known)) in float32, nl the new latent as float32 and known =
    start_latent(a', z0, eps)."""
    ts, step = ddim_timesteps(n_steps)
    x = arith.latent(x)
    x0_prev, h_prev = None, None
    for t in ts[first:]:
        a_t = float(alphas[t])
        a_next = float(alphas[t - step]) if t >= step else 1.0
        pred = guide(x, t)
        x0 = arith.x0(x, pred, a_t)
        if kind == DDIM and eta == 0.0:
            x = arith.ddim(x0, pred, a_next)
        elif kind == DDIM:
            s, dir_ = ddim_coefs(a_t, a_next, eta)
            x = arith.latent(ddim_eta_update(np.asarray(x0), np.asarray(pred), a_next, s, dir_, noise(t, tuple(x.shape))))
        else:
            cx, cd, c2, h = dpmpp_coefs(a_t, a_next, h_prev)
            x0 = np.asarray(x0)
            x = arith.latent(dpmpp_update(np.asarray(x), x0, x0_prev, cx, cd, c2))
            x0_prev, h_prev = x0, h
        if blend is not None:
            w, z0, eps = blend
            nl, known = np.asarray(x, np.float32), start_latent(a_next, z0, eps)
            x = arith.latent(np.add(np.multiply(w, nl), np.multiply(np.subtract(np.float32(1.0), w), known)))
    return x


# ------------------------------------------------------------------------------------------------ the full model
def guided_latent(P, n_steps, latent0, guide, kind=DDIM, eta=0.0, noise_seed=0, first=0, blend=None):
    """step_loop on P: its schedule, the oracle arithmetic in P's dtype and the step noise synth.step_noise(noise_seed, ...).
    pred = guide(latent, t) -> the final latent (torch)."""
    check_sampler(kind, eta)
    return step_loop(latent0, guide, P("alpha_cumulative_products").to(torch.float32), n_steps, oracle(P.dtype), kind, eta,
                     functools.partial(synth.step_noise, noise_seed), first, blend)


def sampler_latent(P, context, uncond, scale, n_steps, init_latent, kind=DDIM, eta=0.0, noise_seed=0, first=0, blend=None):
    """sample_latent (oracle/sd_oracle.py) under any sampler, from schedule index `first` on (img2img), with step_loop's blend.
    With kind = DDIM and eta = 0 every operation is sample_latent's own. -> latent (torch)."""
    return guided_latent(P, n_steps, init_latent, lambda x, t: forward_diffuser(P, x, t, context, uncond, scale), kind, eta,
                         noise_seed, first, blend)


def sampler_img2img_latent(P, context, uncond, scale, n_steps, image_u8, strength, noise, mask_u8=None, kind=DDIM, eta=0.0,
                           noise_seed=0, taps=None):
    """Image-to-image (mask_u8 None) or masked inpainting (DESIGN.md §7 f5) under any sampler -> the final latent [n,4,H,W]
    (torch). NOT a reference function: the reference has no img2img. z0 = scaled_latent(encode_image(x)), x the converted image;
    the run starts at ts[first] (img2img_start) from start_latent(abar[ts[first]], z0, noise [n,4,H,W]); with a mask step_loop
    blends toward z0 (w = mask_to_latent). taps receives "z0" and, with a mask, "w"."""
    first, ts = img2img_start(strength, n_steps)
    a0 = float(P("alpha_cumulative_products").to(torch.float32)[ts[first]])
    z0 = scaled_latent(encode_image(P, torch.from_numpy(IO.image_u8_to_float(image_u8))))
    eps = np.asarray(noise, np.float32)
    w = None if mask_u8 is None else IO.mask_to_latent(mask_u8)[:, None]
    if taps is not None:
        taps["z0"] = z0
        if w is not None:
            taps["w"] = w[:, 0]
    blend = None if w is None else (w, z0, eps)
    return sampler_latent(P, context, uncond, scale, n_steps, start_latent(a0, z0, eps), kind, eta, noise_seed, first, blend)


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
