"""CPU oracle of the Karras schedule (DESIGN.md §7 f15) — TEST INFRASTRUCTURE ONLY.

The grid (k-diffusion's get_sigmas_karras and sigma_to_t, in double exactly as csrc/model.cu: sample_grid computes it) and the
step loop on either grid, with sampler_oracle's update arithmetic; what the full-model oracle needs to run there: the UNet at a
real timestep (oracle/sd_oracle.py embeds int(t), the reference's Int timestep) and the txt2img / img2img runs of the schedule_b2
fixture. It also restates the three k-diffusion samplers in their own
variance-exploding (VE) variables, x_VE = x / sqrt(abar), sigma = sqrt((1 - abar) / abar), as published (k-diffusion:
sample_euler, sample_euler_ancestral, sample_dpmpp_2m), for the VP = VE test.
The fixture tests/golden/schedule_b2.npz is written by tests/golden/make_schedule_golden.py.
"""
from __future__ import annotations

import contextlib
import functools
import math

import numpy as np
import torch

from oracle import sd_oracle as O
from stable_diffusion_burn_b200 import synth

import img2img_oracle as IO
import sampler_oracle as SO

SCHEDULE_DDIM, KARRAS = "ddim", "karras"  # SDB_SCHEDULE_DDIM, SDB_SCHEDULE_KARRAS


# ------------------------------------------------------------------------------------------------ the grids
def karras_sigma_table(alphas):
    """sigma_j = sqrt((1 - abar_j) / abar_j) in float64, abar read as float32 and widened. Rejects a schedule that is not finite,
    in (0, 1) and strictly decreasing, naming the first bad index (the library's check)."""
    a = np.asarray(alphas, np.float32).astype(np.float64)
    for j, v in enumerate(a):
        if not (math.isfinite(v) and 0.0 < v < 1.0 and (j == 0 or v < a[j - 1])):
            raise ValueError(f"alpha_cumulative_products[{j}] = {v!r}: every value must be finite, in (0, 1) and below the one "
                             "before it")
    return [math.sqrt((1.0 - v) / v) for v in a]


def sigma_to_t(log_sigmas, sigma):
    """k-diffusion's sigma_to_t in float64: linear in log sigma between table neighbours, the low index the largest j with
    log sigma_j <= log sigma, clamped to [0, len - 2], w clamped to [0, 1]."""
    ls = math.log(sigma)
    lo = 0
    for j, v in enumerate(log_sigmas):
        if v <= ls:
            lo = j
    lo = min(lo, len(log_sigmas) - 2)
    w = min(1.0, max(0.0, (log_sigmas[lo] - ls) / (log_sigmas[lo] - log_sigmas[lo + 1])))
    return (1.0 - w) * lo + w * (lo + 1)


def karras_sigmas(alphas, n_steps):
    """k-diffusion's get_sigmas_karras at rho = 7 between sigma_max = sigma_999 and sigma_min = sigma_0 (the ends exactly), the
    N = n_steps values without the final 0, in float64."""
    sig = karras_sigma_table(alphas)
    smax, smin = sig[999], sig[0]
    rmax, rmin = math.pow(smax, 1.0 / 7.0), math.pow(smin, 1.0 / 7.0)
    out = []
    for i in range(n_steps):
        out.append(smax if i == 0 else smin if i == n_steps - 1 else math.pow(rmax + i / (n_steps - 1) * (rmin - rmax), 7.0))
    return out


def grid(alphas, n_steps, schedule=SCHEDULE_DDIM):
    """-> (ts, abars, keys): the timestep each step evaluates the UNet at, abar per step plus 1 after the last, and the key of
    each step's eta noise. DDIM grid: ddim_timesteps, abar = alphas[t], key t. Karras grid: t_i = fl32(sigma_to_t(sigma_i)),
    abar_i = 1 / (1 + sigma_i^2), key i."""
    if schedule == SCHEDULE_DDIM:
        ts, _ = O.ddim_timesteps(n_steps)
        return ts, [float(alphas[t]) for t in ts] + [1.0], ts
    sig = karras_sigmas(alphas, n_steps)
    ls = [math.log(v) for v in karras_sigma_table(alphas)]
    ts = [np.float32(sigma_to_t(ls, s)) for s in sig]
    return ts, [1.0 / (1.0 + s * s) for s in sig] + [1.0], list(range(n_steps))


def step_loop(x, guide, alphas, n_steps, arith, kind=SO.DDIM, eta=0.0, noise=None, first=0, blend=None, schedule=KARRAS,
              dt=np.float32):
    """sampler_oracle.step_loop on either grid: from the latent x at step `first` -> the final latent. Per step (a = abar of the
    step, a' the next step's, 1 after the last): pred = guide(x, t), x0 = arith.x0, then kind's update (arith.ddim at eta = 0,
    ddim_eta_update with z = noise(key, shape), dpmpp_update with the history of the steps this call ran) and blend as
    sampler_oracle.step_loop does. The grid, the abar values and the noise keys: see grid. dt: the type the eta and DPM++
    coefficients are rounded to (float64 restates the updates exactly). On the DDIM grid with dt = float32 this is
    sampler_oracle.step_loop."""
    ts, abars, keys = grid(alphas, n_steps, schedule)
    x = arith.latent(x)
    x0_prev, h_prev = None, None
    for i in range(first, len(ts)):
        a_t, a_next = abars[i], abars[i + 1]
        pred = guide(x, ts[i])
        x0 = arith.x0(x, pred, a_t)
        if kind == SO.DDIM and eta == 0.0:
            x = arith.ddim(x0, pred, a_next)
        elif kind == SO.DDIM:
            s, dir_ = SO.ddim_coefs(a_t, a_next, eta)
            z = noise(keys[i], tuple(x.shape))
            x = arith.latent(SO.ddim_eta_update(np.asarray(x0), np.asarray(pred), a_next, s, dir_, z, dt))
        else:
            cx, cd, c2, h = SO.dpmpp_coefs(a_t, a_next, h_prev)
            x0 = np.asarray(x0)
            x = arith.latent(SO.dpmpp_update(np.asarray(x), x0, x0_prev, cx, cd, c2, dt))
            x0_prev, h_prev = x0, h
        if blend is not None:
            w, z0, eps = blend
            nl, known = np.asarray(x, np.float32), SO.start_latent(a_next, z0, eps)
            x = arith.latent(np.add(np.multiply(w, nl), np.multiply(np.subtract(np.float32(1.0), w), known)))
    return x


# ------------------------------------------------------------------------------------------------ the UNet at a real t
@contextlib.contextmanager
def embedding_at(t):
    """Within the block, O.unet_forward embeds the float32 timestep t, whatever t it is given: [cos | sin](fl32(t) freqs) with
    O.timestep_embedding's freqs — the library's real-timestep embedding. Outside it the oracle is the reference's."""
    base = O.timestep_embedding

    def emb(_t, dim=320, max_period=10000, dtype=torch.float32):
        half = dim // 2
        freqs = (torch.arange(0, half, dtype=torch.int64).to(dtype) * (-math.log(max_period) / half)).exp()
        args = torch.tensor([float(np.float32(t))], dtype=torch.float32).to(dtype) * freqs
        return torch.cat([args.cos(), args.sin()], 0).unsqueeze(0)

    O.timestep_embedding = emb
    try:
        yield
    finally:
        O.timestep_embedding = base


def unet_forward_at(P, x, t, context):
    with embedding_at(t):
        return O.unet_forward(P, x, 0, context)


def img2img_first(strength, n_steps):
    """The step img2img starts from on the Karras grid: the last k = floor(strength * N) of its N = n_steps steps run."""
    if not (math.isfinite(strength) and 0.0 < strength <= 1.0):
        raise ValueError("strength must be finite and in (0, 1]")
    k = int(math.floor(strength * n_steps))
    if k == 0:
        raise ValueError(f"strength {strength} runs none of the {n_steps} timesteps; the smallest valid strength is 1/{n_steps}")
    return n_steps - k


# ------------------------------------------------------------------------------------------------ the full model
def karras_latent(P, context, uncond, scale, n_steps, latent0, kind=SO.DDIM, eta=0.0, noise_seed=0, first=0, blend=None):
    """sampler_oracle.sampler_latent on the Karras grid (step_loop): forward_diffuser at each step's real timestep, the oracle
    arithmetic in P's dtype, eta noise synth.step_noise(noise_seed, i) keyed by the grid index i. -> the final latent (torch)."""
    SO.check_sampler(kind, eta)

    def guide(x, t):
        with embedding_at(t):
            return O.forward_diffuser(P, x, 0, context, uncond, scale)

    return step_loop(latent0, guide, P("alpha_cumulative_products").to(torch.float32), n_steps, SO.oracle(P.dtype), kind, eta,
                     functools.partial(synth.step_noise, noise_seed), first, blend, KARRAS)


def karras_img2img_latent(P, context, uncond, scale, n_steps, image_u8, strength, noise, mask_u8=None, kind=SO.DDIM, eta=0.0,
                          noise_seed=0):
    """sampler_oracle.sampler_img2img_latent on the Karras grid: the start sqrt(abar_i0) z0 + sqrt(1 - abar_i0) noise at
    i0 = img2img_first(strength, N), the blend toward z0 at abar_{i+1}."""
    first = img2img_first(strength, n_steps)
    _, abars, _ = grid(P("alpha_cumulative_products").to(torch.float32), n_steps, KARRAS)
    z0 = SO.scaled_latent(O.encode_image(P, torch.from_numpy(IO.image_u8_to_float(image_u8))))
    eps = np.asarray(noise, np.float32)
    blend = None if mask_u8 is None else (IO.mask_to_latent(mask_u8)[:, None], z0, eps)
    return karras_latent(P, context, uncond, scale, n_steps, SO.start_latent(abars[first], z0, eps), kind, eta, noise_seed, first,
                         blend)


# ------------------------------------------------------------------------------------------------ the samplers in VE variables
def ve_sample(kind, eta, x_ve, sigmas, denoise, noise):
    """k-diffusion's samplers on sigmas [sigma_0, ..., sigma_{N-1}, 0] in float64, x_VE = x0 + sigma eps, denoise(x, sigma) ->
    x0, noise(i) -> z_i:
      sample_euler               d = (x - D) / sigma, x += d (sigma' - sigma)
      sample_euler_ancestral     sigma_up = min(sigma', eta sqrt(sigma'^2 (sigma^2 - sigma'^2) / sigma^2)),
                                 sigma_down = sqrt(sigma'^2 - sigma_up^2), x += d (sigma_down - sigma), then + z sigma_up
      sample_dpmpp_2m            t = -ln sigma, h = t' - t, x = (sigma'/sigma) x - expm1(-h) D', D' = D on the first and the final
                                 step, else (1 + 1/(2r)) D - 1/(2r) D_prev with r = h_prev / h."""
    x = np.asarray(x_ve, np.float64)
    old, h_last = None, None
    for i in range(len(sigmas) - 1):
        s, sn = sigmas[i], sigmas[i + 1]
        den = denoise(x, s)
        if kind == SO.DDIM:
            up = min(sn, eta * math.sqrt(sn * sn * (s * s - sn * sn) / (s * s))) if eta else 0.0
            down = math.sqrt(sn * sn - up * up)
            x = x + (x - den) / s * (down - s)
            if sn > 0 and up > 0:
                x = x + noise(i) * up
        else:
            t, tn = -math.log(s), (math.inf if sn == 0 else -math.log(sn))
            h = tn - t
            if old is None or sn == 0:
                d = den
            else:
                r = h_last / h
                d = (1 + 1 / (2 * r)) * den - (1 / (2 * r)) * old
            x = (sn / s) * x - math.expm1(-h) * d
            old, h_last = den, h
    return x
