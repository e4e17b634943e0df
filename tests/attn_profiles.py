"""Attention inputs that drive the lazy online-softmax rescale of the fused attention kernel (csrc/attention.cu), and a numpy
replay of the kernel's rescale rule on them.

The kernel streams keys in sub-tiles (128 keys, or 64 for head dim 160) and keeps a per-row reference point m. It moves m, and
rescales O and l by alpha = 2^(m_old - m_new), only when a sub-tile's maximum logit (log2 units) exceeds m by more than a
threshold (attention.cu:218-221); otherwise the sub-tile is exponentiated against the stale m, so P may exceed 1. Standard-normal
q and k never grow a row's maximum that far after the first sub-tile, so these profiles place the logits on purpose.

Logits are built per (sample, head) along a seeded unit direction u of the head: q_i = d^1/4 (a_i u + r_i) and
k_j = d^1/4 (b_j u + w_j) with r_i, w_j orthogonal to u, so the natural-unit logit q_i.k_j / sqrt(d) = a_i b_j + r_i.w_j:
b_j sets the profile over the keys, a_i (per row) spreads the rows, and r_i.w_j is noise of standard deviation `tau`.
"""
import os
import re

import numpy as np

ATTENTION_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "stable_diffusion_burn_b200", "csrc",
                            "attention.cu")

# name -> (what the profile makes the kernel do, head dims it is run at)
PROFILES = {
    "ramp": ("the maximum grows ~7 (natural units) per sub-tile: every row rescales on every sub-tile", (40, 80, 160)),
    "creep": ("growth ~5 per sub-tile with per-row spread: rows alternate between rescaling and exponentiating against the stale "
              "reference (P > 128), and rows r / r + 8 of a 16-row group decide differently", (40, 80, 160)),
    "late_spike": ("one key of the (partial) last sub-tile sits +40 above the rest: O and l of all earlier keys scale by ~2^-58",
                   (40, 80, 160)),
    "early_peak": ("key 0 sits +40 above the rest: no later rescale, and every later P rounds to 0 in fp16", (40, 80, 160)),
    "subtile_spike": ("a spike in keys 64-127 of tile 0: the rescale happens between the two 64-key sub-tiles of head dim 160",
                      (160,)),
    "fp16_edge": ("a key of tile 1 sits just under 2^16 (log2 units) above tile 0's maximum, with exact logits: a threshold of 16 "
                  "would leave P = 2^15.9998, which rounds to inf in fp16", (40, 80, 160)),
}
HEADS = 2
NQ = 200  # not a multiple of the kernel's 128 query rows


def sub_tile_width(d):
    """keys per S sub-tile (KW in attention.cu): a 128-key tile, split in two for head dims above 128"""
    return 64 if d > 128 else 128


def num_keys(d):
    """4-6 key tiles, the last one partial"""
    return 500 if d > 128 else 700


def kernel_threshold():
    """the rescale threshold (log2 units) the kernel source uses"""
    src = open(ATTENTION_CU).read()
    m = re.search(r"const bool resc = m_cand > m_run\[hh\] \+ ([0-9.]+)f;", src)
    assert m, "rescale rule not found in attention.cu: update tests/attn_profiles.py with the kernel"
    return float(m.group(1))


def _fp16_edge(d, rng, n, Nk):
    """exact logits: q = [1, 2^-11, noise...], keys use channels 0 and 1 only (fp16 values) so every q.k is exact in fp32.
    Tile 0's maximum is 0 (key 0); key 128 + 37 has raw logit x with x * sl2 = 15.9998 as the kernel rounds sl2."""
    C = HEADS * d
    sl2 = np.float32(np.float32(1.0 / np.sqrt(d)) * np.float32(1.4426950408889634))
    x = 15.9998 / np.float64(sl2)
    k0 = np.float16(x)
    k1 = np.float16((x - np.float64(k0)) * 2048.0)
    q = np.zeros((n, NQ, C), np.float32)
    k = np.zeros((n, Nk, C), np.float32)
    for h in range(HEADS):
        c0 = h * d
        q[:, :, c0] = 1.0
        q[:, :, c0 + 1] = 2.0 ** -11
        q[:, :, c0 + 2:c0 + d] = rng.standard_normal((n, NQ, d - 2))  # meets only zero key channels
        k[:, :, c0] = -rng.uniform(0.0, 4.0, (n, Nk)).astype(np.float16)
        k[:, 0, c0] = 0.0
        k[:, 128 + 37, c0] = k0
        k[:, 128 + 37, c0 + 1] = k1
    return q, k


def make_case(profile, d, n=2, seed=0):
    """-> q [n, NQ, HEADS*d], k, v [n, Nk, HEADS*d] float32 for one profile of PROFILES."""
    assert d in PROFILES[profile][1], (profile, d)
    rng = np.random.default_rng([seed, d, list(PROFILES).index(profile)])
    Nk, KW, C = num_keys(d), sub_tile_width(d), HEADS * d
    v = rng.standard_normal((n, Nk, C)).astype(np.float32)
    if profile == "fp16_edge":
        q, k = _fp16_edge(d, rng, n, Nk)
        return q, k, v
    sub = np.arange(Nk) // KW
    a_lo, a_hi, tau = {"ramp": (0.9, 1.1, 0.05), "creep": (0.8, 1.25, 0.05)}.get(profile, (0.9, 1.1, 1.0))
    q = np.empty((n, NQ, C), np.float64)
    k = np.empty((n, Nk, C), np.float64)
    rho = np.sqrt(tau / np.sqrt(d))  # r.w of d terms of variance rho^4 -> standard deviation tau
    for s in range(n):
        for h in range(HEADS):
            u = rng.standard_normal(d)
            u /= np.linalg.norm(u)
            a = rng.uniform(a_lo, a_hi, NQ)
            b = np.zeros(Nk)
            if profile == "ramp":
                b = 7.0 * sub
            elif profile == "creep":
                b = 5.0 * sub
            elif profile == "late_spike":
                b[Nk - 3] = 40.0
            elif profile == "early_peak":
                b[0] = 40.0
            elif profile == "subtile_spike":
                b[100] = 40.0
            r = rng.standard_normal((NQ, d)) * rho
            w = rng.standard_normal((Nk, d)) * rho
            r -= np.outer(r @ u, u)
            w -= np.outer(w @ u, u)
            q[s, :, h * d:(h + 1) * d] = d ** 0.25 * (np.outer(a, u) + r)
            k[s, :, h * d:(h + 1) * d] = d ** 0.25 * (np.outer(b, u) + w)
    return q.astype(np.float32), k.astype(np.float32), v


def replay(q, k, heads, split, threshold=None):
    """The kernel's rescale rule (attention.cu:218-221) on the operands it consumes: q / k as given (split = True: the hi + lo
    pairs, fp32-class) or rounded to fp16. Logits are rounded to fp32 as the kernel accumulates them.
    -> (resc, growth, pmax), each [n, heads, Nq, sub-tiles]: whether the sub-tile moved the reference point, how far the
    sub-tile's maximum sits above the reference point it found (log2 units), and the largest P of the sub-tile before its
    fp16 rounding."""
    thr = np.float32(kernel_threshold() if threshold is None else threshold)
    n, Nq, C = q.shape
    Nk = k.shape[1]
    d = C // heads
    KW = sub_tile_width(d)
    nsub = (Nk + KW - 1) // KW
    sl2 = np.float32(np.float32(1.0 / np.sqrt(d)) * np.float32(1.4426950408889634))
    qq, kk = (np.float64(a if split else a.astype(np.float16)) for a in (q, k))
    resc = np.zeros((n, heads, Nq, nsub), bool)
    growth = np.zeros((n, heads, Nq, nsub))
    pmax = np.zeros((n, heads, Nq, nsub))
    for s in range(n):
        for h in range(heads):
            S = (qq[s, :, h * d:(h + 1) * d] @ kk[s, :, h * d:(h + 1) * d].T).astype(np.float32)
            m_run = np.full(Nq, -np.inf, np.float32)
            for t in range(nsub):
                St = S[:, t * KW:(t + 1) * KW]
                mx = (St.max(axis=1) * sl2).astype(np.float32)
                m_cand = np.maximum(m_run, mx)
                rs = m_cand > (m_run + thr).astype(np.float32)
                growth[s, h, :, t] = np.float64(mx) - np.float64(m_run)
                m_run = np.where(rs, m_cand, m_run)
                resc[s, h, :, t] = rs
                expo = (np.float64(St) * np.float64(sl2) - np.float64(m_run)[:, None]).astype(np.float32)
                pmax[s, h, :, t] = np.exp2(np.float64(expo)).max(axis=1)
    return resc, growth, pmax
