"""Exact references for the split-fp16 GEMM (gemm_tc.cu) and its dispatch policy restated in Python.

* Lo-visible operands: every element is x = s (1 + j 2^-13), s = +-1, j in {0, 1, 2, 3}. It splits exactly into hi = s and
  lo = s j 2^-13, so the lo halves are non-zero, and every product the kernel forms (hi hi, lo hi, hi lo) is a multiple of 2^-13.
  With K <= 1536 the sum of |terms| stays below 2^11, so every fp32 partial sum is exact in any order and each pass count has
  one exact result: 1 pass hi hi; 2 passes + lo(A) hi(B); 3 passes + hi(A) lo(B) (lo lo is never formed).
* split_pair: numpy emulation of the device's fp32 -> fp16 hi + lo split (common.cuh: split_f16x2).
* pick_bn / pick_stages / pick_split: run_gemm's tile width and split-K rule and gemm_tc.cu's stage count, restated so that a
  test can name the kernel instance a shape reaches from the device's SM count, and assert the launch trace agrees.
* INSTANCES: every (BN, passes, epilogue) instance that gemm_tc.cu's launch_inst can build.
"""
import numpy as np

LO_STEP = 2.0 ** -13
LO_MAX_K = 1536  # K * max |term| < 2^11: fp32 partial sums of multiples of 2^-13 stay exact


def lo_visible(shape, seed):
    """x = s (1 + j 2^-13) in fp32 (exact), s = +-1 and j in {0..3} drawn independently."""
    rng = np.random.default_rng(seed)
    s = rng.choice(np.array([-1.0, 1.0]), shape)
    j = rng.integers(0, 4, shape).astype(np.float64)
    return (s * (1.0 + j * LO_STEP)).astype(np.float32)


def split_pair(x):
    """fp32 -> (hi, lo) fp16 pair as the device splits it, returned as float32 arrays: a finite x saturates both halves (hi at
    +-65504, the pair at +-131008), lo = fp16(clip(x) - hi) computed in fp32; +-inf and NaN give NaN in both halves."""
    x = np.asarray(x, np.float32)
    fin = np.isfinite(x)
    with np.errstate(invalid="ignore", over="ignore"):
        hi = np.where(fin, np.clip(x, -65504, 65504), np.nan).astype(np.float16).astype(np.float32)
        lo = np.where(fin, np.clip(x, -131008, 131008).astype(np.float32) - hi, np.nan).astype(np.float16).astype(np.float32)
    return hi, lo


def pass_product(a, w, passes):
    """The exact fp64 sum of the terms a `passes`-pass product forms from the fp16 splits of a [M, K] and w [K, N]."""
    ah, al = (v.astype(np.float64) for v in split_pair(a))
    wh, wl = (v.astype(np.float64) for v in split_pair(w))
    out = ah @ wh
    if passes >= 2:
        out = out + al @ wh
    if passes >= 3:
        out = out + ah @ wl
    return out


def rounded_operands(a, w, passes):
    """The operand values a `passes`-pass product effectively multiplies: fp16 A for 1 pass, fp16 W below 3 passes."""
    f16 = lambda v: np.asarray(v, np.float32).astype(np.float16).astype(np.float32)
    return (f16(a) if passes == 1 else a), (f16(w) if passes < 3 else w)


# ------------------------------------------------------------------ dispatch policy (runtime.cu: run_gemm, gemm_tc.cu)
EPIS = ("PLAIN", "GN", "LNS", "LNC", "GEGLU", "GEGLU_LNC")
BNS = (64, 128, 160, 256)
SMEM_OPTIN = 227 * 1024


def builds(bn, epi):
    """launch_inst: the epilogues each tile width is built with."""
    if epi == "PLAIN":
        return True
    if epi in ("GEGLU", "GEGLU_LNC"):
        return bn == 128
    if epi == "GN":
        return bn >= 128
    if epi == "LNS":
        return bn == 160
    if epi == "LNC":
        return bn in (128, 160)
    raise ValueError(epi)


def pick_stages(bn, passes):
    """pick_stages: as many stages of (A hi [, A lo], B hi [, B lo]) tiles as fit in the opt-in shared memory, at most 8."""
    per = (2 if passes >= 2 else 1) * 128 * 64 * 2 + (2 if passes >= 3 else 1) * bn * 64 * 2
    return min((SMEM_OPTIN - 1024) // (per + 16), 8)


def pick_bn(N, m_tiles, sms, geglu=False, ln_out=False):
    if geglu:
        return 128
    if ln_out:
        assert N % 160 == 0
        return 160
    if N % 160 == 0:
        return 160
    if N % 256 == 0 and m_tiles * (N // 256) >= 2 * sms:
        return 256
    return 128 if N % 128 == 0 else 64


def pick_split(m_tiles, n_tiles, iters, sms, splittable=True):
    """split-K: only a grid of at most half the SMs with at least 32 k-chunks; the CTAs stay within one wave, every split
    keeps >= 8 chunks, at most 16 splits, and no split owns an empty K range."""
    split = 1
    ctas = m_tiles * n_tiles
    if splittable and ctas <= sms // 2 and iters >= 32:
        split = max(min(sms // ctas, iters // 8, 16), 1)
    if split > 1:
        per = -(-iters // split)
        split = -(-iters // per)
    return split


def linear_instance(M, K, N, sms, passes):
    """(BN, stages, split) that a plain Linear M x K x N reaches."""
    m_tiles = -(-M // 128)
    bn = pick_bn(N, m_tiles, sms)
    return bn, pick_stages(bn, passes), pick_split(m_tiles, -(-N // bn), K // 64, sms)


def epi_of(roles):
    """The gemm_tc EPI instance an epilogue-role set (trace "epi") selects in launch_inst."""
    if "geglu" in roles:
        return "GEGLU_LNC" if "lnc" in roles else "GEGLU"
    for r, e in (("gn", "GN"), ("lns", "LNS"), ("lnc", "LNC")):
        if r in roles:
            return e
    return "PLAIN"


# every instance launch_inst can build: (BN, passes, EPI)
INSTANCES = [(bn, p, e)
             for bn, epis in ((128, ("PLAIN", "GN", "LNC", "GEGLU", "GEGLU_LNC")), (160, ("PLAIN", "GN", "LNS", "LNC")),
                              (256, ("PLAIN", "GN")), (64, ("PLAIN",)))
             for e in epis for p in (1, 2, 3)]


def bn256_rows(sms):
    """Rows of a Linear whose N = 1024 takes 256-wide tiles (m_tiles * 4 >= 2 * SMs), the last 128-row tile masked."""
    m_tiles = -(-sms // 2)
    return (m_tiles - 1) * 128 + 72


def find_split_shape(target, sms, N, bn):
    """The smallest (M, K) of an N-wide Linear (tiles of width bn) that the split rule maps to `target` splits, the last M tile
    masked. None if no shape up to 256 k-chunks does."""
    best = None
    n_tiles = -(-N // bn)
    for m_tiles in range(1, sms // 2 + 1):
        for iters in range(32, 257):
            if pick_split(m_tiles, n_tiles, iters, sms) == target:
                cost = m_tiles * iters
                if best is None or cost < best[0]:
                    best = (cost, m_tiles * 128 - 40, iters * 64)
                break
    return None if best is None else best[1:]
