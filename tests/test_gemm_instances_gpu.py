"""Every gemm_tc kernel instance, reached on purpose and checked against an exact or fp64 reference.

* The instance table (gemm_ref.INSTANCES): the 36 (tile width, passes, epilogue) instances launch_inst builds. Each one is reached
  by a named case through one of the GEMM test entries, whose launch trace must show that tile width, stage count, pass count and
  epilogue, with split = 1. The plain instances run lo-visible operands (gemm_ref.py), so the result must equal the exact sum of
  the terms the pass count forms, bit for bit; the statistics and GEGLU epilogues are checked at the fp64 bars of their own tests,
  on a K that wraps their ring.
* The split-K fold, exact: integer operands, shapes that the split rule (restated from the device's SM count) maps to 2, 3, 4,
  5, 8, 9 and 16 splits, i.e. every remainder of the fold's four-at-a-time loop. Bias plus fp32 residual, and the fp16 pair
  output, whose hi and lo must equal the split of the exact result; one 64-wide tile case; and the tickets must clean themselves
  (the same shape twice around another one gives bit-identical results).
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gemm_ref as G

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def rnd(shape, seed, scale=1.0):
    return (np.random.default_rng(seed).standard_normal(shape) * scale).astype(np.float32)


def gelu_erf(x):
    return 0.5 * x * (1.0 + np.vectorize(math.erf)(x / math.sqrt(2.0)))


def assert_reached(g, bn, passes, epi, split=1):
    assert (g["BN"], g["stages"], g["passes"], g["split"], G.epi_of(g["epi"])) == (bn, G.pick_stages(bn, passes), passes, split, epi)


# ------------------------------------------------------------------ the instance table
# the case that reaches each (BN, EPI), at every pass count
CASES = {
    "PLAIN": "test_linear, lo-visible operands, K = 1536 (24 k-chunks), N = 96 / 384 / 320 / 1024 (1024 with rows that fill the SMs)",
    (128, "GN"): "test_conv_groupnorm, 3x3 conv 64 -> 128 channels on 32 x 32 (9 k-chunks)",
    (160, "GN"): "test_conv_groupnorm, 3x3 conv 64 -> 320 channels on 32 x 32 (9 k-chunks)",
    (256, "GN"): "test_conv_groupnorm, 1x1 conv 320 -> 256 channels over 256 x 256 pixels (5 k-chunks)",
    (160, "LNS"): "test_ln_fold producer, K0 = C = 640 (10 k-chunks), consumer N = 384",
    (128, "LNC"): "test_ln_fold consumer, C = 640 (10 k-chunks), N = 384",
    (160, "LNC"): "test_ln_fold consumer, C = 640 (10 k-chunks), N = 320",
    (128, "GEGLU"): "test_gemm_ex GEGLU, K = 640 (10 k-chunks), N = 512",
    (128, "GEGLU_LNC"): "test_ln_fold GEGLU consumer, C = 640 (10 k-chunks), N = 512",
}
PLAIN_N = {64: 96, 128: 384, 160: 320, 256: 1024}
GN_CASES = {128: (1, 64, 32, 32, 128, 3), 160: (1, 64, 32, 32, 320, 3), 256: (1, 320, 256, 256, 256, 1)}
LN_CASES = {(160, "LNS"): (640, 640, 384, False), (128, "LNC"): (640, 640, 384, False), (160, "LNC"): (320, 640, 320, False),
            (128, "GEGLU_LNC"): (320, 640, 512, True)}


def test_every_instance_has_a_case():
    cases = {(bn, "PLAIN") for bn in PLAIN_N} | {(bn, "GN") for bn in GN_CASES} | set(LN_CASES) | {(128, "GEGLU")}
    assert {(bn, e) for bn, _, e in G.INSTANCES} == cases
    assert all(e == "PLAIN" or (bn, e) in CASES for bn, _, e in G.INSTANCES)


def run_plain(ctx, sms, bn, passes):
    N = PLAIN_N[bn]
    M = G.bn256_rows(sms) if bn == 256 else 200
    a = G.lo_visible((M, G.LO_MAX_K), bn + passes)
    w = G.lo_visible((G.LO_MAX_K, N), 7 * bn + passes)
    out, tr = ctx.test_linear(a, w, None, passes=passes, trace=True)
    assert len(tr) == 1
    assert_reached(tr[0], bn, passes, "PLAIN")
    assert np.array_equal(out.astype(np.float64), G.pass_product(a, w, passes))


def run_gn(ctx, bn, passes):
    n, cin, H, W, cout, k = GN_CASES[bn]
    x = rnd((n, cin, H, W), 51 + bn)
    w = rnd((cout, cin, k, k), 52 + bn) / np.sqrt(cin * k * k)
    b = rnd((cout,), 53) * 0.5 + 0.3
    g = 1 + 0.1 * rnd((cout,), 54); be = 0.1 * rnd((cout,), 55)
    out, slots, tr = ctx.test_conv_groupnorm(x, w, b, g, be, passes=passes, silu=True, trace=True)
    assert len(tr) == 1 and slots > 0
    assert_reached(tr[0], bn, passes, "GN")
    xr, wr = G.rounded_operands(x, w, passes)
    conv = F.conv2d(torch.from_numpy(xr).double(), torch.from_numpy(wr).double(), torch.from_numpy(b).double(), padding=k // 2)
    ref = F.silu(F.group_norm(conv, 32, torch.from_numpy(g).double(), torch.from_numpy(be).double(), 1e-5)).numpy()
    assert rel(out, ref) < 3e-5


def run_ln(ctx, bn, passes, epi):
    K0, C, N, geglu = LN_CASES[(bn, epi)]
    M = 300
    rng = np.random.default_rng(K0 + N + passes)
    a = rng.standard_normal((M, K0)).astype(np.float32)
    w0 = (rng.standard_normal((K0, C)) / math.sqrt(K0)).astype(np.float32)
    b0 = (rng.standard_normal(C) * 0.5 + 1.5).astype(np.float32)
    g = (1 + 0.1 * rng.standard_normal(C)).astype(np.float32); be = (0.1 * rng.standard_normal(C)).astype(np.float32)
    w1 = (rng.standard_normal((C, N)) / math.sqrt(C)).astype(np.float32)
    b1 = rng.standard_normal(N).astype(np.float32) * 0.3
    # the producer runs 3 passes unless the precision option forces the pass count of every GEMM: that reaches the row-statistics
    # epilogue at 1 and 2 passes too
    ctx.set_option("precision", passes)
    try:
        out, tr = ctx.test_ln_fold(a, w0, b0, g, be, w1, b1, passes=passes, geglu=geglu, trace=True)
    finally:
        ctx.set_option("precision", 0)
    assert len(tr) == 2
    assert_reached(tr[0], 160, passes, "LNS")
    assert_reached(tr[1], 160 if (N % 160 == 0 and not geglu) else 128, passes, "GEGLU_LNC" if geglu else "LNC")
    ar, w0r = G.rounded_operands(a, w0, passes)
    y = ar.astype(np.float64) @ w0r.astype(np.float64) + b0
    mu = y.mean(-1, keepdims=True); var = ((y - mu) ** 2).mean(-1, keepdims=True)
    pre = ((y - mu) / np.sqrt(var + 1e-5) * g + be) @ w1.astype(np.float64) + b1
    ref = pre[:, :N // 2] * gelu_erf(pre[:, N // 2:]) if geglu else pre
    assert rel(out, ref) < (4e-5 if passes == 3 else 1.5e-3)  # the bars of test_layernorm_folded_into_gemms


def run_geglu(ctx, passes):
    M, K, N = 300, 640, 512
    rng = np.random.default_rng(K + passes)
    a = rng.standard_normal((M, K)).astype(np.float32)
    w = (rng.standard_normal((K, N)) / math.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32) * 0.1
    out, tr = ctx.test_gemm_ex(a, w, bias=b, passes=passes, geglu=True, trace=True)
    assert len(tr) == 1
    assert_reached(tr[0], 128, passes, "GEGLU")
    ar, wr = G.rounded_operands(a, w, passes)
    p = ar.astype(np.float64) @ wr.astype(np.float64) + b
    ref = p[:, :N // 2] * gelu_erf(p[:, N // 2:])
    assert rel(out, ref) < (5e-5 if passes == 3 else 2e-4)  # the bars of test_gemm_geglu_epilogue


@pytest.mark.parametrize("bn,passes,epi", G.INSTANCES)
def test_instance(ctx, sms, bn, passes, epi):
    if epi == "PLAIN":
        run_plain(ctx, sms, bn, passes)
    elif epi == "GN":
        run_gn(ctx, bn, passes)
    elif epi == "GEGLU":
        run_geglu(ctx, passes)
    else:
        run_ln(ctx, bn, passes, epi)


# ------------------------------------------------------------------ the split-K fold, exact
def ints(shape, seed, lo=-8, hi=9):
    return np.random.default_rng(seed).integers(lo, hi, shape).astype(np.float32)


def split_case(sms, target, N, bn, seed):
    shape = G.find_split_shape(target, sms, N, bn)
    assert shape is not None, f"no shape splits {target} ways on {sms} SMs"
    M, K = shape
    a = ints((M, K), seed); w = ints((K, N), seed + 1)
    b = ints((N,), seed + 2, 3000, 5000) + 0.25  # the fraction 0.25 is below the fp16 ulp of any |x| >= 512: non-zero lo halves
    r = ints((M, N), seed + 3, -64, 65)
    ref = a.astype(np.float64) @ w.astype(np.float64) + b + r  # |partial sums| < 2^20 in steps of 0.25: exact in fp32
    assert np.abs(ref).max() < 2 ** 20
    return a, w, b, r, ref


# (splits, N, tile width): 160-wide tiles at every remainder of the four-way fold, and one 64-wide case (N = 96: two column
# tiles, the second half masked)
SPLIT_CASES = [(t, 320, 160) for t in (2, 3, 4, 5, 8, 9, 16)] + [(5, 96, 64)]


@pytest.mark.parametrize("target,N,bn", SPLIT_CASES)
def test_split_k_fold_exact(ctx, sms, target, N, bn):
    a, w, b, r, ref = split_case(sms, target, N, bn, 10 * target + bn)
    passes = 3 if target % 2 else 1
    out, tr = ctx.test_gemm_ex(a, w, bias=b, residual=r, passes=passes, trace=True)
    assert len(tr) == 1
    assert_reached(tr[0], bn, passes, "PLAIN", split=target)
    assert np.array_equal(out.astype(np.float64), ref)
    (hi, lo), tr = ctx.test_gemm_ex(a, w, bias=b, residual=r, passes=passes, planes=True, trace=True)
    assert tr[0]["split"] == target
    ehi, elo = G.split_pair(ref.astype(np.float32))
    assert np.array_equal(hi, ehi) and np.array_equal(lo, elo)
    assert np.count_nonzero(lo) > lo.size // 4


def test_split_k_tickets_clean_themselves(ctx, sms):
    """The fold's tile tickets return to zero after each launch: a split shape, another split shape, the first one again."""
    a, w, b, r, ref = split_case(sms, 5, 320, 160, 1)
    a2, w2, b2, r2, ref2 = split_case(sms, 3, 320, 160, 2)
    first = ctx.test_gemm_ex(a, w, bias=b, residual=r, passes=1)
    between, tr = ctx.test_gemm_ex(a2, w2, bias=b2, residual=r2, passes=1, trace=True)
    again, tr2 = ctx.test_gemm_ex(a, w, bias=b, residual=r, passes=1, trace=True)
    assert tr[0]["split"] == 3 and tr2[0]["split"] == 5
    assert np.array_equal(first, again) and np.array_equal(first.astype(np.float64), ref)
    assert np.array_equal(between.astype(np.float64), ref2)
