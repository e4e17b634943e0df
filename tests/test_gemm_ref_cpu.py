"""Preconditions of the exact GEMM references in gemm_ref.py, and the instance table against the dispatch rules it restates."""
import numpy as np
import pytest

import gemm_ref as G


def test_lo_visible_split_is_exact():
    x = G.lo_visible((64, 257), 3)
    s = np.sign(x)
    hi, lo = G.split_pair(x)
    assert np.array_equal(hi, s) and np.array_equal(x.astype(np.float16).astype(np.float32), s)  # numpy float16 agrees
    assert np.array_equal(hi.astype(np.float64) + lo, x.astype(np.float64))
    j = lo / (s * G.LO_STEP)
    assert np.array_equal(j, np.round(j)) and set(np.unique(j)) == {0.0, 1.0, 2.0, 3.0}
    # the sign of lo follows s: -1 + 3 2^-13 would round to -(1 - 2^-11), not to -1
    assert np.float32(-1 + 3 * G.LO_STEP).astype(np.float16) != np.float16(-1)


def test_lo_visible_terms_are_exact_in_fp32():
    """Each term is a multiple of 2^-13 and K max|term| < 2^11: 24 bits hold every partial sum, so fp32 accumulation in any
    order reproduces the fp64 sum of the terms."""
    K = G.LO_MAX_K
    max_term = 1.0 + 2 * 3 * G.LO_STEP  # hi hi + lo hi + hi lo of one k
    assert K * max_term < 2.0 ** 11
    a = G.lo_visible((8, K), 1); w = G.lo_visible((K, 8), 2)
    ah, al = G.split_pair(a); wh, wl = G.split_pair(w)
    for terms in (ah[:, :, None] * wh[None], al[:, :, None] * wh[None], ah[:, :, None] * wl[None]):
        t = terms.astype(np.float64) / G.LO_STEP
        assert np.array_equal(t, np.round(t))
    for p in (1, 2, 3):
        ref = G.pass_product(a, w, p)
        assert np.array_equal(ref.astype(np.float32).astype(np.float64), ref)
        rng = np.random.default_rng(p)
        order = rng.permutation(K)  # a different summation order in fp32 gives the same result
        acc = np.zeros((8, 8), np.float32)
        for k in order:
            acc += ah[:, k, None] * wh[None, k] + (al[:, k, None] * wh[None, k] if p >= 2 else 0) + \
                   (ah[:, k, None] * wl[None, k] if p >= 3 else 0)
        assert np.array_equal(acc.astype(np.float64), ref)
    assert not np.array_equal(G.pass_product(a, w, 1), G.pass_product(a, w, 2))  # the lo halves are visible
    assert not np.array_equal(G.pass_product(a, w, 2), G.pass_product(a, w, 3))


def test_split_pair_range():
    hi, lo = G.split_pair(np.array([131024.0, -2.0e5, 1.0e30, 65519.0, 100000.0, -131008.0], np.float32))
    assert np.array_equal(hi + lo, np.array([131008.0, -131008.0, 131008.0, 65519.0, 100000.0, -131008.0], np.float32))
    assert np.all(np.abs(hi) <= 65504) and np.all(np.isfinite(lo))
    # the plain split the pair writers used before: fp16(x - 65504) overflows above 131008
    with np.errstate(over="ignore"):
        assert np.isinf(np.float16(np.float32(131024) - np.float32(65504)))
    hi, lo = G.split_pair(np.array([np.nan, np.inf, -np.inf], np.float32))
    assert np.isnan(hi).all() and np.isnan(lo).all()


def test_stage_counts():
    assert {(bn, p): G.pick_stages(bn, p) for bn in G.BNS for p in (1, 2, 3)} == {
        (64, 1): 8, (64, 2): 5, (64, 3): 4, (128, 1): 7, (128, 2): 4, (128, 3): 3,
        (160, 1): 6, (160, 2): 4, (160, 3): 3, (256, 1): 4, (256, 2): 3, (256, 3): 2}


def test_instance_table_matches_dispatch():
    assert len(G.INSTANCES) == len(set(G.INSTANCES)) == 36
    assert set(G.INSTANCES) == {(bn, p, e) for bn in G.BNS for p in (1, 2, 3) for e in G.EPIS if G.builds(bn, e)}


@pytest.mark.parametrize("sms", [132, 114, 78])
def test_ring_and_split_shapes_reach_their_instances(sms):
    """The shapes the GPU tests use reach the tile width they claim under the restated rules, for H100 SXM (132 SMs), PCIe (114)
    and a smaller part."""
    for N, bn in ((96, 64), (384, 128), (320, 160)):
        assert G.linear_instance(200, 64 * 17, N, sms, 1)[0::2] == (bn, 1)
    assert G.linear_instance(G.bn256_rows(sms), 64 * 9, 1024, sms, 1)[0::2] == (256, 1)
    assert G.linear_instance(G.bn256_rows(sms) - 128, 64 * 9, 1024, sms, 1)[0] == 128  # one tile fewer falls back to 128
    for target in (2, 3, 4, 5, 8, 9, 16):
        for N, bn in ((320, 160), (96, 64)):
            M, K = G.find_split_shape(target, sms, N, bn)
            assert G.linear_instance(M, K, N, sms, 3)[0::2] == (bn, target)
