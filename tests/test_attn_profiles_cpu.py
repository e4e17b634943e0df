"""The rescale profiles of tests/attn_profiles.py do what they claim under the kernel's rescale rule (attention.cu:218-221,
threshold read from the source): if the inputs or the threshold change, these fail instead of the GPU tests silently no longer
reaching the rescale branch."""
import numpy as np
import pytest

import attn_profiles as P

CASES = [(p, d) for p, (_, dims) in P.PROFILES.items() for d in dims]


def _replay(profile, d, threshold=None):
    q, k, _ = P.make_case(profile, d)
    return P.replay(q, k, P.HEADS, split=d in (40, 80), threshold=threshold)


def test_threshold_is_read_from_the_kernel():
    assert 1.0 <= P.kernel_threshold() < 16.0  # P < 2^threshold must stay finite in fp16 (max 65504)


@pytest.mark.parametrize("profile,d", CASES)
def test_profile_drives_the_rescale_rule(profile, d):
    resc, growth, pmax = _replay(profile, d)
    later = resc[..., 1:]
    print(f"{profile} d={d}: rescales after the first sub-tile {later.mean():.3f}, largest stale P {pmax[..., 1:][~later].max(initial=0):.1f}")
    assert resc[..., 0].all()  # the first sub-tile always sets the reference point
    if profile == "ramp":
        assert later.all()
    elif profile == "creep":
        assert 0.1 < later.mean() < 0.9
        stale = pmax[..., 1:][~later]  # sub-tiles exponentiated against the stale reference point
        assert stale.max() > 128.0
        # rows r and r + 8 of a 16-row group share a thread (the two row halves of the wgmma accumulator) and need their own
        # alpha: they must decide differently somewhere, or an alpha of the wrong half goes unnoticed
        n, h, Nq, T = resc.shape
        g = resc[:, :, :Nq // 16 * 16].reshape(n, h, -1, 2, 8, T)
        assert (g[:, :, :, 0] != g[:, :, :, 1]).mean() > 0.1
    elif profile == "late_spike":
        assert resc[..., -1].all() and (growth[..., -1] > 32.0).all()
    elif profile == "early_peak":
        assert not later.any()
        assert (pmax[..., 1:].astype(np.float16) == 0).all()  # every later P underflows in fp16
    elif profile == "subtile_spike":
        assert resc[..., 1].all()  # between the two 64-key sub-tiles of tile 0
    elif profile == "fp16_edge":
        t = (128 + 37) // P.sub_tile_width(d)
        assert resc[..., t].all() and not resc[..., 1:t].any()
        # without that rescale (a threshold of 16) P would be 2^15.9998, which rounds to inf in fp16
        r16, g16, p16 = _replay(profile, d, threshold=16.0)
        assert not r16[..., t].any() and (g16[..., t] > 15.9996).all()
        with np.errstate(over="ignore"):
            assert np.isinf(p16[..., t].astype(np.float16)).all()
    else:
        raise AssertionError(f"no claim checked for profile {profile}")
