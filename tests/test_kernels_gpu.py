"""GPU parity of the individual kernels, called through the C ABI, against torch-CPU fp32 references
of the same op (the op definitions the oracle uses)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gemm_ref as G

pytestmark = pytest.mark.gpu

# tolerance per number of tensor-core passes (relative L2): 1 pass = fp16 operand rounding,
# 2 = activations exact, 3 = fp32-class
TOL = {1: 1.0e-3, 2: 8.0e-4, 3: 2.0e-5}


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def rnd(shape, seed, scale=1.0):
    return (np.random.default_rng(seed).standard_normal(shape) * scale).astype(np.float32)


@pytest.mark.parametrize("passes", [1, 2, 3])
@pytest.mark.parametrize("M,K,N", [(300, 320, 320), (128, 2560, 1280), (77, 64, 64), (4096, 128, 512),
                                    (19072, 128, 512), (1, 768, 640), (1000, 1280, 960)])
def test_linear(ctx, M, K, N, passes):
    a = rnd((M, K), 1); w = rnd((K, N), 2, K ** -0.5); b = rnd((N,), 3)
    ref = a.astype(np.float64) @ w.astype(np.float64) + b
    out = ctx.test_linear(a, w, b, passes=passes)
    assert rel(out, ref) < TOL[passes]


def test_linear_exact_small_integers(ctx):
    """Integer-valued operands are exact in fp16: the GEMM must be bit-exact (catches layout bugs)."""
    rng = np.random.default_rng(0)
    a = rng.integers(-4, 5, (256, 192)).astype(np.float32)
    w = rng.integers(-4, 5, (192, 128)).astype(np.float32)
    out = ctx.test_linear(a, w, None, passes=1)
    assert np.array_equal(out, a @ w)


CONV_CASES = [
    # n, cin, H, W, cout, k, stride, upsample
    (2, 64, 16, 16, 64, 3, 1, 0),
    (1, 128, 32, 32, 320, 3, 1, 0),
    (2, 64, 8, 8, 128, 3, 1, 0),
    (1, 64, 24, 24, 64, 3, 1, 0),
    (1, 64, 64, 64, 64, 3, 1, 0),
    (3, 64, 8, 8, 64, 3, 1, 0),
    (2, 64, 16, 16, 128, 3, 2, 0),
    (1, 128, 64, 64, 64, 3, 2, 0),
    (2, 64, 8, 8, 64, 3, 1, 1),
    (1, 64, 16, 16, 128, 3, 1, 1),
    (2, 128, 16, 16, 64, 1, 1, 0),
    (1, 64, 256, 256, 64, 3, 1, 0),
]


@pytest.mark.parametrize("passes", [1, 3])
@pytest.mark.parametrize("n,cin,H,W,cout,k,stride,up", CONV_CASES)
def test_conv2d(ctx, n, cin, H, W, cout, k, stride, up, passes):
    x = rnd((n, cin, H, W), 11); w = rnd((cout, cin, k, k), 12, (cin * k * k) ** -0.5); b = rnd((cout,), 13)
    xt = torch.from_numpy(x).double()
    if up:
        xt = F.interpolate(xt, scale_factor=2, mode="nearest")
    ref = F.conv2d(xt, torch.from_numpy(w).double(), torch.from_numpy(b).double(), stride=stride, padding=k // 2).numpy()
    out = ctx.test_conv2d(x, w, b, stride=stride, upsample=up, passes=passes)
    assert out.shape == ref.shape
    assert rel(out, ref) < TOL[passes]


# n, cin, H, W, cout, ksize: plain tiles (one image per tile), two / four images per tile (8x8, 8x4), split-K (small grid, long
# K), a 1x1 conv over flattened tokens, a VAE width (bucket = group size), an awkward 12x12 map (masked tile rows)
GN_FROM_GEMM = [(2, 320, 32, 32, 320, 3), (2, 1280, 8, 8, 1280, 3), (4, 640, 8, 4, 640, 3), (2, 1280, 16, 16, 640, 3),
                (2, 320, 16, 16, 640, 1), (2, 640, 8, 8, 320, 1), (1, 512, 32, 32, 512, 3), (1, 256, 64, 64, 128, 3), (2, 320, 12, 12, 320, 3),
                # n = 3 on 8x8 maps: two images per tile with the second image of the last tile masked, without and with split-K
                (3, 64, 8, 8, 320, 3), (3, 1280, 8, 8, 1280, 3)]


@pytest.mark.parametrize("n,cin,H,W,cout,k", GN_FROM_GEMM)
@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_from_gemm_statistics(ctx, n, cin, H, W, cout, k, silu):
    """GroupNorm whose statistics come from the epilogue of the GEMM that wrote the tensor (no statistics pass)."""
    x = rnd((n, cin, H, W), 51)
    w = rnd((cout, cin, k, k), 52) / np.sqrt(cin * k * k)
    b = rnd((cout,), 53) * 0.5 + 0.3  # a non-zero mean makes sum^2 / sumsq cancellation visible
    g = 1 + 0.1 * rnd((cout,), 54); be = 0.1 * rnd((cout,), 55)
    conv = F.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), torch.from_numpy(b).double(), padding=k // 2)
    ref = F.group_norm(conv, 32, torch.from_numpy(g).double(), torch.from_numpy(be).double(), 1e-5)
    if silu:
        ref = F.silu(ref)
    out, slots = ctx.test_conv_groupnorm(x, w, b, g, be, passes=3, silu=silu)
    e = rel(out, ref.numpy())
    print(f"GN from GEMM statistics n={n} {cin}->{cout} {H}x{W} k={k}: {slots} slots/image, rel L2 {e:.3e}")
    assert slots > 0 and e < 3e-5


# n, cin, H, W, cout, stride, upsample: the UNet downsample convs (stride 2; the 16x16 -> 8x8 one packs two images per tile and
# splits K) and the folded nearest-2x upsample convs, whose four output phases write separate partial slots
GN_FROM_RESAMPLING_GEMM = [(2, 320, 32, 32, 320, 2, 0), (2, 640, 16, 16, 640, 2, 0), (1, 320, 64, 64, 320, 2, 0),
                           (2, 1280, 8, 8, 1280, 1, 1), (2, 640, 16, 16, 640, 1, 1), (1, 512, 32, 32, 512, 1, 1),
                           (3, 1280, 8, 8, 1280, 1, 1)]


@pytest.mark.parametrize("n,cin,H,W,cout,stride,up", GN_FROM_RESAMPLING_GEMM)
@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_from_resampling_gemm_statistics(ctx, n, cin, H, W, cout, stride, up, silu):
    """GroupNorm from the statistics the stride-2 and upsample conv epilogues leave (the UNet's downsample and upsample blocks)."""
    x = rnd((n, cin, H, W), 56)
    w = rnd((cout, cin, 3, 3), 57) / np.sqrt(cin * 9)
    b = rnd((cout,), 58) * 0.5 + 0.3
    g = 1 + 0.1 * rnd((cout,), 59); be = 0.1 * rnd((cout,), 60)
    xt = torch.from_numpy(x).double()
    if up:
        xt = F.interpolate(xt, scale_factor=2, mode="nearest")
    conv = F.conv2d(xt, torch.from_numpy(w).double(), torch.from_numpy(b).double(), stride=stride, padding=1)
    ref = F.group_norm(conv, 32, torch.from_numpy(g).double(), torch.from_numpy(be).double(), 1e-5)
    if silu:
        ref = F.silu(ref)
    out, slots = ctx.test_conv_groupnorm(x, w, b, g, be, passes=3, silu=silu, stride=stride, upsample=up)
    assert out.shape == ref.shape
    e = rel(out, ref.numpy())
    print(f"GN from GEMM statistics n={n} {cin}->{cout} {H}x{W} stride={stride} up={up}: {slots} slots/image, rel L2 {e:.3e}")
    assert slots > 0 and e < 3e-5


@pytest.mark.parametrize("rows,c", [(100, 320), (64, 640), (33, 1280)])
def test_layernorm(ctx, rows, c):
    x = rnd((rows, c), 31) * 2 - 0.3
    g = 1 + 0.1 * rnd((c,), 32); b = 0.1 * rnd((c,), 33)
    ref = F.layer_norm(torch.from_numpy(x).double(), (c,), torch.from_numpy(g).double(), torch.from_numpy(b).double(), 1e-5)
    out = ctx.test_layernorm(x, g, b)
    assert rel(out, ref.numpy()) < 5e-6


@pytest.mark.parametrize("scale", [1.0e3, 3.0e4, 1.0e5, 3.0e5, 1.0e6])
def test_raw_operand_fp16_range(ctx, scale):
    """Raw (un-normalised) GEMM operands — skip 1x1 convs, upsample / downsample convs, the VAE's nin_shortcut — are staged as
    fp16 hi + lo pairs. The hi half saturates at 65504 and the lo half carries the excess, so the multi-pass product stays finite
    and accurate for |x| <= 131008 (a trained VAE decoder is known to exceed the fp16 range); beyond that the pair clips at
    +-131008, and single-pass operands clip at 65504, instead of turning into inf / NaN.

    The 3-pass conv must equal the fp64 sum of the three terms it forms from the operand splits (gemm_ref.pass_product). Against
    the fp64 conv of clip(x, +-131008) it is accurate to the pair's precision: 2^-22 below 65504, but above it lo = x - 65504 holds
    only 11 bits (relative step <= 2^-12 of x) and the omitted lo * lo term is no longer negligible, so the bar there is 2 * 2^-12."""
    rng = np.random.default_rng(7)
    x = (rng.standard_normal((1, 128, 16, 16)) * scale / 4).astype(np.float32)  # |x| up to ~4.5 sigma = 1.1 * scale
    x[0, 5, 3, 3] = 1.2 * scale
    w = (rng.standard_normal((64, 128, 1, 1)) / np.sqrt(128)).astype(np.float32)
    ref = F.conv2d(torch.from_numpy(np.clip(x, -131008, 131008)).double(), torch.from_numpy(w).double()).numpy()
    terms = G.pass_product(x[0].reshape(128, 256).T, w[:, :, 0, 0].T, 3).T.reshape(1, 64, 16, 16)
    out = ctx.test_conv2d(x, w, None, passes=3)
    assert np.isfinite(out).all()
    e, et = rel(out, ref), rel(out, terms)
    print(f"raw operand range, max |x| = {np.abs(x).max():.3g}: 3-pass rel L2 {e:.3e} (against the 3-pass terms {et:.3e})")
    assert et < 5e-5
    assert e < (5e-5 if scale <= 1.0e5 else 2 * 2.0 ** -12)
    out1 = ctx.test_conv2d(x, w, None, passes=1)
    assert np.isfinite(out1).all()  # single pass: clipped at 65504 above the fp16 range, never inf / NaN
    if scale <= 3.0e4:
        assert rel(out1, ref) < 1e-3


@pytest.mark.parametrize("passes", [1, 2, 3])
def test_gemm_fp16_pair_output_saturates(ctx, passes):
    """An fp16 hi + lo output beyond the pair's range holds +-131008 exactly, never inf / NaN; inside it both halves equal the
    split of the exact fp32 result. Integer operands, exact in fp16, so every pass count gives the same exact product."""
    rng = np.random.default_rng(passes)
    a = rng.integers(-8, 9, (200, 64)).astype(np.float32)
    w = (rng.integers(-8, 9, (64, 320)) * 1024).astype(np.float32)  # |products| up to 2^16: results up to ~1e6, exact in fp32
    ref = a.astype(np.float64) @ w.astype(np.float64)
    big = np.abs(ref) > 131008
    assert big.mean() > 0.2 and (~big).mean() > 0.2 and (np.abs(ref[~big]) > 65520).any()
    hi, lo = ctx.test_gemm_ex(a, w, passes=passes, planes=True)
    assert np.isfinite(hi).all() and np.isfinite(lo).all()
    assert np.array_equal((hi + lo)[big], np.sign(ref[big]) * 131008)
    ehi, elo = G.split_pair(ref.astype(np.float32))
    assert np.array_equal(hi, ehi) and np.array_equal(lo, elo)


@pytest.mark.parametrize("passes", [1, 2, 3])
def test_gemm_nan_operand_stays_nan(ctx, passes):
    """A NaN in row r of A makes output row r NaN at every pass count (the operand split keeps it NaN in both halves instead of
    clipping it to a finite value); every other row is exact."""
    rng = np.random.default_rng(10 + passes)
    a = rng.integers(-4, 5, (200, 192)).astype(np.float32)
    w = rng.integers(-4, 5, (192, 128)).astype(np.float32)
    w[37] = 0.0  # NaN * 0 is NaN too
    ref = a @ w
    r = 131
    a[r, 37] = np.nan
    out = ctx.test_gemm_ex(a, w, passes=passes)
    assert np.isnan(out[r]).all()
    keep = np.arange(200) != r
    assert np.array_equal(out[keep], ref[keep])
