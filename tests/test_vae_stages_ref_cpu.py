"""The fp64 stage references of tests/test_vae_stages_gpu.py, chained in the model's order, reproduce the oracle's decode_latent
and encode_image (the op definitions the decode / encode goldens are made with). A reference that drifted from the model's order,
or restated an op differently, fails here without a GPU."""
import os

import numpy as np
import pytest
import torch

import inpaint_oracle as IP
import test_vae_stages_gpu as V
from oracle import sd_oracle as O
from stable_diffusion_burn_b200 import synth, topology

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def P():
    torch.set_num_threads(os.cpu_count() or 1)
    return O.Params(synth.make_params(0, which=topology.vae_decoder_params() + topology.vae_encoder_params()), dtype=torch.float64)


def close(a, b, bar=1e-10):
    return float((a - b).abs().max() / b.abs().max()) <= bar


def chained_decode(P, latent, pre_scale=1.0):
    x = V.ref_dec_in(P, latent, pre_scale)
    x = O.resnet_block(P, f"{V.DEC}/mid/block_1", x)
    x = V.ref_attention(P, V.ATTN["dec_attn"], x)[0].reshape(x.shape)
    x = O.resnet_block(P, f"{V.DEC}/mid/block_2", x)
    nb = len(topology.VAE_DECODER_BLOCKS)
    for i in range(nb):
        for r in ("res1", "res2", "res3"):
            x = O.resnet_block(P, f"{V.DEC}/blocks/{i}/{r}", x)
        if i != nb - 1:
            x = O.conv2d(P, f"{V.DEC}/blocks/{i}/upsampler", O.upsample_nearest2x(x), padding=1)
    norm, conv, _, _ = V.OUT["dec_out"]
    return V.ref_norm_conv(P, norm, conv, x)


def chained_encode(P, img):
    x4 = torch.cat([img, torch.zeros_like(img[:, :1])], 1)  # the encoder's input with its zero fourth plane
    x = O.conv2d(P, f"{V.ENC}/conv_in", x4[:, :3], padding=1)
    nb = len(topology.VAE_ENCODER_BLOCKS)
    for i in range(nb):
        for r in ("res1", "res2"):
            x = O.resnet_block(P, f"{V.ENC}/blocks/{i}/{r}", x)
        if i != nb - 1:
            x = V.ref_down(P, V.DOWN[i][0], x)
    x = O.resnet_block(P, f"{V.ENC}/mid/block_1", x)
    x = V.ref_attention(P, V.ATTN["enc_attn"], x)[0].reshape(x.shape)
    x = O.resnet_block(P, f"{V.ENC}/mid/block_2", x)
    norm, conv, _, _ = V.OUT["enc_out"]
    return V.ref_quant(P, V.ref_norm_conv(P, norm, conv, x))


def test_chained_stages_reproduce_decode_latent(P):
    """the 16x16 latent of the vae_16 golden"""
    lat = torch.from_numpy(synth.make_latent(1, 16, 16, seed=21).astype(np.float64))
    with torch.no_grad():
        a = chained_decode(P, lat)
        b = O.decode_latent(P, lat)
    assert a.shape == b.shape == (1, 3, 128, 128)
    assert close(a, b)


def test_chained_stages_reproduce_encode_image(P):
    """the ramp64 image of the vae_enc golden"""
    img = torch.from_numpy(np.load(os.path.join(GOLD, "vae_enc.npz"))["img:ramp64"].astype(np.float64))
    with torch.no_grad():
        a = chained_encode(P, img)
        b = O.encode_image(P, img)
    assert a.shape == b.shape == (1, 4, 8, 8)
    assert close(a, b)


def test_pre_scale_folds_into_the_latent(P):
    """conv_in's folded pre-scale is latent_to_image's `latent * (1 / 0.18215)` ahead of decode_latent's post_quant_conv"""
    lat = torch.from_numpy(synth.make_latent(2, 5, 7, seed=3).astype(np.float64))
    with torch.no_grad():
        a = V.ref_dec_in(P, lat, V.PRE_SCALE)
        b = O.conv2d(P, f"{V.DEC}/conv_in", O.conv2d(P, "autoencoder/post_quant_conv", lat * V.PRE_SCALE), padding=1)
    assert close(a, b, 0.0)


@pytest.mark.parametrize("stage", list(V.ATTN))
def test_v_bias_after_pv_is_the_oracle_block(P, stage):
    """softmax rows sum to one, so the v bias added after P.V is the oracle's v = conv(h) + b_v ahead of the softmax average;
    with a v bias 10x the projection, and with the query rows computed in a strided subset"""
    name = V.ATTN[stage]
    x = torch.from_numpy(V.split22(V.activation(f"cpu/{stage}", 2, 512, 6, 4)))
    P2 = O.Params({}, dtype=torch.float64)
    P2.t = dict(P.t)
    P2.t[f"{name}/v/bias"] = P(f"{name}/v/bias") * 0 + 10.0 * float(P(f"{name}/v/weight").abs().mean() * 512)
    for p in (P, P2):
        with torch.no_grad():
            a = V.ref_attention(p, name, x)[0].reshape(x.shape)
            b = O.conv_self_attention_block(p, name, x)
            sub = V.ref_attention(p, name, x, rows=slice(1, 24, 5))[0]
        assert close(a, b)
        assert close(sub, b.reshape(2, 512, 24)[:, :, 1:24:5])


def test_rounded_attention_differs_by_fp16_rounding(P):
    """the precision = 1 reference (fp16 operands and fp16 q, k, V^T, P and o) moves the block by an fp16-sized amount"""
    name = V.ATTN["dec_attn"]
    x = torch.from_numpy(V.split22(V.activation("cpu/rnd", 1, 512, 4, 4)))
    with torch.no_grad():
        a = V.ref_attention(P, name, x, rnd=True)[0].reshape(x.shape)
        b = V.ref_attention(P, name, x)[0].reshape(x.shape)
    d = float((a - b).abs().max() / b.abs().max())
    assert 1e-6 < d < 1e-2, d  # the rounding is applied, and it is fp16-sized


def strided_quant(y8, w, b, scale, out):
    """the index arithmetic of quant_conv_slice_scaled_kernel on a flat buffer: sample i, channel c, pixel p lands at
    base + i * 5 HW + c * HW + p with base = HW (channels 1-4 of [n, 5, H, W]), value fl32(acc * scale)"""
    n, _, h, wd = y8.shape
    hw = h * wd
    flat = out.reshape(-1)
    acc = (np.einsum("oc,ncp->nop", w.reshape(8, 8)[:4], y8.reshape(n, 8, hw).astype(np.float64)) + b[:4, None]).astype(np.float32)
    for i in range(n):
        for c in range(4):
            flat[hw + i * 5 * hw + c * hw:hw + i * 5 * hw + (c + 1) * hw] = np.multiply(acc[i, c], np.float32(scale))
    return out


def test_strided_quant_slice_is_the_inpainting_layout(P):
    """the strided, scaled quant slice writes [n, 5, H, W] the way inpaint_oracle.inpaint_cond lays it out: the latent mask in
    channel 0 (left untouched), fl(z * 0.18215) in channels 1-4"""
    rng = np.random.default_rng(4)
    n, h, w = 3, 4, 6
    y8 = rng.standard_normal((n, 8, h, w)).astype(np.float32)
    mask = (rng.random((n, 8 * h, 8 * w)) < 0.5).astype(np.uint8) * 255
    m_lat = IP.latent_mask(mask)
    out = np.zeros((n, 5, h, w), np.float32)
    out[:, 0] = m_lat
    qw = P("autoencoder/quant_conv/weight").numpy().astype(np.float32)
    qb = P("autoencoder/quant_conv/bias").numpy().astype(np.float32)
    strided_quant(y8, qw, qb, 0.18215, out)
    z = O.conv2d(O.Params({"q/weight": qw, "q/bias": qb}), "q", torch.from_numpy(y8))[:, :4].numpy()
    want = np.concatenate([m_lat[:, None], np.multiply(z, np.float32(0.18215))], 1)
    assert np.array_equal(out[:, 0], want[:, 0])
    assert np.allclose(out, want, rtol=1e-6, atol=1e-6 * np.abs(want).max())
    with torch.no_grad():
        ref = V.ref_quant(P, torch.from_numpy(y8.astype(np.float64)), float(np.float32(0.18215))).numpy()
    assert np.allclose(out[:, 1:], ref, rtol=1e-6, atol=1e-6 * np.abs(ref).max())
