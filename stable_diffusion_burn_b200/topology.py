"""Parameter inventory of the SD-v1.4 sampling hot path (UNet + VAE decoder half).

Names are the reference's dump-dir paths (directory names == Rust field names):
  reference src/model/unet/load.rs:213-306, src/model/autoencoder/load.rs:16-198,
  src/model/load.rs:65-160 (Linear weight stored [in,out]; Conv weight OIHW),
  src/model/groupnorm/load.rs:13-37 (GroupNorm "weight"/"bias").
Shapes come from the topology in src/model/unet/mod.rs:35-93 and
src/model/autoencoder/mod.rs:29-45,153-192.

Each entry: (name, shape, kind, fan_in) with kind in
  {"conv_w","conv_b","lin_w","lin_b","norm_g","norm_b","emb"}.
The C++ library builds the same list independently (csrc/model.cu); a test
cross-checks the two through sdb_tensor_count / sdb_tensor_info.
"""
from __future__ import annotations

N_HEAD = 8
CTX_DIM = 768
EMB_DIM = 1280


def _conv(out, name, cin, cout, k, bias=True):
    out.append((f"{name}/weight", (cout, cin, k, k), "conv_w", cin * k * k))
    if bias:
        out.append((f"{name}/bias", (cout,), "conv_b", cin * k * k))


def _lin(out, name, cin, cout, bias=True):
    out.append((f"{name}/weight", (cin, cout), "lin_w", cin))
    if bias:
        out.append((f"{name}/bias", (cout,), "lin_b", cin))


def _norm(out, name, c):
    out.append((f"{name}/weight", (c,), "norm_g", c))
    out.append((f"{name}/bias", (c,), "norm_b", c))


def _resblock(out, name, cin, cout):
    # reference ResBlockConfig::init unet/mod.rs:662-697
    _norm(out, f"{name}/norm_in", cin)
    _conv(out, f"{name}/conv_in", cin, cout, 3)
    _lin(out, f"{name}/lin_embed", EMB_DIM, cout)
    _norm(out, f"{name}/norm_out", cout)
    _conv(out, f"{name}/conv_out", cout, cout, 3)
    if cin != cout:
        _conv(out, f"{name}/skip_connection", cin, cout, 1)


def _mha(out, name, c, cctx):
    # unet/mod.rs:601-630: q/k/v no bias, out with bias
    _lin(out, f"{name}/query", c, c, bias=False)
    _lin(out, f"{name}/key", cctx, c, bias=False)
    _lin(out, f"{name}/value", cctx, c, bias=False)
    _lin(out, f"{name}/out", c, c)


def _spatial_transformer(out, name, c):
    # unet/mod.rs:436-451, 490-508, 535-570
    _norm(out, f"{name}/norm", c)
    _conv(out, f"{name}/proj_in", c, c, 1)
    t = f"{name}/transformer"
    _norm(out, f"{t}/norm1", c)
    _mha(out, f"{t}/attn1", c, c)
    _norm(out, f"{t}/norm2", c)
    _mha(out, f"{t}/attn2", c, CTX_DIM)
    _norm(out, f"{t}/norm3", c)
    _lin(out, f"{t}/mlp/geglu/proj", c, 8 * c)
    _lin(out, f"{t}/mlp/lin", 4 * c, c)
    _conv(out, f"{name}/proj_out", c, c, 1)


# (field, kind, cin, cout) in as_array() order; unet/mod.rs:41-73, 161-193
UNET_INPUT_BLOCKS = [
    ("conv", "conv", 4, 320),
    ("rt1", "rt", 320, 320), ("rt2", "rt", 320, 320), ("d1", "down", 320, 320),
    ("rt3", "rt", 320, 640), ("rt4", "rt", 640, 640), ("d2", "down", 640, 640),
    ("rt5", "rt", 640, 1280), ("rt6", "rt", 1280, 1280), ("d3", "down", 1280, 1280),
    ("r1", "r", 1280, 1280), ("r2", "r", 1280, 1280),
]
UNET_OUTPUT_BLOCKS = [
    ("r1", "r", 2560, 1280), ("r2", "r", 2560, 1280), ("ru", "ru", 2560, 1280),
    ("rt1", "rt", 2560, 1280), ("rt2", "rt", 2560, 1280), ("rtu1", "rtu", 1920, 1280),
    ("rt3", "rt", 1920, 640), ("rt4", "rt", 1280, 640), ("rtu2", "rtu", 960, 640),
    ("rt5", "rt", 960, 320), ("rt6", "rt", 640, 320), ("rt7", "rt", 640, 320),
]


def _unet_block(out, name, kind, cin, cout):
    if kind == "conv":
        _conv(out, name, cin, cout, 3)
    elif kind == "down":
        _conv(out, name, cin, cout, 3)
    elif kind == "r":
        _resblock(out, name, cin, cout)
    elif kind == "rt":
        _resblock(out, f"{name}/res", cin, cout)
        _spatial_transformer(out, f"{name}/transformer", cout)
    elif kind == "ru":
        _resblock(out, f"{name}/res", cin, cout)
        _conv(out, f"{name}/upsample/conv", cout, cout, 3)
    elif kind == "rtu":
        _resblock(out, f"{name}/res", cin, cout)
        _spatial_transformer(out, f"{name}/transformer", cout)
        _conv(out, f"{name}/upsample/conv", cout, cout, 3)
    else:
        raise ValueError(kind)


def unet_params(prefix="unet", in_channels=4, pix2pix=False):
    """in_channels: 4 (SD-v1) or 9 (an inpainting UNet: conv_in reads latent | mask | masked-image latent, DESIGN.md §7 f9).
    pix2pix=True (with in_channels 4): the InstructPix2Pix UNet, whose conv_in reads latent | image latent, 8 channels (f10)."""
    if in_channels not in (4, 9):
        raise ValueError(f"in_channels must be 4 or 9, got {in_channels} (the 8-channel InstructPix2Pix UNet is pix2pix=True)")
    if pix2pix and in_channels != 4:
        raise ValueError("pix2pix=True widens the 4-channel conv_in to 8 channels; in_channels must be 4")
    conv_in = 8 if pix2pix else in_channels
    out = []
    _lin(out, f"{prefix}/lin1_time_embed", 320, EMB_DIM)
    _lin(out, f"{prefix}/lin2_time_embed", EMB_DIM, EMB_DIM)
    for i, (f, kind, cin, cout) in enumerate(UNET_INPUT_BLOCKS):
        _unet_block(out, f"{prefix}/input_blocks/{f}", kind, conv_in if i == 0 else cin, cout)
    # conv_in's bias keeps the 4-channel fan-in: only the weight of a wider registry differs (its synthetic stream too)
    b = next(i for i, e in enumerate(out) if e[0] == f"{prefix}/input_blocks/conv/bias")
    out[b] = out[b][:3] + (4 * 9,)
    # middle: ResTransformerRes(1280,1280,1280,768,8) unet/mod.rs:58, 328-351
    m = f"{prefix}/middle_block"
    _resblock(out, f"{m}/res1", 1280, 1280)
    _spatial_transformer(out, f"{m}/transformer", 1280)
    _resblock(out, f"{m}/res2", 1280, 1280)
    for f, kind, cin, cout in UNET_OUTPUT_BLOCKS:
        _unet_block(out, f"{prefix}/output_blocks/{f}", kind, cin, cout)
    _norm(out, f"{prefix}/norm_out", 320)
    _conv(out, f"{prefix}/conv_out", 320, 4, 3)
    return out


VAE_DECODER_BLOCKS = [(512, 512), (512, 512), (512, 256), (256, 128)]  # autoencoder/mod.rs:33-34


def _resnet(out, name, cin, cout):
    # autoencoder/mod.rs:471-503
    _norm(out, f"{name}/norm1", cin)
    _conv(out, f"{name}/conv1", cin, cout, 3)
    _norm(out, f"{name}/norm2", cout)
    _conv(out, f"{name}/conv2", cout, cout, 3)
    if cin != cout:
        _conv(out, f"{name}/nin_shortcut", cin, cout, 1)


def vae_decoder_params(prefix="autoencoder"):
    out = []
    _conv(out, f"{prefix}/post_quant_conv", 4, 4, 1)
    d = f"{prefix}/decoder"
    _conv(out, f"{d}/conv_in", 4, 512, 3)
    _resnet(out, f"{d}/mid/block_1", 512, 512)
    a = f"{d}/mid/attn"
    _norm(out, f"{a}/norm", 512)
    for n in ("q", "k", "v", "proj_out"):
        _conv(out, f"{a}/{n}", 512, 512, 1)
    _resnet(out, f"{d}/mid/block_2", 512, 512)
    for i, (cin, cout) in enumerate(VAE_DECODER_BLOCKS):
        b = f"{d}/blocks/{i}"
        _resnet(out, f"{b}/res1", cin, cout)
        _resnet(out, f"{b}/res2", cout, cout)
        _resnet(out, f"{b}/res3", cout, cout)
        if i != len(VAE_DECODER_BLOCKS) - 1:
            _conv(out, f"{b}/upsampler", cout, cout, 3)
    _norm(out, f"{d}/norm_out", 128)
    _conv(out, f"{d}/conv_out", 128, 3, 3)
    return out


VAE_ENCODER_BLOCKS = [(128, 128), (128, 256), (256, 512), (512, 512)]  # autoencoder/mod.rs:31


def vae_encoder_params(prefix="autoencoder"):
    """VAE encoder + quant_conv (SURVEY §8f row f4): autoencoder/mod.rs:60-66, 122-145, 249-266; names from
    autoencoder/load.rs:100-181. Shapes are the SD-v1 ones a dump carries (mid / norm_out / conv_out at 512 channels);
    EncoderConfig::init would size them from channels.first().0 = 128 (:84), which no loaded model uses."""
    out = []
    e = f"{prefix}/encoder"
    _conv(out, f"{e}/conv_in", 3, 128, 3)
    for i, (cin, cout) in enumerate(VAE_ENCODER_BLOCKS):
        b = f"{e}/blocks/{i}"
        _resnet(out, f"{b}/res1", cin, cout)
        _resnet(out, f"{b}/res2", cout, cout)
        if i != len(VAE_ENCODER_BLOCKS) - 1:
            _conv(out, f"{b}/downsampler/conv", cout, cout, 3)  # PaddedConv2d (0,1,0,1), stride 2 (:229-236)
    _resnet(out, f"{e}/mid/block_1", 512, 512)
    a = f"{e}/mid/attn"
    _norm(out, f"{a}/norm", 512)
    for n in ("q", "k", "v", "proj_out"):
        _conv(out, f"{a}/{n}", 512, 512, 1)
    _resnet(out, f"{e}/mid/block_2", 512, 512)
    _norm(out, f"{e}/norm_out", 512)
    _conv(out, f"{e}/conv_out", 512, 8, 3)
    _conv(out, f"{prefix}/quant_conv", 8, 8, 1)
    return out


CLIP_VOCAB, CLIP_STATE, CLIP_HEADS, CLIP_CTX, CLIP_LAYERS = 49408, 768, 12, 77, 12  # stablediffusion/mod.rs:29


def clip_params(prefix="clip"):
    """CLIP text transformer (SURVEY §8f row f1): src/model/clip/mod.rs:25-44, names from src/model/clip/load.rs:15-81."""
    out = []
    out.append((f"{prefix}/token_embedding/weight", (CLIP_VOCAB, CLIP_STATE), "emb", CLIP_STATE))
    out.append((f"{prefix}/position_embedding/weight", (CLIP_CTX, CLIP_STATE), "emb", CLIP_STATE))
    for i in range(CLIP_LAYERS):
        b = f"{prefix}/blocks/{i}"
        _norm(out, f"{b}/attn_ln", CLIP_STATE)
        for n in ("query", "key", "value", "out"):
            _lin(out, f"{b}/attn/{n}", CLIP_STATE, CLIP_STATE)
        _norm(out, f"{b}/mlp_ln", CLIP_STATE)
        _lin(out, f"{b}/mlp/fc1", CLIP_STATE, 4 * CLIP_STATE)
        _lin(out, f"{b}/mlp/fc2", 4 * CLIP_STATE, CLIP_STATE)
    _norm(out, f"{prefix}/layer_norm", CLIP_STATE)
    return out


def all_params(inpaint=False, pix2pix=False):
    """The registry in sdb_create's order; inpaint=True: sdb_create_inpaint's (a 9-channel unet/input_blocks/conv);
    pix2pix=True: sdb_create_pix2pix's (an 8-channel one)."""
    if inpaint and pix2pix:
        raise ValueError("a registry is either the inpainting (inpaint=True) or the InstructPix2Pix (pix2pix=True) one")
    return (unet_params(in_channels=9 if inpaint else 4, pix2pix=pix2pix) + vae_decoder_params() + clip_params() +
            vae_encoder_params())


def conv_in_width_params(width):
    """all_params of the registry whose unet/input_blocks/conv/weight has `width` input channels (4, 8 or 9)."""
    if width not in (4, 8, 9):
        raise ValueError(f"no registry has a {width}-channel conv_in (4, 8 or 9)")
    return all_params(inpaint=width == 9, pix2pix=width == 8)


if __name__ == "__main__":
    import math
    ps = all_params()
    tot = sum(math.prod(s) for _, s, _, _ in ps)
    print(len(ps), "tensors", tot / 1e6, "M params")
