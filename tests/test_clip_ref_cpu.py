"""The fp64 block reference of tests/test_clip_blocks_gpu.py (tests/clip_oracle.py), chained in the encoder's order, reproduces
the oracle's clip_forward (the op definitions the CLIP goldens are made with); the value-bias fold finalize_weights applies is an
identity; and synth.realistic_stats reshapes the CLIP weights as it does the UNet's. A reference that drifted from the model, or a
realistic-statistics set that left the text encoder i.i.d., fails here without a GPU."""
import os

import numpy as np
import pytest
import torch

import clip_oracle as CO
from oracle import sd_oracle as O
from stable_diffusion_burn_b200 import synth, topology


@pytest.fixture(scope="module")
def raw():
    torch.set_num_threads(os.cpu_count() or 1)
    return synth.make_params(0, which=topology.clip_params())


@pytest.fixture(scope="module")
def W(raw):
    return {k: torch.from_numpy(v.astype(np.float64)) for k, v in raw.items() if k.startswith("clip/")}


def close(a, b, bar=1e-10):
    return float((a - b).abs().max() / b.abs().max()) <= bar


def tokens(n, L, seed):
    t = np.random.default_rng(seed).integers(0, 49406, (n, L))
    t[:, 0] = 49406  # start of text
    return torch.from_numpy(t)


@pytest.mark.parametrize("n,L", [(1, 1), (2, 11), (1, 77)])
def test_chained_blocks_reproduce_clip_forward(W, n, L):
    tok = tokens(n, L, 100 * n + L)
    P = O.Params({k: v.numpy() for k, v in W.items()}, dtype=torch.float64)
    with torch.no_grad():
        want = O.clip_forward(P, tok)
        x = CO.embed(W["clip/token_embedding/weight"], W["clip/position_embedding/weight"], tok)
        for i in range(CO.LAYERS):
            x = CO.block(W, i, x)["out"]
        got = CO.final_layer_norm(W, x)
    assert close(got, want), float((got - want).abs().max())


def test_value_bias_fold_is_an_identity(W):
    """P (V + 1 b_v^T) = P V + 1 b_v^T because every row of P sums to one: folding b_v into the out-projection bias (as
    pack_clip_block does) changes nothing but the place the bias enters. A value bias 30x the synthetic one makes it count."""
    Wb = dict(W)
    Wb["clip/blocks/3/attn/value/bias"] = 30 * W["clip/blocks/3/attn/value/bias"]
    x = torch.from_numpy(np.random.default_rng(5).standard_normal((2, 19, 768)))
    with torch.no_grad():
        folded = CO.block(Wb, 3, x, fold_value_bias=True)
        plain = CO.block(Wb, 3, x, fold_value_bias=False)
        dropped = CO.block(Wb, 3, x, fold_value_bias=True)["x_attn"] - (Wb["clip/blocks/3/attn/value/bias"] @
                                                                        Wb["clip/blocks/3/attn/out/weight"])
    assert close(folded["x_attn"], plain["x_attn"], 1e-12) and close(folded["out"], plain["out"], 1e-12)
    # the fold carries weight: the same block without it is visibly different
    assert not close(dropped, plain["x_attn"], 1e-3)


def test_realistic_stats_reshape_the_clip_weights(raw):
    clip = {k: v for k, v in raw.items() if k.startswith("clip/")}
    rs = synth.realistic_stats(clip)
    for name in ("clip/token_embedding/weight", "clip/position_embedding/weight"):
        assert np.array_equal(rs[name], clip[name]), name
    norms = [f"clip/blocks/{i}/{ln}" for i in range(12) for ln in ("attn_ln", "mlp_ln")] + ["clip/layer_norm"]
    for nm in norms:
        g, b = rs[f"{nm}/weight"], rs[f"{nm}/bias"]
        assert g.min() >= 0.4 and g.max() <= 1.6 and g.std() > 0.3, nm
        assert np.abs(b).max() <= 0.4 and b.std() > 0.15, nm
    for i in (0, 11):
        b = f"clip/blocks/{i}"
        for lin, gain in (("attn/query", 1.7), ("attn/key", 1.7), ("attn/value", 1.0), ("attn/out", 1.0), ("mlp/fc1", 1.0),
                          ("mlp/fc2", 1.0)):
            w0, w1 = clip[f"{b}/{lin}/weight"].astype(np.float64), rs[f"{b}/{lin}/weight"].astype(np.float64)
            g = np.sqrt((w1 ** 2).sum(0) / (w0 ** 2).sum(0))  # per output column ([in, out] layout)
            assert abs(np.sqrt(np.mean(g ** 2)) - gain) < 1e-3 * gain, (b, lin)
            assert g.max() / g.min() > 3, (b, lin)  # log-normal gains: outlier channels
            assert np.allclose(rs[f"{b}/{lin}/bias"], 3 * clip[f"{b}/{lin}/bias"]), (b, lin)
