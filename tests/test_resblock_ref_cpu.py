"""The fp64 ResBlock reference of tests/test_resblock_gpu.py equals the oracle's res_block / resnet_block (the op definitions the
whole-model goldens are made with), on parameter dicts built from the same arrays, without operand-rounding emulation."""
import numpy as np
import pytest
import torch

import test_resblock_gpu as R
from oracle import sd_oracle as O


def small_block(rng, c0, c1, co, skip, emb):
    cin = c0 + c1
    d = {"x0": R.activation(rng, 2, c0, 8, 8, 1.0, 4.0), "x1": R.activation(rng, 2, c1, 8, 8, 2.5, -3.0) if c1 else None}
    d["norm1"] = (1 + 0.1 * rng.standard_normal(cin), 0.1 * rng.standard_normal(cin))
    d["conv1"] = (rng.standard_normal((co, cin, 3, 3)) / np.sqrt(9 * cin), 0.1 * rng.standard_normal(co))
    d["norm2"] = (1 + 0.1 * rng.standard_normal(co), 0.1 * rng.standard_normal(co))
    d["conv2"] = (rng.standard_normal((co, co, 3, 3)) / np.sqrt(9 * co), 0.1 * rng.standard_normal(co))
    d["skip"] = (rng.standard_normal((co, cin, 1, 1)) / np.sqrt(cin), 0.1 * rng.standard_normal(co)) if skip else None
    d["emb_bias"] = None
    x = torch.from_numpy(np.concatenate([d["x0"]] + ([d["x1"]] if c1 else []), axis=1).astype(np.float64))
    return d, x


@pytest.mark.parametrize("c0,c1,co,skip", [(64, 32, 64, True), (64, 0, 64, False), (64, 64, 96, True)])
def test_reference_equals_oracle_res_block(c0, c1, co, skip):
    rng = np.random.default_rng(c0 + c1 + co)
    d, x = small_block(rng, c0, c1, co, skip, True)
    emb = rng.standard_normal((1, 64))
    lw, lb = rng.standard_normal((64, co)) / 8, 0.1 * rng.standard_normal(co)
    # what the model hands the block: conv_in.bias + lin_embed(silu(emb)), one row for the whole batch
    d["emb_bias"] = d["conv1"][1] + (emb * (1 / (1 + np.exp(-emb)))) @ lw + lb
    d["emb_bias"] = d["emb_bias"][0]
    arrays = {"b/norm_in/weight": d["norm1"][0], "b/norm_in/bias": d["norm1"][1], "b/conv_in/weight": d["conv1"][0],
              "b/conv_in/bias": d["conv1"][1], "b/lin_embed/weight": lw, "b/lin_embed/bias": lb,
              "b/norm_out/weight": d["norm2"][0], "b/norm_out/bias": d["norm2"][1], "b/conv_out/weight": d["conv2"][0],
              "b/conv_out/bias": d["conv2"][1]}
    if skip:
        arrays.update({"b/skip_connection/weight": d["skip"][0], "b/skip_connection/bias": d["skip"][1]})
    P = O.Params(arrays, dtype=torch.float64)
    with torch.no_grad():
        ref = R.ref_block(x, d, 3).numpy()
        ora = O.res_block(P, "b", x, torch.from_numpy(emb)).numpy()
    assert np.abs(ref - ora).max() <= 1e-12 * np.abs(ora).max()


@pytest.mark.parametrize("c0,co,skip", [(64, 64, False), (128, 64, True)])
def test_reference_equals_oracle_resnet_block(c0, co, skip):
    rng = np.random.default_rng(c0 + co + 7)
    d, x = small_block(rng, c0, 0, co, skip, False)
    arrays = {"b/norm1/weight": d["norm1"][0], "b/norm1/bias": d["norm1"][1], "b/conv1/weight": d["conv1"][0],
              "b/conv1/bias": d["conv1"][1], "b/norm2/weight": d["norm2"][0], "b/norm2/bias": d["norm2"][1],
              "b/conv2/weight": d["conv2"][0], "b/conv2/bias": d["conv2"][1]}
    if skip:
        arrays.update({"b/nin_shortcut/weight": d["skip"][0], "b/nin_shortcut/bias": d["skip"][1]})
    P = O.Params(arrays, dtype=torch.float64)
    with torch.no_grad():
        ref = R.ref_block(x, d, 3).numpy()
        ora = O.resnet_block(P, "b", x).numpy()
    assert np.abs(ref - ora).max() <= 1e-12 * np.abs(ora).max()


def test_reference_rounding_matches_oracle_emulation():
    """the 1-pass reference (GroupNorm outputs, raw skip input and weights rounded to fp16) is the oracle's fp16 emulation of
    the conv operands"""
    rng = np.random.default_rng(5)
    d, x = small_block(rng, 64, 64, 64, True, False)
    arrays = {"b/norm1/weight": d["norm1"][0], "b/norm1/bias": d["norm1"][1], "b/conv1/weight": d["conv1"][0],
              "b/conv1/bias": d["conv1"][1], "b/norm2/weight": d["norm2"][0], "b/norm2/bias": d["norm2"][1],
              "b/conv2/weight": d["conv2"][0], "b/conv2/bias": d["conv2"][1], "b/nin_shortcut/weight": d["skip"][0],
              "b/nin_shortcut/bias": d["skip"][1]}
    P = O.Params(arrays, dtype=torch.float64)
    saved = dict(O._EMU)
    try:
        O.set_emulation("fp16", "AW")
        with torch.no_grad():
            ora = O.resnet_block(P, "b", x).numpy()
    finally:
        O._EMU.clear()
        O._EMU.update(saved)
    with torch.no_grad():
        ref = R.ref_block(x, d, 1).numpy()
    assert np.abs(ref - ora).max() <= 1e-12 * np.abs(ora).max()
