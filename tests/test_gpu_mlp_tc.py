"""Whole-tower MLP kernel (mm_mlp_tc: layer 1 TMA-fed wgmma, layers 2..n on chip with the A operand
in registers) against the fp64 NumPy chain of oracle.dense — the reference's MLPBlock
(merlin/models/tf/blocks/mlp.py:97-139) + BinaryOutput Dense(1) (outputs/classification.py:114).
Tolerance: 5e-5 of the output scale per layer (3-pass split-bf16), 20x inside the north-star 1e-3."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import blocks, ops
from oracle import oracle
from tests import helpers as H

pytestmark = pytest.mark.gpu


def dev(a, device):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def _tower(rng, K, widths):
    Ws, bs, k = [], [], K
    for n in widths:
        Ws.append((rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32))
        bs.append((rng.standard_normal(n) * 0.1).astype(np.float32))
        k = n
    return Ws, bs


def _oracle_chain(x, Ws, bs, acts):
    for W, b, a in zip(Ws, bs, acts):
        x = oracle.dense(x, W, b, a)
    return x


@pytest.mark.parametrize("M,K,widths", [
    (65536 // 16, 415, [128, 64, 32]),      # README top tower
    (1000, 13, [128, 64]),                  # README bottom tower
    (777, 415, [128, 64]),
    (129, 69, [32, 128, 64, 128]),          # wide chain: 96 KB of resident weights
    (5, 200, [100, 50, 20]),                # widths that are not multiples of 16 / 32
    (300, 64, [16, 16]),
    (4096, 129, [96, 48, 112, 8]),
])
@pytest.mark.parametrize("acts", ["relu", "mixed"])
def test_mlp_tc_matches_oracle_chain(device, M, K, widths, acts):
    rng = np.random.default_rng(11)
    x = rng.standard_normal((M, K)).astype(np.float32)
    Ws, bs = _tower(rng, K, widths)
    names = ["relu"] * len(widths) if acts == "relu" else (["tanh", "relu", "sigmoid", "linear"] * 2)[: len(widths)]
    a = ops.split_rows(dev(x, device))
    out = torch.full((M, widths[-1]), 7.0, dtype=torch.float32, device=device)
    ops.mlp_tc(a, K, [ops.split_weights(dev(W, device)) for W in Ws], widths, [dev(b, device) for b in bs], names, out=out)
    ref = _oracle_chain(x, Ws, bs, names)
    assert H.rel_err(out.cpu().numpy(), ref) < 5e-5 * len(widths)


@pytest.mark.parametrize("head_act", ["sigmoid", "linear"])
@pytest.mark.parametrize("widths", [[128, 64, 32], [64, 16], [128, 24]])
def test_mlp_tc_fused_head(device, widths, head_act):
    rng = np.random.default_rng(12)
    M, K = 3000, 415
    x = rng.standard_normal((M, K)).astype(np.float32)
    Ws, bs = _tower(rng, K, widths)
    hw = (rng.standard_normal((widths[-1], 1)) / np.sqrt(widths[-1])).astype(np.float32)
    hb = np.float32(0.25)
    a = ops.split_rows(dev(x, device))
    w = [ops.split_weights(dev(W, device)) for W in Ws]
    b = [dev(v, device) for v in bs]
    acts = ["relu"] * len(widths)
    head_out = torch.empty((M, 1), dtype=torch.float32, device=device)
    body = torch.empty((M, widths[-1]), dtype=torch.float32, device=device)
    ops.mlp_tc(a, K, w, widths, b, acts, out=body, head_w=dev(hw.reshape(-1), device), head_b=float(hb), head_act=head_act,
               head_out=head_out)
    h = _oracle_chain(x, Ws, bs, acts)
    assert H.rel_err(body.cpu().numpy(), h) < 2e-4
    ref = oracle.dense(h, hw, np.array([hb], np.float32), head_act)
    assert H.rel_err(head_out.cpu().numpy(), ref) < 2e-4
    only_head = torch.empty((M, 1), dtype=torch.float32, device=device)
    ops.mlp_tc(a, K, w, widths, b, acts, head_w=dev(hw.reshape(-1), device), head_b=float(hb), head_act=head_act,
               head_out=only_head)
    assert torch.equal(only_head, head_out)


def test_mlp_tc_equals_layer_by_layer_tc(device):
    """Same arithmetic as the per-layer mm_dense_tc chain (3-pass split-bf16, fp32 accumulate): the
    fused tower must agree with it to the last few ulps, on many tiles (persistent CTAs wrap around)."""
    rng = np.random.default_rng(13)
    M, K, widths = 132 * 128 * 2 + 77, 415, [128, 64, 32]
    x = rng.standard_normal((M, K)).astype(np.float32)
    Ws, bs = _tower(rng, K, widths)
    a = ops.split_rows(dev(x, device))
    w = [ops.split_weights(dev(W, device)) for W in Ws]
    b = [dev(v, device) for v in bs]
    fused = torch.empty((M, 32), dtype=torch.float32, device=device)
    ops.mlp_tc(a, K, w, widths, b, ["relu"] * 3, out=fused)
    cur, k = a, K
    for i, n in enumerate(widths):
        last = i == len(widths) - 1
        nxt = None if last else torch.zeros((M, 2 * ops.tc_padded_k(n)), dtype=torch.bfloat16, device=device)
        o = torch.empty((M, n), dtype=torch.float32, device=device) if last else None
        ops.dense_tc(cur, k, w[i], n, b[i], "relu", passes=3, out_f32=o, out_split=nxt)
        cur, k = nxt, n
    # same operands, different accumulation order of the three passes: a few fp32 ulps per layer
    diff = float((fused - o).abs().max())
    assert diff < 2e-5, diff
    again = torch.empty_like(fused)
    ops.mlp_tc(a, K, w, widths, b, ["relu"] * 3, out=again)
    assert torch.equal(again, fused)  # deterministic


def test_mlp_block_uses_fused_tower_and_matches_fp32_engine(device):
    rng = np.random.default_rng(14)
    x = dev(rng.standard_normal((2049, 415)).astype(np.float32), device)
    mm.set_seed(5)
    mlp = mm.MLPBlock([128, 64, 32])
    got = mlp(x)
    assert blocks.last_dense_path() == "mlp_tc"
    blocks.set_dense_engine("fp32")
    try:
        ref = mlp(x)
    finally:
        blocks.set_dense_engine("auto")
    assert H.rel_err(got.cpu().numpy(), ref.cpu().numpy()) < 2e-4
    wide = mm.MLPBlock([256, 64])  # first width > 128: layer-by-layer path
    wide(x)
    assert blocks.last_dense_path() == "dense_tc"


def test_mlp_tc_argument_errors(device):
    a = ops.split_rows(torch.zeros((8, 13), device=device))
    w1 = ops.split_weights(torch.zeros((13, 128), device=device))
    w2 = ops.split_weights(torch.zeros((128, 64), device=device))
    out = torch.empty((8, 64), device=device)
    with pytest.raises(ValueError):
        ops.mlp_tc(a, 13, [w1, w2], [128, 64], [None], ["relu", "relu"], out=out)
    with pytest.raises(ValueError):
        ops.mlp_tc(a, 13, [w1, w1], [128, 64], [None, None], ["relu", "relu"], out=out)  # wrong layout for layer 2
    with pytest.raises(ValueError, match="no output"):
        ops.mlp_tc(a, 13, [w1, w2], [128, 64], [None, None], ["relu", "relu"])
    assert not ops.mlp_tc_supported(13, [256, 64]) and not ops.mlp_tc_supported(13, [128])
    assert ops.mlp_tc_supported(415, [128, 64, 32], head=True) and not ops.mlp_tc_supported(415, [128, 64], head=True)
    assert not ops.mlp_tc_supported(69, [128, 128, 128, 128])  # 192 KB of resident weights do not fit
    with pytest.raises(ValueError, match="does not fit"):
        w = ops.split_weights(torch.zeros((128, 128), device=device))
        ops.mlp_tc(ops.split_rows(torch.zeros((8, 128), device=device)), 128, [w] * 4, [128] * 4, [None] * 4, ["relu"] * 4,
                   out=torch.empty((8, 128), device=device))


def test_concat_split_equals_concat_then_split(device):
    """mm_concat_split == mm_split_rows(mm_concat_columns(...)) bit for bit, mixed dtypes / widths / strides."""
    rng = np.random.default_rng(15)
    B = 1000
    wide = dev(rng.standard_normal((B, 40)).astype(np.float32), device)
    pieces = [dev(rng.standard_normal(B).astype(np.float32), device),
              dev(rng.integers(-5, 5, B).astype(np.int64), device),
              wide[:, 3:20],                                   # strided view, unit inner stride
              dev(rng.standard_normal((B, 1)).astype(np.float64), device),
              dev(rng.integers(0, 100, (B, 2)).astype(np.int32), device)]
    a, K = ops.concat_split(pieces)
    assert K == 1 + 1 + 17 + 1 + 2 and tuple(a.shape) == (B, 2 * 64)
    ref = torch.empty((B, K), dtype=torch.float32, device=device)
    ops.concat_columns(pieces, ref)
    assert torch.equal(a, ops.split_rows(ref))
    thirteen = [dev(rng.random(B).astype(np.float32), device) for _ in range(13)]
    a13, K13 = ops.concat_split(thirteen)
    ref13 = torch.empty((B, 13), dtype=torch.float32, device=device)
    ops.concat_columns(thirteen, ref13)
    assert K13 == 13 and torch.equal(a13, ops.split_rows(ref13))
    assert not ops.concat_split_supported([wide] * 9)  # 360 columns > 320


def test_mlp_block_on_feature_dict_uses_concat_split(device):
    rng = np.random.default_rng(16)
    feats = {f"I{i}": dev(rng.random(777).astype(np.float32), device) for i in range(1, 14)}
    mm.set_seed(6)
    mlp = mm.MLPBlock([128, 64])
    blocks._SMALL_TOWER[0] = False  # the narrow-input kernel (mm_tower2_small) would take this tower: test the TMA tower path
    try:
        got = mlp(feats)
    finally:
        blocks._SMALL_TOWER[0] = True
    assert blocks.last_dense_path() == "mlp_tc"
    x = torch.stack([feats[k] for k in sorted(feats)], dim=1)  # ConcatFeatures order: I1, I10, ..., I13, I2, ...
    layers = [{"kernel": l.kernel.cpu().numpy(), "bias": l.bias.cpu().numpy(), "activation": l.activation} for l in mlp.dense_layers]
    ref = x.cpu().numpy()
    for l in layers:
        ref = oracle.dense(ref, l["kernel"], l["bias"], l["activation"])
    assert H.rel_err(got.cpu().numpy(), ref) < 1e-4


@pytest.mark.parametrize("dims,K,acts", [([128, 64], 13, "relu"), ([64, 32], 5, ["tanh", "linear"]), ([32, 16], 16, ["gelu", "sigmoid"]),
                                         ([128, 16], 1, "relu")])
@pytest.mark.parametrize("B", [1, 17, 4099])
def test_tower2_small_matches_oracle_and_tower_kernel(device, dims, K, acts, B):
    """mm_tower2_small: <= 16 scalar columns (mixed dtypes, (B,) and (B,1) and one (B,2) piece) -> two dense layers, fp32 rows and
    split-bf16 rows; against the oracle MLP over the sorted-name concat, and against the TMA/wgmma tower path."""
    import models_b200 as mm
    from models_b200 import blocks
    from oracle import oracle

    rng = np.random.default_rng(K * 100 + B)
    mm.set_seed(K)
    cols = {}
    k = 0
    while k < K:
        name = f"I{k}"
        if k == 2 and K - k >= 2:
            cols[name] = rng.standard_normal((B, 2)).astype(np.float32)
            k += 2
        elif k % 4 == 1:
            cols[name] = rng.integers(-3, 4, B).astype(np.int64)
            k += 1
        elif k % 4 == 3:
            cols[name] = rng.standard_normal((B, 1)).astype(np.float64)
            k += 1
        else:
            cols[name] = rng.standard_normal(B).astype(np.float32)
            k += 1
    mlp = mm.MLPBlock(dims, activation=acts)
    dcols = {n: torch.from_numpy(v).to(device) for n, v in cols.items()}
    got = mlp(dcols).cpu().numpy()
    assert blocks._LAST_PATH[0] == "tower2_small"
    x = oracle.concat_features({n: np.asarray(v, dtype=np.float32) for n, v in cols.items()})
    assert x.shape == (B, K)
    layers = [{"kernel": l.kernel.cpu().numpy(), "bias": l.bias.cpu().numpy(), "activation": l.activation} for l in mlp.dense_layers]
    ref = oracle.mlp(x, layers)
    np.testing.assert_allclose(got, ref, rtol=2e-4, atol=2e-5)
    op = mlp(dcols, operand_out=True)
    assert op.dtype == torch.bfloat16 and tuple(op.shape) == (B, 2 * dims[-1])
    assert torch.equal(op.view(torch.int16), ops.split_rows(torch.from_numpy(got).to(device))[:, : 2 * dims[-1]].view(torch.int16)) or dims[-1] % 64
    rec = op.float().cpu().numpy()
    np.testing.assert_allclose(rec[:, : dims[-1]] + rec[:, dims[-1]:], got, rtol=2e-5, atol=1e-6)  # hi + lo carries 16-17 bits
    blocks._SMALL_TOWER[0] = False
    try:
        other = mlp(dcols).cpu().numpy()
        assert blocks._LAST_PATH[0] != "tower2_small"
    finally:
        blocks._SMALL_TOWER[0] = True
    np.testing.assert_allclose(got, other, rtol=1e-5, atol=1e-5)  # two fp32-grade paths: different accumulation order
