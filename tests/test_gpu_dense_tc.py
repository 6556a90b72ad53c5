"""Tensor-core dense path (wgmma + TMA, split-bf16) against the fp32 oracle.

passes=3 (hi*hi + hi*lo + lo*hi in one fp32 accumulator) must be fp32-grade: asserted at
5e-5 of the output scale, 20x inside the north-star 1e-3.  passes=1 is plain bf16 (~1e-2)."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets, ops
from oracle import oracle
from tests import helpers as H

pytestmark = pytest.mark.gpu


def dev(a, device):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def test_split_rows_layout_and_accuracy(device):
    rng = np.random.default_rng(0)
    M, K = 300, 415
    x = (rng.standard_normal((M, K)) * 3).astype(np.float32)
    s = ops.split_rows(dev(x, device))
    Kp = ops.tc_padded_k(K)
    assert tuple(s.shape) == (M, 2 * Kp) and Kp == 448
    hi, lo = s[:, :Kp].float().cpu().numpy(), s[:, Kp:].float().cpu().numpy()
    assert np.all(hi[:, K:] == 0) and np.all(lo[:, K:] == 0)
    rec = hi[:, :K] + lo[:, :K]
    assert np.max(np.abs(rec - x) / np.maximum(np.abs(x), 1e-30)) < 2.0 ** -15


@pytest.mark.parametrize("M,K,N", [(1000, 415, 128), (128, 64, 32), (5, 13, 128), (777, 128, 64), (4096, 32, 1),
                                   (300, 1037, 1037), (129, 200, 256), (64, 512, 272)])
@pytest.mark.parametrize("act", ["relu", "sigmoid"])
def test_dense_tc_matches_fp32_oracle(device, M, K, N, act):
    rng = np.random.default_rng(1)
    x = rng.standard_normal((M, K)).astype(np.float32)
    W = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    b = (rng.standard_normal(N) * 0.1).astype(np.float32)
    a = ops.split_rows(dev(x, device))
    w = ops.split_weights(dev(W, device))
    out = torch.full((M, N), 7.0, dtype=torch.float32, device=device)
    ops.dense_tc(a, K, w, N, dev(b, device), act, passes=3, out_f32=out)
    ref = oracle.dense(x, W, b, act)
    assert H.rel_err(out.cpu().numpy(), ref) < 5e-5
    out1 = torch.empty((M, N), dtype=torch.float32, device=device)
    ops.dense_tc(a, K, w, N, dev(b, device), act, passes=1, out_f32=out1)
    assert H.rel_err(out1.cpu().numpy(), ref) < 3e-2


def test_dense_tc_split_output_feeds_next_layer(device):
    rng = np.random.default_rng(2)
    M, K, N = 513, 415, 128
    x = rng.standard_normal((M, K)).astype(np.float32)
    W = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    a = ops.split_rows(dev(x, device))
    nxt = torch.zeros((M, 2 * ops.tc_padded_k(N)), dtype=torch.bfloat16, device=device)
    out = torch.empty((M, N), dtype=torch.float32, device=device)
    ops.dense_tc(a, K, ops.split_weights(dev(W, device)), N, None, "relu", out_f32=out, out_split=nxt)
    Kp = ops.tc_padded_k(N)
    rec = nxt[:, :N].float() + nxt[:, Kp:Kp + N].float()
    assert torch.allclose(rec, out, rtol=2.0 ** -14, atol=1e-7)
    assert torch.equal(ops.split_rows(out), nxt)  # identical to splitting the fp32 output


def test_dense_chain_tc_vs_fp32_engine(device):
    mm.set_seed(3)
    rng = np.random.default_rng(3)
    x = dev(rng.standard_normal((2000, 415)).astype(np.float32), device)
    mlp = mm.MLPBlock([128, 64, 32])
    mm.set_dense_engine("tc")
    try:
        y_tc = mlp(x).cpu().numpy()
        mm.set_dense_engine("fp32")
        y_32 = mlp(x).cpu().numpy()
    finally:
        mm.set_dense_engine("auto")
    ref = oracle.mlp(x.cpu().numpy(), H.mlp_layers(mlp))
    assert H.rel_err(y_32, ref) < 2e-5
    assert H.rel_err(y_tc, ref) < 5e-5


def test_cross_block_tc_matches_oracle(device):
    mm.set_seed(4)
    rng = np.random.default_rng(4)
    B, d = 700, 1037
    x0 = rng.standard_normal((B, d)).astype(np.float32)
    cross = mm.CrossBlock(3)
    for eng in ("tc", "fp32"):
        mm.set_dense_engine(eng)
        try:
            y = cross(dev(x0, device)).cpu().numpy()
        finally:
            mm.set_dense_engine("auto")
        layers = [{"kernel": H.to_numpy(l.dense.kernel), "bias": H.to_numpy(l.dense.bias)} for l in cross.cross_layers]
        ref = oracle.cross_layers(x0, layers)
        assert H.rel_err(y, ref) < 5e-5, eng


def test_dense_tc_argument_errors(device):
    a = torch.zeros((128, 128), dtype=torch.bfloat16, device=device)
    w = torch.zeros((16, 128), dtype=torch.bfloat16, device=device)
    out = torch.zeros((128, 1), dtype=torch.float32, device=device)
    with pytest.raises(ValueError, match="passes"):
        ops.dense_tc(a, 64, w, 1, None, "relu", passes=2, out_f32=out)
    with pytest.raises(ValueError, match="no output"):
        ops.dense_tc(a, 64, w, 1, None, "relu")


@pytest.mark.parametrize("N,head_act", [(32, "sigmoid"), (16, "linear"), (24, "relu")])
def test_dense_tc_fused_head(device, N, head_act):
    rng = np.random.default_rng(6)
    M, K = 3000, 64
    x = rng.standard_normal((M, K)).astype(np.float32)
    W = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    b = (rng.standard_normal(N) * 0.1).astype(np.float32)
    hw = (rng.standard_normal((N, 1)) * 0.3).astype(np.float32)
    out = torch.empty((M, 1), dtype=torch.float32, device=device)
    ops.dense_tc_head(ops.split_rows(dev(x, device)), K, ops.split_weights(dev(W, device)), N, dev(b, device), "relu",
                      dev(hw.reshape(-1), device), 0.25, head_act, out)
    ref = oracle.dense(oracle.dense(x, W, b, "relu"), hw, np.array([0.25], np.float32), head_act)
    assert H.rel_err(out.cpu().numpy(), ref) < 5e-5


def test_mlp_plus_head_chain_equals_unfused(device):
    mm.set_seed(8)
    rng = np.random.default_rng(8)
    x = dev(rng.standard_normal((1500, 415)).astype(np.float32), device)
    mlp = mm.MLPBlock([128, 64, 32])
    head = mm.BinaryOutput("label")
    from models_b200.blocks import run_dense_chain

    fused = run_dense_chain(x, mlp.dense_layers + [head.to_call]).cpu().numpy()
    body = mlp(x)
    unfused = head(body).cpu().numpy()
    ref = oracle.dense(oracle.mlp(x.cpu().numpy(), H.mlp_layers(mlp)), H.to_numpy(head.to_call.kernel),
                       H.to_numpy(head.to_call.bias), "sigmoid")
    assert H.rel_err(fused, ref) < 5e-5 and H.rel_err(unfused, ref) < 5e-5


@pytest.mark.parametrize("lo,hi", [(0, 300), (2**33, 2**33 + 300), (-150, 150)])
def test_scorer_false_negative_mask_narrow_and_wide_ids(device, lo, hi):
    """The scorer epilogue compares 32-bit low words when every id of the tile fits (fast path) and falls back
    to the exact 64-bit compare otherwise; ids that agree in the low word only must not be masked."""
    rng = np.random.default_rng(30)
    B, D = 700, 64
    q = rng.standard_normal((B, D)).astype(np.float32)
    it = rng.standard_normal((B, D)).astype(np.float32)
    ids = rng.integers(lo, hi, B).astype(np.int64)       # many duplicates -> many false negatives
    ids[5], ids[6] = 7 + lo, 7 + lo + 2**32              # same low word, different id
    dq, dit, dids = dev(q, device), dev(it, device), dev(ids, device)
    out = torch.empty((B, 4 + B), dtype=torch.float32, device=device)[:, 3:4 + B]
    ops.inbatch_scores(dq, dit, dit, out, pos_ids=dids, neg_ids=dids)
    got = out.cpu().numpy()
    fns = np.float32(oracle.MIN_FLOAT)
    same = ids[:, None] == ids[None, :]
    assert np.array_equal(got[:, 1:] == fns, same)
    assert not same[5, 6] and got[5, 1 + 6] != fns
    ref = (q.astype(np.float64) @ it.astype(np.float64).T)
    np.testing.assert_allclose(got[:, 1:][~same], ref[~same], rtol=1e-4, atol=5e-4)
