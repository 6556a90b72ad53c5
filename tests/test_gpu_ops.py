"""GPU parity of every C-ABI entry point against the CPU oracle (seeded inputs, oracle-sized).

Bars: bit-exact for gathered rows / integer work; fp32 results within rtol 1e-4 of the oracle
(the north-star tolerance for logits is 1e-3 relative; kernels on CUDA cores are held tighter).
"""
import numpy as np
import pytest
import torch

from models_b200 import ops
from oracle import oracle

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-4, 1e-5


def dev(a, device):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def test_init_uniform_hash_matches_host(device):
    n = 100_003
    w = torch.empty(n, dtype=torch.float32, device=device)
    ops.init_uniform_hash(w, seed=1234567, lo=-0.05, hi=0.05)
    ref = oracle.hash_uniform(np.arange(n), 1234567, -0.05, 0.05)
    assert np.array_equal(w.cpu().numpy(), ref)
    assert ref.min() >= -0.05 and ref.max() < 0.05 and abs(ref.mean()) < 1e-3


@pytest.mark.parametrize("idx_dtype", [np.int32, np.int64])
@pytest.mark.parametrize("dim", [64, 16, 128, 4, 8, 24, 7])
def test_gather_multi_bit_exact(device, idx_dtype, dim):
    rng = np.random.default_rng(0)
    B, T = 777, 5
    rows = [3, 100, 4097, 19, 1000]
    tables = [rng.standard_normal((r, dim)).astype(np.float32) for r in rows]
    idx = [rng.integers(0, r, B).astype(idx_dtype) for r in rows]
    slots = [3, 0, 4, 1, 2]
    out = torch.full((B, T * dim + 5), -7.0, dtype=torch.float32, device=device)
    oob = torch.zeros(1, dtype=torch.int32, device=device)
    ops.gather_multi([dev(t, device) for t in tables], [dev(i, device) for i in idx], [s * dim for s in slots], out, oob)
    got = out.cpu().numpy()
    for t in range(T):
        assert np.array_equal(got[:, slots[t] * dim:(slots[t] + 1) * dim], oracle.embedding_lookup(tables[t], idx[t]))
    assert np.all(got[:, T * dim:] == -7.0)  # columns outside the features are untouched
    assert int(oob.item()) == 0


def test_gather_multi_mixed_dims_concat_layout(device):
    rng = np.random.default_rng(1)
    B = 301
    dims = [8, 16, 120, 40]
    rows = [10, 200, 3000, 7]
    tables = [rng.standard_normal((r, d)).astype(np.float32) for r, d in zip(rows, dims)]
    idx = [rng.integers(0, r, B).astype(np.int32) for r in rows]
    cols = np.concatenate([[0], np.cumsum(dims)[:-1]]).tolist()
    out = torch.empty((B, sum(dims)), dtype=torch.float32, device=device)
    ops.gather_multi([dev(t, device) for t in tables], [dev(i, device) for i in idx], cols, out)
    ref = np.concatenate([oracle.embedding_lookup(t, i) for t, i in zip(tables, idx)], axis=1)
    assert np.array_equal(out.cpu().numpy(), ref)


def test_gather_multi_out_of_range_counts_and_zeroes(device):
    table = np.ones((10, 64), dtype=np.float32)
    idx = np.array([0, 9, 10, -1, 3], dtype=np.int64)
    out = torch.full((5, 64), 5.0, dtype=torch.float32, device=device)
    oob = torch.zeros(1, dtype=torch.int32, device=device)
    ops.gather_multi([dev(table, device)], [dev(idx, device)], [0], out, oob)
    got = out.cpu().numpy()
    assert int(oob.item()) == 2
    assert np.all(got[[0, 1, 4]] == 1.0) and np.all(got[[2, 3]] == 0.0)


def test_gather_multi_empty_batch_and_many_tables(device):
    rng = np.random.default_rng(2)
    out = torch.empty((0, 64), dtype=torch.float32, device=device)
    ops.gather_multi([dev(np.ones((3, 64), np.float32), device)], [torch.empty(0, dtype=torch.int32, device=device)], [0], out)
    T, B, D = 70, 64, 8  # > MM_MAX_TABLES: chunked launches
    tables = [rng.standard_normal((11, D)).astype(np.float32) for _ in range(T)]
    idx = [rng.integers(0, 11, B).astype(np.int32) for _ in range(T)]
    out = torch.empty((B, T * D), dtype=torch.float32, device=device)
    ops.gather_multi([dev(t, device) for t in tables], [dev(i, device) for i in idx], [t * D for t in range(T)], out)
    ref = np.concatenate([t[i] for t, i in zip(tables, idx)], axis=1)
    assert np.array_equal(out.cpu().numpy(), ref)


@pytest.mark.parametrize("combiner", ["mean", "sum", "sqrtn"])
@pytest.mark.parametrize("dim", [64, 20])
def test_gather_bag_matches_safe_embedding_lookup_sparse(device, combiner, dim):
    rng = np.random.default_rng(3)
    B, rows = 257, 19
    table = rng.standard_normal((rows, dim)).astype(np.float32)
    lens = rng.integers(0, 6, B)  # includes empty bags
    offsets = np.zeros(B + 1, dtype=np.int32)
    np.cumsum(lens, out=offsets[1:])
    values = rng.integers(-1, rows, offsets[-1]).astype(np.int32)  # includes ids < 0 (pruned)
    out = torch.full((B, dim + 3), 9.0, dtype=torch.float32, device=device)
    ops.gather_bag(dev(table, device), dev(values, device), dev(offsets, device), combiner, out, out_col=2)
    ref = oracle.embedding_bag(table, values, offsets, combiner)
    got = out.cpu().numpy()
    assert np.array_equal(got[:, 2:2 + dim], ref)  # same left-to-right fp32 order -> bit exact
    assert np.all(got[:, :2] == 9.0) and np.all(got[:, 2 + dim:] == 9.0)


@pytest.mark.parametrize("combiner", ["mean", "sum", "max"])
def test_gather_seq_matches_sequence_combiner(device, combiner):
    rng = np.random.default_rng(4)
    B, L, rows, dim = 130, 5, 50, 32
    table = rng.standard_normal((rows, dim)).astype(np.float32)
    ids = rng.integers(0, rows, (B, L)).astype(np.int64)
    out = torch.empty((B, dim), dtype=torch.float32, device=device)
    ops.gather_seq(dev(table, device), dev(ids, device), combiner, out)
    ref = oracle.sequence_combiner(oracle.embedding_lookup(table, ids), combiner)
    assert np.array_equal(out.cpu().numpy(), ref)


def test_concat_columns_sorted_cast(device):
    rng = np.random.default_rng(5)
    B = 1000
    d = {"I1": rng.random(B).astype(np.float32), "I10": rng.integers(0, 9, B).astype(np.int64),
         "I2": rng.random((B, 1)).astype(np.float64), "emb": rng.random((B, 300)).astype(np.float32),
         "a": rng.integers(-5, 5, (B, 3)).astype(np.int32)}
    keys = sorted(d)
    width = sum(1 if d[k].ndim == 1 else d[k].shape[1] for k in keys)
    out = torch.empty((B, width), dtype=torch.float32, device=device)
    ops.concat_columns([dev(d[k], device) for k in keys], out)
    assert np.array_equal(out.cpu().numpy(), oracle.concat_features(d))


def test_l2_normalize(device):
    rng = np.random.default_rng(6)
    x = rng.standard_normal((300, 64)).astype(np.float32)
    x[7] = 0.0
    got = ops.l2_normalize(dev(x, device)).cpu().numpy()
    nrm = np.sqrt(np.maximum((x * x).sum(-1, keepdims=True), 1e-12))
    np.testing.assert_allclose(got, x / nrm, rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(np.linalg.norm(got[:7], axis=1), 1.0, rtol=1e-5)
    assert np.all(got[7] == 0.0)


@pytest.mark.parametrize("F,D", [(27, 64), (3, 16), (8, 128), (40, 8), (2, 4), (1, 64)])
@pytest.mark.parametrize("self_inter", [False, True])
def test_dot_interaction_matches_oracle(device, F, D, self_inter):
    rng = np.random.default_rng(7)
    B = 203
    x = rng.standard_normal((B, F, D)).astype(np.float32)
    n = F * (F + 1) // 2 if self_inter else F * (F - 1) // 2
    out = torch.full((B, n + 2), 3.0, dtype=torch.float32, device=device)
    ops.dot_interaction(dev(x, device), out, self_interaction=self_inter)
    ref = oracle.dot_interaction(x, self_inter)
    assert ref.shape == (B, n)
    got = out.cpu().numpy()
    # fast path = 3-pass split-bf16 on tensor cores: error ~ 2^-16 * sum|x_k y_k| (absolute)
    np.testing.assert_allclose(got[:, :n], ref, rtol=RTOL, atol=2e-4 * max(1.0, np.sqrt(D / 64)))
    assert np.all(got[:, n:] == 3.0)


def test_dot_interaction_with_prefix_is_bottom_first(device):
    rng = np.random.default_rng(8)
    B, F, D = 100, 27, 64
    x = rng.standard_normal((B, F, D)).astype(np.float32)
    bottom = x[:, 26].copy()
    out = torch.empty((B, D + F * (F - 1) // 2), dtype=torch.float32, device=device)
    ops.dot_interaction(dev(x, device), out, prefix=dev(bottom, device))
    got = out.cpu().numpy()
    assert np.array_equal(got[:, :D], bottom)
    np.testing.assert_allclose(got[:, D:], oracle.dot_interaction(x), rtol=RTOL, atol=2e-4)


@pytest.mark.parametrize("act", ["relu", "linear", "sigmoid", "tanh", "selu", "elu", "gelu"])
def test_dense_fp32_activations(device, act):
    rng = np.random.default_rng(10)
    B, K, N = 300, 415, 128
    x = rng.standard_normal((B, K)).astype(np.float32)
    W = (rng.standard_normal((K, N)) * 0.05).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    out = torch.empty((B, N), dtype=torch.float32, device=device)
    ops.dense_fp32(dev(x, device), dev(W, device), dev(b, device), act, out)
    np.testing.assert_allclose(out.cpu().numpy(), oracle.dense(x, W, b, act), rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("B,K,N", [(1, 13, 128), (65, 32, 1), (129, 1037, 70), (64, 64, 64)])
def test_dense_fp32_shapes_and_no_bias(device, B, K, N):
    rng = np.random.default_rng(11)
    x = rng.standard_normal((B, K)).astype(np.float32)
    W = (rng.standard_normal((K, N)) * 0.1).astype(np.float32)
    out = torch.empty((B, N), dtype=torch.float32, device=device)
    ops.dense_fp32(dev(x, device), dev(W, device), None, "relu", out)
    np.testing.assert_allclose(out.cpu().numpy(), oracle.dense(x, W, None, "relu"), rtol=RTOL, atol=ATOL)


def test_dense_fp32_cross_epilogue(device):
    rng = np.random.default_rng(12)
    B, d = 200, 100
    x0 = rng.standard_normal((B, d)).astype(np.float32)
    x = rng.standard_normal((B, d)).astype(np.float32)
    W = (rng.standard_normal((d, d)) * 0.05).astype(np.float32)
    b = rng.standard_normal(d).astype(np.float32)
    out = torch.empty((B, d), dtype=torch.float32, device=device)
    ops.dense_fp32(dev(x, device), dev(W, device), dev(b, device), None, out, x0=dev(x0, device))
    ref = x0 * (x @ W + b) + x
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=RTOL, atol=ATOL)


def test_rowwise_dot(device):
    rng = np.random.default_rng(13)
    q = rng.standard_normal((500, 64)).astype(np.float32)
    it = rng.standard_normal((500, 64)).astype(np.float32)
    out = torch.empty((500, 1), dtype=torch.float32, device=device)
    ops.rowwise_dot(dev(q, device), dev(it, device), out)
    np.testing.assert_allclose(out.cpu().numpy(), oracle.retrieval_scores(q, it), rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("tc", [True, False])
@pytest.mark.parametrize("id_dtype", [np.int32, np.int64])
@pytest.mark.parametrize("temperature", [1.0, 0.5])
def test_inbatch_scores_false_negative_diagonal(device, id_dtype, temperature, tc):
    """tests/unit/tf/outputs/test_contrastive.py:173-206: in-batch negatives' diagonal equals the
    false-negative score, off-diagonal does not."""
    rng = np.random.default_rng(14)
    B, D = 300, 64
    q = rng.standard_normal((B, D)).astype(np.float32)
    it = rng.standard_normal((B, D)).astype(np.float32)
    ids = rng.permutation(10 * B)[:B].astype(id_dtype)
    ids[5] = ids[17]  # a duplicated item id -> extra accidental hits (5,17) and (17,5)
    out = torch.empty((B, 1 + B), dtype=torch.float32, device=device)
    ops.inbatch_scores(dev(q, device), dev(it, device), dev(it, device), out, pos_ids=dev(ids, device),
                       neg_ids=dev(ids, device), downscore=True, false_neg_score=oracle.MIN_FLOAT,
                       temperature=temperature, tensor_cores=tc)
    ref, targets = oracle.contrastive_logits(q, it, it, ids, ids, True, oracle.MIN_FLOAT, temperature=temperature)
    got = out.cpu().numpy()
    # split-bf16 x3: |err| ~ 2^-16 * sum|q_k n_k| (absolute), scaled by 1/T
    np.testing.assert_allclose(got, ref, rtol=RTOL, atol=(3e-4 / temperature) if tc else ATOL)
    fns = np.float32(oracle.MIN_FLOAT) / np.float32(temperature)
    assert np.all(np.diag(got[:, 1:]) == fns)
    assert got[5, 1 + 17] == fns and got[17, 1 + 5] == fns
    off = got[:, 1:][~(ids[:, None] == ids[None, :])]
    assert np.all(off != fns)
    assert targets[:, 0].all() and not targets[:, 1:].any()


@pytest.mark.parametrize("tc", [True, False])
@pytest.mark.parametrize("B,N,D", [(100, 77, 32), (300, 1000, 64), (129, 256, 128)])
def test_inbatch_scores_logq_and_no_downscore(device, tc, B, N, D):
    rng = np.random.default_rng(15)
    q = rng.standard_normal((B, D)).astype(np.float32)
    pos = rng.standard_normal((B, D)).astype(np.float32)
    neg = rng.standard_normal((N, D)).astype(np.float32)
    pp = rng.random(B).astype(np.float32)
    npb = rng.random(N).astype(np.float32)
    out = torch.empty((B, 1 + N), dtype=torch.float32, device=device)
    ops.inbatch_scores(dev(q, device), dev(pos, device), dev(neg, device), out, downscore=False,
                       pos_prob=dev(pp, device), neg_prob=dev(npb, device), tensor_cores=tc)
    ref, _ = oracle.contrastive_logits(q, pos, neg, downscore=False, pos_prob=pp, neg_prob=npb)
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=RTOL, atol=5e-4 if tc else ATOL)


def test_ops_reject_cpu_tensors():
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.l2_normalize(torch.zeros(2, 4))


# ---- tensor-core interaction path (mma.sync split-bf16, cp.async.bulk row staging) ---------------
def _unsplit(t, width):
    Kp = t.shape[1] // 2
    f = t.float().cpu().numpy()
    return f[:, :width] + f[:, Kp:Kp + width], f


@pytest.mark.parametrize("B", [1, 31, 1000, 5000])
def test_dot_interaction_split_output(device, B):
    rng = np.random.default_rng(20)
    F, D = 27, 64
    x = rng.standard_normal((B, F, D)).astype(np.float32)
    bottom = x[:, 26].copy()
    W = D + F * (F - 1) // 2
    Kp = ops.tc_padded_k(W)
    out = torch.full((B, 2 * Kp), 3.0, dtype=torch.bfloat16, device=device)
    ops.dot_interaction(dev(x, device), out, prefix=dev(bottom, device))
    rec, raw = _unsplit(out, W)
    ref = np.concatenate([bottom, oracle.dot_interaction(x)], axis=1)
    np.testing.assert_allclose(rec, ref, rtol=2e-4, atol=2e-4)  # hi+lo carries ~16 bits
    assert np.all(raw[:, W:Kp] == 0) and np.all(raw[:, Kp + W:] == 0)  # zero padding for the next GEMM
    # identical to splitting the fp32 result of the same kernel
    o32 = torch.empty((B, W), dtype=torch.float32, device=device)
    ops.dot_interaction(dev(x, device), o32, prefix=dev(bottom, device))
    assert torch.equal(ops.split_rows(o32), out)


@pytest.mark.parametrize("F,D", [(2, 16), (32, 32), (17, 48), (9, 256)])
def test_dot_interaction_tensor_core_shapes(device, F, D):
    rng = np.random.default_rng(22)
    B = 257
    x = rng.standard_normal((B, F, D)).astype(np.float32)
    out = torch.empty((B, F * (F - 1) // 2), dtype=torch.float32, device=device)
    ops.dot_interaction(dev(x, device), out)
    np.testing.assert_allclose(out.cpu().numpy(), oracle.dot_interaction(x), rtol=1e-4, atol=2e-4 * np.sqrt(D / 64))
