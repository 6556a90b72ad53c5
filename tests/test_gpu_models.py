"""Model-level GPU parity: mm.DLRMModel / mm.DCNModel / mm.TwoTowerModel forward against the CPU
oracle on identical synthetic inputs and identical weights (BASELINE.json configs at
oracle-friendly sizes; the full-size properties live in test_gpu_fullsize.py).

Tolerance: north-star 1e-3 relative on fp32 logits; asserted here at 2e-4 of the logit scale.
"""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets
from oracle import oracle
from tests import helpers as H

pytestmark = pytest.mark.gpu


def small_criteo(cap=5000):
    return datasets.criteo_schema({k: min(v, cap) for k, v in datasets.CRITEO_MAX.items()})


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("index_dtype", [np.int32, np.int64])
def test_dlrm_model_matches_oracle(device, fused, index_dtype):
    mm.set_seed(7)
    schema = small_criteo()
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([128, 64]),
                         top_block=mm.MLPBlock([128, 64, 32]))
    model.body.fused = fused
    batch = datasets.generate_batch(schema, 1000, seed=1234, index_law="uniform", index_dtype=index_dtype)
    feats, _ = datasets.split_targets(schema, batch)
    out = model(H.device_batch(feats, device))
    assert out.shape == (1000, 1) and out.dtype == torch.float32
    ref, inter = H.oracle_dlrm(model, feats, return_intermediates=True)
    got = out.cpu().numpy()
    assert H.rel_err(got, ref) < 2e-4
    assert np.all((got > 0) & (got < 1))  # sigmoid output
    # block-level: [bottom | interactions] layout and the stack order (bottom_block last)
    bottom = model.body.bottom_forward(H.device_batch(feats, device))
    body_in = model.body.interaction_forward(H.device_batch(feats, device), bottom).cpu().numpy()
    assert body_in.shape == (1000, 64 + 27 * 26 // 2)
    np.testing.assert_allclose(body_in[:, :64], inter["bottom"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(body_in[:, 64:], inter["interactions"], rtol=1e-4, atol=1e-5)


def test_dlrm_block_output_widths(device):
    """tests/unit/tf/blocks/test_dlrm.py:26-52: without top block the output is the interactions
    only: F(F-1)/2 with F = #categorical + 1 (bottom) ; without continuous features F = #categorical."""
    mm.set_seed(1)
    schema = small_criteo(100)
    dlrm = mm.DLRMBlock(schema, embedding_dim=16, bottom_block=mm.MLPBlock([32, 16]))
    batch = datasets.generate_batch(schema, 50, seed=1, index_law="uniform")
    feats, _ = datasets.split_targets(schema, batch)
    out = dlrm(H.device_batch(feats, device))
    assert tuple(out.shape) == (50, 27 * 26 // 2)
    cat_only = schema.select_by_tag(mm.Tags.CATEGORICAL)
    dlrm2 = mm.DLRMBlock(cat_only, embedding_dim=16, top_block=mm.MLPBlock([8]))
    out2 = dlrm2(H.device_batch({k: v for k, v in feats.items() if k.startswith("C")}, device))
    assert tuple(out2.shape) == (50, 8)


def test_dlrm_shared_table_features_identical(device):
    """tests/unit/tf/inputs/test_embedding.py:231-253: two columns with the same int_domain name
    share one table; equal ids give equal rows."""
    mm.set_seed(2)
    a = datasets._cat("item_a", 99, domain_name="item")
    b = datasets._cat("item_b", 99, domain_name="item")
    emb = mm.Embeddings(mm.Schema([a, b]), dim=32)
    assert list(emb.tables) == ["item"]
    ids = torch.arange(50, dtype=torch.int32, device=device)
    out = emb({"item_a": ids, "item_b": ids})
    assert torch.equal(out["item_a"], out["item_b"])
    assert torch.equal(out["item_a"], emb.tables["item"].embeddings[:50])


def test_dlrm_out_of_range_index_raises(device):
    mm.set_seed(3)
    schema = small_criteo(50)
    model = mm.DLRMModel(schema, embedding_dim=16, bottom_block=mm.MLPBlock([16]), top_block=mm.MLPBlock([8]))
    batch = datasets.generate_batch(schema, 20, seed=3, index_law="uniform")
    feats, _ = datasets.split_targets(schema, batch)
    feats["C3"] = feats["C3"].copy()
    feats["C3"][4] = 10_000
    with pytest.raises(IndexError, match="out of range"):
        model(H.device_batch(feats, device))


@pytest.mark.parametrize("n_cat,D", [(26, 8), (33, 16)])
def test_dlrm_model_outside_the_fused_kernel(device, n_cat, D):
    """Shapes the fused lookup + interaction kernel does not take (D = 8; F = 34 > 32 feature slots): fused=True
    gives the same predictions as fused=False, bit for bit, matches the oracle, and still reports bad ids."""
    mm.set_seed(41)
    schema = mm.Schema(list(small_criteo(3000)) + [datasets._cat(f"C{i}", 3000) for i in range(27, n_cat + 1)])
    model = mm.DLRMModel(schema, embedding_dim=D, bottom_block=mm.MLPBlock([32, D]), top_block=mm.MLPBlock([64, 16]))
    assert not model.body.can_emit_split()
    feats, _ = datasets.split_targets(schema, datasets.generate_batch(schema, 500, seed=8, index_law="uniform"))
    batch = H.device_batch(feats, device)
    fused = model(batch).cpu().numpy()
    model.body.fused = False
    staged = model(batch).cpu().numpy()
    model.body.fused = True
    assert np.array_equal(fused, staged)
    assert H.rel_err(fused, H.oracle_dlrm(model, feats)) < 2e-4
    bad = dict(feats)
    bad["C3"] = feats["C3"].copy()
    bad["C3"][4] = 10_000
    with pytest.raises(IndexError, match="out of range"):
        model(H.device_batch(bad, device))


@pytest.mark.parametrize("stacked", [True, False])
def test_dcn_model_matches_oracle(device, stacked):
    mm.set_seed(11)
    schema = small_criteo(2000)
    model = mm.DCNModel(schema, depth=3, deep_block=mm.MLPBlock([256, 128]), stacked=stacked)
    batch = datasets.generate_batch(schema, 300, seed=5, index_law="uniform")
    feats, _ = datasets.split_targets(schema, batch)
    out = model(H.device_batch(feats, device))
    assert out.shape == (300, 1)
    ref = H.oracle_dcn(model, feats)
    assert H.rel_err(out.cpu().numpy(), ref) < 2e-4


def test_dcn_default_input_width_is_1037_on_bundled_criteo():
    """Inferred dims on the bundled Criteo cardinalities sum to 1024 (+13 continuous) — SURVEY §8(a) a10."""
    model = mm.DCNModel(datasets.criteo_schema(), depth=3, deep_block=mm.MLPBlock([256, 128]))
    assert model.body.input_block.layout()[2] == 1037


@pytest.mark.parametrize("temperature", [1.0, 2.0])
def test_two_tower_movielens_config1(device, temperature):
    """BASELINE config 1: mm.TwoTowerModel on the MovieLens-1M schema, batch 256: inference (256,1)
    and training (256,257) logits vs the oracle."""
    mm.set_seed(21)
    schema = datasets.movielens_1m_schema()
    model = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([128, 64]), logits_temperature=temperature)
    batch = datasets.generate_batch(schema, 256, seed=1234)
    feats, _ = datasets.split_targets(schema, batch)
    dfeats = H.device_batch(feats, device)
    inf = model(dfeats)
    assert tuple(inf.shape) == (256, 1)
    q = H.oracle_tower(model.body.query, feats)
    it = H.oracle_tower(model.body.item, feats)
    assert q.shape == (256, 64) and it.shape == (256, 64)
    np.testing.assert_allclose(inf.cpu().numpy(), oracle.retrieval_scores(q, it), rtol=2e-4, atol=2e-5)

    pred = model(dfeats, training=True)
    assert tuple(pred.outputs.shape) == (256, 257) and tuple(pred.targets.shape) == (256, 257)
    ids = feats["movieId"]
    ref, tref = oracle.contrastive_logits(q, it, it, ids, ids, True, oracle.MIN_FLOAT, temperature=temperature)
    got = pred.outputs.cpu().numpy()
    fns = np.float32(oracle.MIN_FLOAT) / np.float32(temperature)
    mask = ids[:, None] == ids[None, :]
    assert np.all(got[:, 1:][mask] == fns)  # accidental hits incl. the diagonal
    np.testing.assert_allclose(got[:, 1:][~mask], ref[:, 1:][~mask], rtol=2e-4, atol=2e-5)
    np.testing.assert_allclose(got[:, 0], ref[:, 0], rtol=2e-4, atol=2e-5)
    assert np.array_equal(pred.targets.cpu().numpy(), tref)
    # tower input layouts follow the sorted-name concat (SURVEY §8(a) a11)
    assert model.body.query.inputs.layout()[2] == 69 and model.body.item.inputs.layout()[2] == 129


def test_two_tower_l2_norm_post(device):
    """tests/unit/tf/blocks/retrieval/test_two_tower.py:94-107."""
    mm.set_seed(22)
    schema = datasets.movielens_1m_schema()
    block = mm.TwoTowerBlock(schema, query_tower=mm.MLPBlock([64, 32]), post="l2-norm")
    batch = datasets.generate_batch(schema, 100, seed=2)
    feats, _ = datasets.split_targets(schema, batch)
    out = block(H.device_batch(feats, device))
    for k in ("query", "item"):
        np.testing.assert_allclose(np.linalg.norm(out[k].cpu().numpy(), axis=1), 1.0, rtol=1e-5)


def test_contrastive_output_v2(device):
    rng = np.random.default_rng(3)
    B, D = 64, 32
    q = rng.standard_normal((B, D)).astype(np.float32)
    c = rng.standard_normal((B, D)).astype(np.float32)
    ids = rng.integers(0, 40, B).astype(np.int64)
    out = mm.ContrastiveOutput(negative_samplers="in-batch")
    dq, dc, dids = (torch.from_numpy(a).to(device) for a in (q, c, ids))
    inf = out({"query": dq, "candidate": dc})
    assert tuple(inf.shape) == (B, 1)
    pred = out({"query": dq, "candidate": dc}, candidate_ids=dids, training=True)
    ref, _ = oracle.contrastive_logits(q, c, c, ids, ids, True, oracle.MIN_FLOAT)
    np.testing.assert_allclose(pred.outputs.cpu().numpy(), ref, rtol=2e-4, atol=5e-4)
    # logQ correction with the log-uniform sampling probabilities (popularity.py:141-165)
    probs = mm.log_uniform_sampling_probs(max_id=39, min_id=0, max_num_samples=B, unique=True)
    assert np.allclose(probs, oracle.log_uniform_probs(39, 0, True, B))
    out_q = mm.ContrastiveOutput(negative_samplers="in-batch", logq_sampling_correction=True)
    pred_q = out_q({"query": dq, "candidate": dc}, candidate_ids=dids, training=True,
                   sampling_probs=torch.from_numpy(probs).to(device))
    ref_q, _ = oracle.contrastive_logits(q, c, c, ids, ids, True, oracle.MIN_FLOAT, pos_prob=probs[ids], neg_prob=probs[ids])
    np.testing.assert_allclose(pred_q.outputs.cpu().numpy(), ref_q, rtol=2e-4, atol=5e-4)


def test_forward_host_roundtrip(device):
    mm.set_seed(5)
    schema = small_criteo(300)
    model = mm.DLRMModel(schema, embedding_dim=16, bottom_block=mm.MLPBlock([32, 16]), top_block=mm.MLPBlock([16, 8]))
    batch = datasets.generate_batch(schema, 128, seed=9, index_law="uniform")
    feats, _ = datasets.split_targets(schema, batch)
    a = model.forward_host(feats).numpy()
    b = model(H.device_batch(feats, device)).cpu().numpy()
    assert np.array_equal(a, b)


def test_compiled_forward_matches_eager_and_checks_indices(device):
    """Model.compile: CUDA-graph replay over static buffers, packed pinned host batch in, pinned
    host predictions out; out-of-range ids are still reported (deferred check after the replay)."""
    mm.set_seed(31)
    schema = small_criteo(500)
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([32, 64]), top_block=mm.MLPBlock([64, 16]))
    b0, _ = datasets.split_targets(schema, datasets.generate_batch(schema, 700, seed=1, index_law="uniform"))
    b1, _ = datasets.split_targets(schema, datasets.generate_batch(schema, 700, seed=2, index_law="uniform"))
    cf = model.compile(b0)
    assert cf.launches_per_replay >= 3  # concat+split, bottom tower, gather+interaction, top tower (+head)
    for b in (b0, b1, b0):
        hb = mm.HostBatch.like(b, model.input_columns())
        got = cf(hb).clone().numpy()
        want = model(H.device_batch(b, device)).cpu().numpy()
        assert np.array_equal(got, want)
    bad = {k: v.copy() for k, v in b1.items()}
    bad["C5"][3] = 10 ** 6
    with pytest.raises(IndexError, match="out of range"):
        cf(mm.HostBatch.like(bad, model.input_columns()))
    # the counter was reset: a good batch works again
    assert np.array_equal(cf(mm.HostBatch.like(b0, model.input_columns())).numpy(), model(H.device_batch(b0, device)).cpu().numpy())
    with pytest.raises(ValueError, match="layout"):
        cf(mm.HostBatch.like({k: v[:10] for k, v in b0.items()}, model.input_columns()))


def test_compiled_two_tower_training_logits(device):
    mm.set_seed(32)
    schema = datasets.movielens_1m_schema()
    model = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([64, 32]))
    b, _ = datasets.split_targets(schema, datasets.generate_batch(schema, 256, seed=5))
    cf = model.compile(b, training=True)
    got = cf(mm.HostBatch.like(b, model.input_columns())).clone().numpy()
    want = model(H.device_batch(b, device), training=True).outputs.cpu().numpy()
    assert got.shape == (256, 257) and np.array_equal(got, want)


def test_pipelined_forward_overlapping_batches(device):
    mm.set_seed(33)
    schema = small_criteo(400)
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([32, 64]), top_block=mm.MLPBlock([64, 16]))
    batches = [datasets.split_targets(schema, datasets.generate_batch(schema, 600, seed=s, index_law="uniform"))[0]
               for s in range(5)]
    hbs = [mm.HostBatch.like(b, model.input_columns()) for b in batches]
    pf = model.pipeline(batches[0], depth=2)
    want = [model(H.device_batch(b, device)).cpu().numpy() for b in batches]
    got, tickets = [], []
    for hb in hbs:
        tickets.append(pf.submit(hb))
        if len(tickets) == 2:
            got.append(pf.result(tickets.pop(0)).clone().numpy())
    while tickets:
        got.append(pf.result(tickets.pop(0)).clone().numpy())
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    t = pf.submit(hbs[0])
    pf.submit(hbs[1])
    with pytest.raises(RuntimeError, match="uncollected"):
        pf.submit(hbs[2])
    pf.result(t)
