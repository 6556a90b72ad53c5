"""Top-k retrieval / evaluation on the H100 (SURVEY §8f-2) against the oracle restatement of
TopKIndexBlock (core/index.py:232-284), BruteForce (outputs/topk.py:180-243), RetrievalModel.evaluate
(models/base.py:2266-2351) and metrics/topk.py.  Scores: 3-pass split-bf16 (atol 2e-4 at |q.v| ~ 10);
identifiers: exact whenever the gap between neighbouring scores exceeds the score tolerance."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets, topk
from oracle import oracle

pytestmark = pytest.mark.gpu


def dev(a, device):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def _check_topk(scores, ids, ref_s, ref_ids, atol=3e-4):
    np.testing.assert_allclose(scores, ref_s, rtol=1e-4, atol=atol)
    if ref_s.shape[1] == 1:  # no neighbour to measure the gap against: near-ties may flip the single winner
        assert (ids == ref_ids).mean() > 0.99
        return
    gap = np.abs(np.diff(ref_s, axis=1)).min(axis=1) > 4 * atol  # rows whose ordering cannot flip within tolerance
    assert gap.any()
    assert np.array_equal(ids[gap], ref_ids[gap])


@pytest.mark.parametrize("N,D,k", [(5000, 64, 20), (1000, 32, 1), (70000, 64, 32), (333, 48, 10)])
def test_topk_index_block_matches_oracle(device, N, D, k):
    rng = np.random.default_rng(20)
    B = 257
    q = rng.standard_normal((B, D)).astype(np.float32)
    v = rng.standard_normal((N, D)).astype(np.float32)
    ids = rng.permutation(10 * N)[:N].astype(np.int64)  # identifiers are not row numbers
    index = mm.TopKIndexBlock(k, dev(v, device), dev(ids, device))
    s, i = index(dev(q, device))
    assert tuple(s.shape) == (B, k) and i.dtype == torch.int64
    ref_s, ref_i = oracle.topk_index(q, v, ids, k)
    _check_topk(s.cpu().numpy(), i.cpu().numpy(), ref_s, ref_i)
    assert np.all(np.diff(s.cpu().numpy(), axis=1) <= 0)  # sorted, best first
    s5, i5 = index(dev(q, device), k=min(5, k))  # call-time k overrides the constructor's
    assert torch.equal(s5, s[:, :min(5, k)]) and torch.equal(i5, i[:, :min(5, k)])
    # default identifiers = row numbers
    plain = mm.TopKIndexBlock(k, dev(v, device))
    _, rows = plain(dev(q, device))
    assert torch.equal(dev(ids, device)[rows], i)
    # evaluation outputs: one-hot of the positive among the top-k
    pos = ref_i[np.arange(B), rng.integers(0, k, B)]
    pos[::7] = -5  # some positives are not retrieved at all
    out = index.call_outputs(dev(pos, device), dev(q, device))
    np.testing.assert_array_equal(out.targets.cpu().numpy() > 0, oracle.topk_targets(pos, i.cpu().numpy()) > 0)
    assert float(out.extra["label_relevant_counts"].sum()) == B


def test_topk_beyond_the_fused_limit_uses_materialised_scores(device):
    rng = np.random.default_rng(21)
    q = rng.standard_normal((64, 64)).astype(np.float32)
    v = rng.standard_normal((3000, 64)).astype(np.float32)
    index = mm.TopKIndexBlock(50, dev(v, device))
    s, i = index(dev(q, device))
    ref_s, ref_i = oracle.topk_index(q, v, None, 50)
    _check_topk(s.cpu().numpy(), i.cpu().numpy(), ref_s, ref_i)
    with pytest.raises(ValueError, match="exceeds the number of candidates"):
        index(dev(q, device), k=3001)


def test_brute_force_layer_protocol(device):
    rng = np.random.default_rng(22)
    q = rng.standard_normal((100, 64)).astype(np.float32)
    v = rng.standard_normal((2000, 64)).astype(np.float32)
    ids = np.arange(2000, dtype=np.int64) * 3
    bf = mm.BruteForce(k=10)
    with pytest.raises(ValueError, match="call the `index` method first"):
        bf(dev(q, device))
    bf.index(dev(v, device), dev(ids, device))
    pred = bf(dev(q, device))
    assert isinstance(pred, mm.TopKPrediction)
    ref_s, ref_i = oracle.topk_index(q, v, ids, 10)
    _check_topk(pred.scores.cpu().numpy(), pred.identifiers.cpu().numpy(), ref_s, ref_i)
    targets = ref_i[:, 2].copy()
    ev = bf(dev(q, device), targets=dev(targets, device), testing=True)
    assert np.array_equal(ev.targets.cpu().numpy(), oracle.topk_targets(targets, pred.identifiers.cpu().numpy()))
    with pytest.raises(ValueError, match="Targets should be provided"):
        bf(dev(q, device), testing=True)
    with pytest.raises(ValueError, match="same embedding size"):
        bf(dev(q[:, :32], device))
    with pytest.raises(ValueError, match="same number of rows"):
        mm.BruteForce().index(dev(v, device), dev(ids[:10], device))
    with pytest.raises(ValueError, match="2-D"):
        mm.BruteForce().index(dev(v[0], device))
    import pandas as pd

    bf2 = mm.BruteForce(k=10).index_from_dataset(pd.DataFrame(v, index=ids))
    assert torch.equal(bf2(dev(q, device)).identifiers, pred.identifiers)
    with pytest.raises(ValueError, match="unique indices"):
        mm.BruteForce().index_from_dataset(pd.DataFrame(v[:4], index=[1, 1, 2, 3]))


@pytest.fixture(scope="module")
def ml1m():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    device = torch.device("cuda", 0)
    mm.set_seed(23)
    schema = datasets.movielens_1m_schema()
    model = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([128, 64]))
    batch, _ = datasets.split_targets(schema, datasets.generate_batch(schema, 2048, seed=7))
    model.build(device)
    return schema, model, batch


def _numpy_eval(q, item_emb, item_ids, positives, k):
    s, top = oracle.topk_index(q, item_emb, item_ids, k)
    y = oracle.topk_targets(positives, top)
    rel = np.ones(len(y), np.float32)
    return {"recall_at_%d" % k: float(oracle.recall_at(y, rel, k).mean()), "ndcg_at_%d" % k: float(oracle.ndcg_at(y, rel, k).mean()),
            "mrr_at_%d" % k: float(oracle.mrr_at(y, rel, k).mean())}


def test_retrieval_model_evaluate_against_item_corpus(device, ml1m):
    """evaluate(item_corpus=item features): corpus deduplicated by item id, encoded by the item tower in batches,
    every query ranked against it by the fused kernel; metrics == NumPy top-k + metrics on the same embeddings."""
    schema, model, batch = ml1m
    k = 10
    metrics = [mm.RecallAt(k), mm.NDCGAt(k), mm.MRRAt(k)]
    got = model.evaluate(batch, item_corpus=batch, metrics=metrics, batch_size=500)
    corpus = topk.unique_rows_by_features(batch, "movieId")
    ids, item_emb = model.item_embeddings(corpus, batch_size=300)
    assert len(np.unique(ids)) == len(ids) == len(np.unique(batch["movieId"]))
    _, q = model.query_embeddings(batch, batch_size=700)
    want = _numpy_eval(q.cpu().numpy(), item_emb.cpu().numpy(), ids, batch["movieId"].reshape(-1), k)
    for name, v in want.items():
        assert abs(got[name] - v) < 2e-3, (name, got[name], v)
    assert 0.0 < got["recall_at_10"] <= 1.0
    # the same through a prebuilt index, several batches
    index = mm.TopKIndexBlock(k, item_emb, torch.from_numpy(ids).to(device))
    halves = [topk.slice_rows(batch, 0, 1000), topk.slice_rows(batch, 1000, 2048)]
    again = model.evaluate(halves, item_corpus=index, metrics=metrics)
    for name in want:
        assert abs(again[name] - got[name]) < 1e-6
    with pytest.raises(ValueError, match="the metrics need"):
        model.evaluate(batch, item_corpus=mm.TopKIndexBlock(5, item_emb), metrics=[mm.RecallAt(10)])
    with pytest.raises(ValueError, match="must be either"):
        model.evaluate(batch, item_corpus=[1, 2, 3])


def test_in_batch_evaluate_and_top_k_encoder(device, ml1m):
    schema, model, batch = ml1m
    sub = topk.slice_rows(batch, 0, 256)
    got = model.evaluate(sub, metrics=[mm.RecallAt(5), mm.NDCGAt(5)])
    out = model({k: torch.from_numpy(v).to(device) for k, v in sub.items()}, testing=True)
    logits, targets = out.outputs.cpu().numpy(), out.targets.cpu().numpy()
    s, order = oracle.topk(logits, 5)
    y = np.take_along_axis(targets, order, axis=1)
    rel = targets.sum(-1)
    assert abs(got["recall_at_5"] - float(oracle.recall_at(y, rel, 5).mean())) < 1e-6
    assert abs(got["ndcg_at_5"] - float(oracle.ndcg_at(y, rel, 5).mean())) < 1e-6

    corpus = topk.unique_rows_by_features(batch, "movieId")
    enc = model.to_top_k_encoder(corpus, k=7, batch_size=400)
    scores, ids = enc.batch_predict([topk.slice_rows(batch, 0, 300), topk.slice_rows(batch, 300, 512)])
    assert scores.shape == (512, 7) and ids.shape == (512, 7)
    cids, item_emb = model.item_embeddings(corpus)
    _, q = model.query_embeddings(topk.slice_rows(batch, 0, 512))
    ref_s, ref_i = oracle.topk_index(q.cpu().numpy(), item_emb.cpu().numpy(), cids, 7)
    _check_topk(scores, ids, ref_s, ref_i, atol=2e-6)  # tower outputs are O(0.1): absolute error ~1e-7
    ev = enc.evaluate([topk.slice_rows(batch, 0, 512)], metrics=[mm.RecallAt(7)])
    y = oracle.topk_targets(batch["movieId"][:512].reshape(-1), ids)
    assert abs(ev["recall_at_7"] - float(oracle.recall_at(y, np.ones(512, np.float32), 7).mean())) < 2e-3
    # precomputed candidates: (ids, embeddings) pair
    enc2 = model.to_top_k_encoder((cids, item_emb), k=7)
    s2, i2 = enc2.batch_predict([topk.slice_rows(batch, 0, 512)])
    assert np.array_equal(i2, ids)
