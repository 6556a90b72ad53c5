"""BASELINE.json's FULL sizes on the H100, checked through size-independent properties and sampled
oracle comparisons (the oracle cannot run 65 536 x 45.6 M-row lookups in seconds, but the tables are
hash-initialised, so any row can be regenerated on the host bit-exactly).

  config 2: mm.DLRMModel, bundled Criteo cardinalities (45 621 194 rows, 11.7 GB), batch 65 536
  config 3: two-tower in-batch scorer, batch 16 384 (268 M logits)
"""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets, ops
from oracle import oracle
from tests import helpers as H

pytestmark = pytest.mark.gpu

SEED = 4321


def _table_seed(name):
    from models_b200.inputs import _stable_hash

    return (SEED * 1000003 + _stable_hash(name)) & (2**63 - 1)


@pytest.fixture(scope="module")
def criteo_full():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    free, _ = torch.cuda.mem_get_info()
    if free < 40 * 2**30:
        pytest.skip("needs 40 GB of free HBM")
    mm.set_seed(77)
    schema = datasets.criteo_schema()
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([128, 64]), top_block=mm.MLPBlock([128, 64, 32]),
                         embedding_options=mm.EmbeddingOptions(embeddings_initializers={"hash_seed": SEED}))
    dev = torch.device("cuda", 0)
    model.build(dev)
    B = 65536
    batch, _ = datasets.split_targets(schema, datasets.generate_batch(schema, B, seed=2024, index_law="uniform"))
    yield schema, model, batch, {k: torch.from_numpy(v).to(dev) for k, v in batch.items()}
    del model
    torch.cuda.empty_cache()


def test_full_criteo_tables_are_the_hash_tables(criteo_full):
    schema, model, batch, dbatch = criteo_full
    rng = np.random.default_rng(0)
    total = 0
    for name, t in model.body.embeddings.tables.items():
        total += t.input_dim
        rows = np.unique(np.concatenate([[0, t.input_dim - 1], rng.integers(0, t.input_dim, 64)]))
        got = t.embeddings[torch.from_numpy(rows).cuda()].cpu().numpy()
        assert np.array_equal(got, oracle.hash_table_rows(rows, 64, _table_seed(name)))
    assert total == 45_621_194


def test_full_gather_bit_exact_everywhere(criteo_full):
    """Every one of the 65 536 x 26 gathered rows equals table[idx] (torch indexing on the device is
    the independent checker at this size) and sampled rows equal the host-regenerated hash rows."""
    schema, model, batch, dbatch = criteo_full
    emb = model.body.embeddings
    names = emb.feature_names
    slots = {n: i for i, n in enumerate(sorted(names))}
    B, D = 65536, 64
    out = torch.empty((B, len(names) * D), dtype=torch.float32, device="cuda")
    oob = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.gather_multi([emb.feature_to_table[n].table for n in names], [dbatch[n] for n in names], [slots[n] * D for n in names],
                     out, oob)
    assert int(oob.item()) == 0
    for n in names:
        assert torch.equal(out[:, slots[n] * D:(slots[n] + 1) * D], emb.feature_to_table[n].table[dbatch[n].long()])
    rows = np.random.default_rng(1).integers(0, B, 32)
    got = out[torch.from_numpy(rows).cuda()].cpu().numpy()
    for n in names:
        want = oracle.hash_table_rows(batch[n][rows], D, _table_seed(emb.feature_to_table[n].table_name))
        assert np.array_equal(got[:, slots[n] * D:(slots[n] + 1) * D], want)


def test_full_dlrm_forward_sampled_against_oracle(criteo_full):
    """Full batch through the fused path; 256 sampled samples are recomputed by the NumPy oracle from
    host-regenerated table rows and the model's MLP weights; fused == staged == graph replay."""
    schema, model, batch, dbatch = criteo_full
    out = model(dbatch)
    assert tuple(out.shape) == (65536, 1)
    assert torch.equal(out, model(dbatch))  # deterministic / idempotent
    model.body.fused = False
    staged = model(dbatch)
    model.body.fused = True
    assert torch.allclose(out, staged, rtol=0, atol=2e-6)
    cf = model.compile(batch)
    assert torch.equal(cf(mm.HostBatch.like(batch, model.input_columns())).cuda(), out)
    rows = np.sort(np.random.default_rng(2).choice(65536, 256, replace=False))
    sub = {k: v[rows] for k, v in batch.items()}
    # compact per-table mini tables holding exactly the rows the sampled samples touch
    tables, f2t, sub_idx = {}, {}, dict(sub)
    for f, t in model.body.embeddings.feature_to_table.items():
        uniq, inv = np.unique(sub[f], return_inverse=True)
        tables[f] = oracle.hash_table_rows(uniq, 64, _table_seed(t.table_name))
        f2t[f] = f
        sub_idx[f] = inv.astype(np.int64)
    ref = oracle.dlrm_forward(sub_idx, tables, f2t, model.body.continuous.features, H.mlp_layers(model.body.bottom_block),
                              H.mlp_layers(model.body.top_block), H.head_layer(model.prediction))
    got = out.cpu().numpy()[rows]
    assert H.rel_err(got, ref) < 2e-4
    assert np.all(np.isfinite(out.cpu().numpy()))


def test_full_inbatch_scorer_16384(device):
    """268 M logits: diagonal and duplicate-id hits == false-negative score, column 0 == row-wise dot,
    1 000 sampled entries == fp32 dot products, determinism, targets view."""
    rng = np.random.default_rng(3)
    B, D = 16384, 64
    q = rng.standard_normal((B, D)).astype(np.float32)
    it = rng.standard_normal((B, D)).astype(np.float32)
    ids = np.minimum(rng.zipf(1.05, B) - 1, 9_999_999).astype(np.int64)  # Zipf: many duplicated items
    dq, dit, dids = (torch.from_numpy(a).to(device) for a in (q, it, ids))
    out = mm.ContrastiveOutput(negative_samplers="in-batch")({"query": dq, "candidate": dit}, candidate_ids=dids, training=True)
    logits = out.outputs
    assert tuple(logits.shape) == (B, B + 1) and tuple(out.targets.shape) == (B, B + 1)
    fns = np.float32(oracle.MIN_FLOAT)
    assert torch.all(torch.diagonal(logits[:, 1:]) == float(fns))
    hit = dids[:, None] == dids[None, :]
    assert torch.all(logits[:, 1:][hit] == float(fns))
    n_hits = int(hit.sum().item())
    assert n_hits > B  # the Zipf ids really produce accidental hits beyond the diagonal
    assert int((logits[:, 1:] == float(fns)).sum().item()) == n_hits  # nothing else is masked
    np.testing.assert_allclose(logits[:, 0].cpu().numpy(), (q * it).sum(-1), rtol=1e-4, atol=1e-4)
    r = rng.integers(0, B, 1000)
    c = rng.integers(0, B, 1000)
    keep = ids[r] != ids[c]
    got = logits[torch.from_numpy(r).to(device), torch.from_numpy(c + 1).to(device)].cpu().numpy()
    want = (q[r].astype(np.float64) * it[c].astype(np.float64)).sum(-1)
    np.testing.assert_allclose(got[keep], want[keep], rtol=1e-4, atol=5e-4)
    again = mm.ContrastiveOutput(negative_samplers="in-batch")({"query": dq, "candidate": dit}, candidate_ids=dids, training=True)
    assert torch.equal(again.outputs, logits)
    assert float(out.targets[:, 0].min()) == 1.0 and float(out.targets[:, 1:].max()) == 0.0
