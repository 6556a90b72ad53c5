"""MatrixFactorizationModel without a GPU: the constructor against the reference's (models/retrieval.py:27-103,
blocks/retrieval/matrix_factorization.py:31-112), tag selection, checkpoint names, and the float64 restatement of its
training step (tests/mf_train_oracle.py) against the reference's torch step and the closed-form L2 gradient."""
import inspect
from pathlib import Path

import numpy as np
import pytest

import models_b200 as mm
from models_b200 import datasets
from models_b200.schema import Schema, Tags
from tests import mf_train_oracle as O

GOLDEN = Path(__file__).parent / "golden" / "mf_train" / "ref_torch_mf_train.npz"


def test_signature_and_defaults_follow_the_reference():
    sig = inspect.signature(mm.MatrixFactorizationModel)
    want = [("schema", inspect.Parameter.empty), ("dim", inspect.Parameter.empty), ("query_id_tag", Tags.USER_ID),
            ("item_id_tag", Tags.ITEM_ID), ("embeddings_initializers", None), ("embeddings_l2_reg", 0.0), ("post", None),
            ("prediction_tasks", None), ("logits_temperature", 1.0), ("samplers", ())]
    params = [p for p in sig.parameters.values() if p.kind != inspect.Parameter.VAR_KEYWORD]
    assert [(p.name, p.default) for p in params] == want
    assert any(p.kind == inspect.Parameter.VAR_KEYWORD for p in sig.parameters.values())
    blk = inspect.signature(mm.QueryItemIdsEmbeddingsBlock)
    assert list(blk.parameters)[:6] == ["schema", "dim", "query_id_tag", "item_id_tag", "embeddings_initializers",
                                        "embeddings_l2_reg"]


def test_positional_dim_builds_id_towers_without_mlp():
    schema = datasets.movielens_1m_schema()
    model = mm.MatrixFactorizationModel(schema, 32, embeddings_l2_reg=1e-4, post="l2-norm", logits_temperature=0.5)
    assert isinstance(model, mm.RetrievalModel) and isinstance(model.body, mm.TwoTowerBlock)
    assert isinstance(model.body, mm.QueryItemIdsEmbeddingsBlock)
    q, it = model.body.query, model.body.item
    assert q.mlp is None and it.mlp is None
    assert q.inputs.embeddings.feature_names == ["userId"] and it.inputs.embeddings.feature_names == ["movieId"]
    assert q.inputs.continuous is None and it.inputs.continuous is None
    assert all(t.dim == 32 for tw in (q, it) for t in tw.inputs.embeddings.tables.values())
    assert q.inputs.embedding_options.embeddings_l2_reg == 1e-4 and it.inputs.embedding_options.embeddings_l2_reg == 1e-4
    assert isinstance(model.body.post, mm.L2Norm)
    assert model.prediction.logits_temperature == 0.5
    assert isinstance(model.prediction.scorer.samplers[0], mm.InBatchSampler)
    assert set(model.input_columns()) == {"userId", "movieId"}


def test_tag_selection_and_its_errors():
    schema = datasets.movielens_1m_schema()
    m = mm.MatrixFactorizationModel(schema, 16, query_id_tag=Tags.USER, item_id_tag=Tags.ITEM)
    assert "userId" in m.body.query.inputs.embeddings.feature_names and "genres" in m.body.item.inputs.embeddings.feature_names
    no_user = Schema([c for c in schema if Tags.USER_ID not in c.tags])
    with pytest.raises(ValueError, match="USER_ID"):
        mm.QueryItemIdsEmbeddingsBlock(no_user, 16)
    no_item = Schema([c for c in schema if Tags.ITEM_ID not in c.tags and c.name != "movieId"])
    with pytest.raises(ValueError, match="ITEM_ID"):
        mm.QueryItemIdsEmbeddingsBlock(no_item, 16)
    with pytest.raises(ValueError, match="post"):
        mm.MatrixFactorizationModel(schema, 16, post="softmax")


def test_checkpoint_variable_names():
    schema = datasets.movielens_1m_schema()
    model = mm.MatrixFactorizationModel(schema, 8)
    model.build("cpu")
    w = model.weights()
    # TwoTowerModel's layout: the query / item towers' input blocks under the model's body
    assert sorted(w) == ["body/item/inputs/movieId/embeddings", "body/query/inputs/userId/embeddings"]
    assert tuple(w["body/query/inputs/userId/embeddings"].shape) == (6041, 8)


def _golden():
    z = np.load(GOLDEN)
    return z, [(f"T{float(t):g}".replace(".", "p"), float(t)) for t in z["temperatures"]]


@pytest.mark.parametrize("variant", [0, 1])
def test_restatement_matches_the_reference_step(variant):
    z, variants = _golden()
    vt, T = variants[variant]
    batch, towers, _ = O.golden_inputs(z)
    loss, reg, out, grads = O.mf_loss_and_grads(batch, towers, "movieId", temperature=T)
    assert reg == 0.0
    assert abs(loss - float(z[f"{vt}_loss"])) <= 1e-5 * abs(float(z[f"{vt}_loss"]))
    np.testing.assert_allclose(out["query"], z[f"{vt}_query_out"], rtol=1e-6, atol=1e-7)
    for tag in ("query", "item"):
        f = str(z[f"{tag}_cols"][0])
        want = z[f"{vt}_grad_{tag}_table_{f}_rows"]
        np.testing.assert_allclose(grads[f"{tag}/table/{f}"], want, rtol=2e-5, atol=2e-5 * np.abs(want).max())


def test_l2_term_and_its_closed_form_gradient():
    """reg = l2 sum_b ||e_b||^2 per tower; its gradient adds 2 l2 n_r e_r to row r looked up n_r times."""
    z, _ = _golden()
    batch, towers, _ = O.golden_inputs(z)
    lam = {"query": 3e-3, "item": 5e-4}
    l0, r0, _, g0 = O.mf_loss_and_grads(batch, towers, "movieId", temperature=0.5)
    l1, r1, _, g1 = O.mf_loss_and_grads(batch, towers, "movieId", temperature=0.5, l2_reg=lam)
    want_reg = 0.0
    for tag in ("query", "item"):
        f = next(iter(towers[tag]["tables"]))
        w = np.asarray(towers[tag]["tables"][f], np.float64)
        ids = np.asarray(batch[f]).reshape(-1)
        want_reg += lam[tag] * float((w[ids] ** 2).sum())
        n = np.bincount(ids, minlength=w.shape[0]).astype(np.float64)
        np.testing.assert_allclose(g1[f"{tag}/table/{f}"] - g0[f"{tag}/table/{f}"], 2 * lam[tag] * n[:, None] * w, rtol=1e-9,
                                   atol=1e-12)
    assert r0 == 0.0 and abs(r1 - want_reg) <= 1e-12 * want_reg
    assert abs((l1 - l0) - r1) <= 1e-12 * abs(l1)
