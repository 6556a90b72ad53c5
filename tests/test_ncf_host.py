"""NCFModel without a GPU: the constructor and its defaults, the four tables and their names, the column orders, the
kwargs that reach the mf branch only, the refusals, the float64 restatement against the reference's torch fixture and
its L2 gradient against finite differences, and the GPU kernel cases' reach."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets
from models_b200.schema import ColumnSchema, Schema, Tags
from tests.ncf_train_oracle import golden_inputs, ncf_loss_and_grads

GOLDEN = Path(__file__).resolve().parent / "golden" / "ncf_train" / "ref_torch_ncf_train.npz"


def _cat(name, rows, tags, is_list=False):
    props = {"domain": {"min": 0, "max": rows - 1, "name": name}}
    if is_list:
        props["value_count"] = {"min": 1, "max": None}
    return ColumnSchema(name, tags=(Tags.CATEGORICAL,) + tuple(tags), dtype="int64", properties=props, is_list=is_list,
                        is_ragged=is_list)


def _schema(user="a_user", item="z_item", extra=()):
    return Schema([_cat(user, 50, (Tags.USER, Tags.USER_ID)), _cat(item, 70, (Tags.ITEM, Tags.ITEM_ID)), *extra,
                   ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64")])


def test_constructor_defaults_and_path():
    import inspect

    assert mm.benchmark.NCFModel is mm.benchmark.__dict__["NCFModel"]
    sig = inspect.signature(mm.benchmark.NCFModel)
    assert list(sig.parameters)[:5] == ["schema", "embedding_dim", "mlp_block", "prediction_tasks", "embeddings_l2_reg"]
    assert sig.parameters["prediction_tasks"].default is None and sig.parameters["embeddings_l2_reg"].default == 0.0
    model = mm.benchmark.NCFModel(datasets.movielens_1m_schema(), 16, mm.MLPBlock([32, 8]))
    assert isinstance(model, mm.models.RankingModel) and isinstance(model.body, mm.models.NCFBody)
    assert sorted(o.name for o in model.output_blocks()) == ["rating/regression_output", "rating_binary/binary_output"]
    assert all(l.activation == "relu" for l in model.body.mlp.dense_layers)


def test_four_tables_names_and_independent_initial_values():
    mm.set_seed(3)
    model = mm.benchmark.NCFModel(_schema(), 8, mm.MLPBlock([16, 4]))
    model.build("cpu")
    w = model.weights()
    tables = {k: v for k, v in w.items() if k.endswith("/embeddings")}
    assert sorted(tables) == ["body/mf/item/inputs/z_item/embeddings", "body/mf/query/inputs/a_user/embeddings",
                              "body/mlp/item/inputs/z_item/embeddings", "body/mlp/query/inputs/a_user/embeddings"]
    assert not torch.equal(tables["body/mf/query/inputs/a_user/embeddings"], tables["body/mlp/query/inputs/a_user/embeddings"])
    assert not torch.equal(tables["body/mf/item/inputs/z_item/embeddings"], tables["body/mlp/item/inputs/z_item/embeddings"])
    assert len({id(t) for t in tables.values()}) == 4
    mlp = [k for k in w if k.startswith("body/mlp/mlp/")]
    assert len(mlp) == 4 and all(k.endswith(("/kernel", "/bias")) for k in mlp)


def test_column_orders_item_first_then_mf_before_mlp():
    model = mm.benchmark.NCFModel(_schema("a_user", "z_item"), 8, mm.MLPBlock([16, 4]))
    model.build("cpu")
    body = model.body
    assert body.mlp_columns == {"z_item": 0, "a_user": 8}  # [item | query] although the user column sorts first
    assert body.mlp.dense_layers[0].kernel.shape == (16, 16)
    assert body.output_width() == 8 + 4 and model.prediction.to_call.kernel.shape == (12, 1)  # rows [mf (8) | mlp (4)]


def test_kwargs_reach_the_mf_branch_only():
    # query_id_tag reaching the mf branch: a tag that selects one column there, while the mlp branch keeps USER_ID
    s = Schema([_cat("a_user", 50, (Tags.USER_ID,)), _cat("u2", 40, ("my_user",)), _cat("z_item", 70, (Tags.ITEM_ID,)),
                ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64")])
    model = mm.benchmark.NCFModel(s, 8, mm.MLPBlock([4]), query_id_tag="my_user", embeddings_initializers="zeros")
    model.build("cpu")
    body = model.body
    assert body.feature("mf", "query") == "u2" and body.feature("mlp", "query") == "a_user"
    assert not body.table("mf", "query").embeddings.any() and not body.table("mf", "item").embeddings.any()
    assert body.table("mlp", "query").embeddings.abs().sum() > 0 and body.table("mlp", "item").embeddings.abs().sum() > 0


def test_refusals():
    mlp = lambda: mm.MLPBlock([8])  # noqa: E731
    with pytest.raises(ValueError, match="embeddings_l2_reg"):
        mm.benchmark.NCFModel(_schema(), 8, mlp(), embeddings_l2_reg=-1.0)
    with pytest.raises(ValueError, match="user_id|USER_ID|Tags.USER_ID"):
        mm.benchmark.NCFModel(Schema([_cat("i", 5, (Tags.ITEM_ID,)), ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION))]),
                              8, mlp())
    with pytest.raises(NotImplementedError, match="exactly one non-list id column"):
        mm.benchmark.NCFModel(_schema(extra=[_cat("u2", 9, (Tags.USER_ID,))]), 8, mlp())
    with pytest.raises(NotImplementedError, match="exactly one non-list id column"):
        s = Schema([_cat("u", 9, (Tags.USER_ID,), is_list=True), _cat("i", 9, (Tags.ITEM_ID,)),
                    ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION))])
        mm.benchmark.NCFModel(s, 8, mlp())
    for d in (6, 132):
        with pytest.raises(NotImplementedError, match="embedding_dim"):
            mm.benchmark.NCFModel(_schema(), d, mlp())
    with pytest.raises(NotImplementedError, match="256 units"):
        mm.benchmark.NCFModel(_schema(), 8, mm.MLPBlock([300]))
    with pytest.raises(NotImplementedError, match="task_blocks|per-task towers"):
        mm.benchmark.NCFModel(_schema(), 8, mlp(), prediction_tasks=mm.OutputBlock(_schema(), task_blocks=mm.MLPBlock([4])))
    with pytest.raises(NotImplementedError, match="post"):
        mm.benchmark.NCFModel(_schema(), 8, mlp(), post="l2-norm")


@pytest.mark.parametrize("what", ["group", "fp32", "sharded", "normalization", "dropout", "activation"])
def test_training_refusals(what):
    from models_b200.blocks import set_dense_engine
    from models_b200.train import trainer_for

    block = {"normalization": mm.MLPBlock([8], normalization="batch_norm"), "dropout": mm.MLPBlock([8], dropout=0.1),
             "activation": mm.MLPBlock([8], activation="tanh")}.get(what, mm.MLPBlock([8]))
    model = mm.benchmark.NCFModel(_schema(), 8, block)
    if what == "sharded":
        model.body.mf.item.inputs.embeddings.sharded = object()
    set_dense_engine("fp32" if what == "fp32" else "auto")
    try:
        match = {"group": "process group", "fp32": "tensor-core engine", "sharded": "row-sharded", "normalization": "normalization",
                 "dropout": "dropout", "activation": "activations"}[what]
        with pytest.raises(NotImplementedError, match=match):
            trainer_for(model, mm.SGD(0.1), 8, group=object() if what == "group" else None)
    finally:
        set_dense_engine("auto")


def test_restatement_matches_fixture():
    z = np.load(GOLDEN)
    ids, p, ys, losses = golden_inputs(z)
    loss, reg, per, Z, g = ncf_loss_and_grads(ids, p, losses, ys)
    assert reg == 0.0 and abs(loss - float(z["loss"])) < 1e-6 * abs(loss)
    outs = [str(n) for n in z["outputs"]]
    for t, n in enumerate(outs):
        pred = Z[t] if losses[t] == "mse" else 1 / (1 + np.exp(-Z[t]))
        np.testing.assert_allclose(pred, z[f"pred_{n}"], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(g["head_kernel"][:, t:t + 1], z[f"grad_head_{n}_kernel"], rtol=1e-4, atol=1e-6)
    for b in ("mf", "mlp"):
        for s in ("query", "item"):
            np.testing.assert_allclose(g[f"{b}/{s}"], z[f"grad_{b}_{s}_rows"], rtol=1e-4, atol=1e-7)
    for i in range(len(z["units"])):
        np.testing.assert_allclose(g[f"kernel_{i}"], z[f"grad_mlp_kernel_{i}"], rtol=1e-4, atol=1e-7)


def test_restatement_l2_gradient_matches_finite_differences():
    z = np.load(GOLDEN)
    ids, p, ys, losses = golden_inputs(z)
    l2 = 0.05
    _, reg, _, _, g = ncf_loss_and_grads(ids, p, losses, ys, l2=l2)
    _, _, _, _, g0 = ncf_loss_and_grads(ids, p, losses, ys, l2=0.0)
    assert reg > 0
    eps = 1e-6
    for k in ("mf/query", "mlp/item"):
        for r, c in ((0, 0), (3, 5)):
            q = {kk: (np.array(v, dtype=np.float64) if kk == k else v) for kk, v in p.items()}
            q[k][r, c] += eps
            lp = ncf_loss_and_grads(ids, q, losses, ys, l2=l2)[0]
            q[k][r, c] -= 2 * eps
            lm = ncf_loss_and_grads(ids, q, losses, ys, l2=l2)[0]
            fd = (lp - lm) / (2 * eps)
            assert abs(fd - g[k][r, c]) < 1e-6 + 1e-5 * abs(fd)
            # the L2 part alone: 2 l2 e times the row's number of occurrences in the batch
            n = int((ids[k.split("/")[1]] == r).sum())
            assert abs((g[k][r, c] - g0[k][r, c]) - 2 * l2 * n * np.asarray(p[k])[r, c]) < 1e-7


def test_kernel_cases_reach_every_instantiation():
    from tests.test_gpu_ncf import KERNEL_CASES

    nh = lambda h: 1 if h == 1 else 2 if h == 2 else 4 if h <= 4 else 8  # noqa: E731
    cd = lambda d: 1 if d <= 32 else 2 if d <= 64 else 4  # noqa: E731
    cu = lambda u: 1 if u <= 32 else 2 if u <= 64 else 4 if u <= 128 else 8  # noqa: E731
    reached = {(nh(H), cd(D), cu(U)) for D, U, H, *_ in KERNEL_CASES}
    assert reached == {(a, b, c) for a in (1, 2, 4, 8) for b in (1, 2, 4) for c in (1, 2, 4, 8)}
    assert {D for D, *_ in KERNEL_CASES} >= {4, 16, 64, 128} and {U for _, U, *_ in KERNEL_CASES} >= {8, 48, 64, 200, 256}
    assert {B for *_, B, _, _, _ in [(c[0], c[1], c[2], c[3], c[4], c[5], c[6]) for c in KERNEL_CASES]} >= {1, 37, 4099, 65536}
    assert {c[4] for c in KERNEL_CASES} == {1, 2, 3, 4, 8} and {c[5] for c in KERNEL_CASES} == {0.0, 1e-3}
