"""Model(InputBlockV2, MLPBlock, CategoricalOutput) without a GPU: the float64 restatement of the step
(tests/catalog_model_oracle.py) against the kernel-level restatement and central finite differences, the constructor's
rules and refusals, `target_name`, the weight names, and the dense update rule of the tied table."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200.schema import Tags
from tests import catalog_model_oracle as O
from tests.catalog_train_oracle import catalog_ce


def cpu_model(n_items, D, tied, **kw):
    """The model with its variables created on the CPU (the restatement reads them; nothing runs a kernel)."""
    model, s, table = O.build(n_items, D, tied, **kw)
    g = torch.Generator().manual_seed(0)
    for tb in list(model.body.input_block.embeddings.tables.values()) + [table]:
        if tb.table is None:
            tb.table = torch.randn(tb.input_dim, tb.dim, generator=g, dtype=torch.float64).float() * 0.3
    d = model.body.input_block.layout()[2]
    for l in model.mlp.dense_layers:
        l.kernel = torch.randn(d, l.units, generator=g).float() * 0.3
        l.bias = torch.randn(l.units, generator=g).float() * 0.1
        d = l.units
    if model.prediction.use_bias:
        model.prediction.bias = torch.randn(n_items, generator=g).float() * 0.2
    return model, s, table


@pytest.mark.parametrize("tied", ["onehot", "list", "none"])
def test_restatement_output_side_matches_kernel_restatement(tied):
    """The output layer's part of the step equals catalog_train_oracle.catalog_ce (the kernels' float64 restatement)."""
    model, s, table = cpu_model(60, 8, tied, T=0.05)
    feats, y = O.batch(s, 60, 20, seed=1, hot=3)
    sw = np.linspace(0.5, 1.5, 20)
    loss, g = O.restated_step(model, feats, y, sw)
    # the query x, restated once more in numpy
    ib = model.body.input_block
    cols, _, d = ib.layout()
    x = np.zeros((20, d))
    for f, tb in ib.embeddings.feature_to_table.items():
        E = tb.table.double().numpy()
        ids = feats[f]
        x[:, cols[f]:cols[f] + tb.dim] = E[ids] if ids.ndim == 1 else E[ids].mean(1)
    for n in ("c1", "c2"):
        x[:, cols[n]] = feats[n]
    for l in model.mlp.dense_layers:
        x = x @ l.kernel.double().numpy() + l.bias.double().numpy()
        if l.activation == "relu":
            x = np.maximum(x, 0)
    rl, _, rde, rdb = catalog_ce(x, table.table.double().numpy(), model.prediction.bias.double().numpy(), y, 0.05, sw)
    assert abs(loss - rl) < 1e-10
    np.testing.assert_allclose(g["bias"], rdb, rtol=1e-9, atol=1e-12)
    if tied == "none":  # no input side: the tied gradient is the output side alone
        np.testing.assert_allclose(g["tables/item_id"], rde, rtol=1e-9, atol=1e-12)
    else:  # the input side adds rows only where the batch looked items up
        looked = np.unique(feats["last_item" if tied == "onehot" else "item_history"])
        other = np.setdiff1d(np.arange(60), looked)
        np.testing.assert_allclose(g["tables/item_id"][other], rde[other], rtol=1e-9, atol=1e-12)
        assert np.abs(g["tables/item_id"][looked] - rde[looked]).max() > 1e-6


@pytest.mark.parametrize("tied", ["onehot", "list"])
def test_restatement_gradients_against_finite_differences(tied):
    model, s, table = cpu_model(30, 4, tied, T=0.5, widths=(6,))
    feats, y = O.batch(s, 30, 9, seed=2, hot=2)
    _, g = O.restated_step(model, feats, y)
    rng = np.random.default_rng(0)
    for name, var in (("tables/item_id", table), ("bias", model.prediction), ("mlp/0/kernel", model.mlp.dense_layers[0])):
        t = var.table if name.startswith("tables") else (var.bias if name == "bias" else var.kernel)
        base = t.clone()
        for _ in range(4):
            idx = tuple(int(rng.integers(0, n)) for n in t.shape)
            h = 1e-3
            vals = []
            for sgn in (1, -1):
                t.copy_(base)
                t[idx] += sgn * h
                vals.append(O.restated_step(model, feats, y)[0])
            t.copy_(base)
            fd = (vals[0] - vals[1]) / (2 * h)
            assert abs(fd - g[name][idx]) <= 2e-3 * max(1e-3, abs(fd)), (name, idx, fd, g[name][idx])


def test_target_name_defaults_to_the_tables_column():
    s = O.schema(40, "onehot")
    emb = mm.Embeddings(s.select_by_tag(Tags.CATEGORICAL), dim=8)
    assert mm.CategoricalOutput(emb.tables["item_id"]).target_name == "last_item"
    assert mm.CategoricalOutput(emb.tables["item_id"], target_name="next_item").target == "next_item"
    assert mm.CategoricalOutput(emb.tables["item_id"]).use_bias  # the torch EmbeddingTablePrediction default, kept
    assert mm.CategoricalOutput(emb.tables["item_id"], target="next_item").target_name == "next_item"  # the Keras keyword
    with pytest.raises(ValueError, match="different columns"):
        mm.CategoricalOutput(emb.tables["item_id"], target="a", target_name="b")


def test_restatement_against_the_reference_golden():
    """One step of the reference's torch modules (tests/golden/make_golden_catalog_train.py: a mean-pooled item history
    tied to EmbeddingTablePrediction, duplicate ids, T = 0.05, a bias, sample weights) against the restatement: the
    sorted-name concat, the pooling, T on the bias and the tied gradient's two paths."""
    model, feats, y, sw, z = O.golden_model()
    loss, g = O.restated_step(model, feats, y, sw)
    assert abs(loss - float(z["loss"])) <= 1e-6 * abs(loss)
    np.testing.assert_allclose(O.restated_query(model, feats), z["query"], rtol=1e-5, atol=1e-6)
    for name, want in O.golden_grads(z).items():
        np.testing.assert_allclose(g[name], want, rtol=1e-4, atol=1e-6 * np.abs(want).max(), err_msg=name)


def test_constructor_rules():
    model, s, table = O.build(40, 8, "onehot")
    assert isinstance(model, mm.CatalogModel) and model.mlp.dense_layers[-1].units == 8
    emb = model.body.input_block.embeddings
    ib = mm.InputBlockV2(s, categorical=emb)
    with pytest.raises(ValueError, match="16 units.*8 wide"):
        mm.Model(ib, mm.MLPBlock([16]), mm.CategoricalOutput(table))
    with pytest.raises(NotImplementedError, match="MMOEBlock"):
        mm.Model(ib, mm.MLPBlock([8]), mm.MMOEBlock(outputs=["a"], num_experts=2, expert_block=mm.MLPBlock([8])), mm.CategoricalOutput(table))
    with pytest.raises(NotImplementedError, match="exactly one MLPBlock"):
        mm.Model(ib, mm.MLPBlock([8]), mm.MLPBlock([8]), mm.CategoricalOutput(table))
    with pytest.raises(NotImplementedError, match="exactly one MLPBlock"):
        mm.Model(ib, mm.CategoricalOutput(table))


def test_training_refusals():
    from models_b200.blocks import set_dense_engine

    model, s, table = O.build(40, 8, "onehot")
    model.compile(optimizer="sgd")
    with pytest.raises(NotImplementedError, match="process group"):
        mm.train.CatalogTrainer(model, model.optimizer, 4, group=object())
    set_dense_engine("fp32")
    try:
        with pytest.raises(NotImplementedError, match="fp32"):
            mm.train.CatalogTrainer(model, model.optimizer, 4)
    finally:
        set_dense_engine("tc")
    wide, _, _ = O.build(40, 132, "none")
    wide.compile(optimizer="sgd")
    with pytest.raises(NotImplementedError, match="128"):
        mm.train.CatalogTrainer(wide, wide.optimizer, 4)
    multi, _, _ = O.build(40, 8, "list")  # a multi-hot tied table at a width the bag backward does not take
    multi.compile(optimizer="sgd")
    with pytest.raises(NotImplementedError, match="item_history"):
        mm.train.CatalogTrainer(multi, multi.optimizer, 4, device="cpu")
    with pytest.raises(NotImplementedError, match="categorical_crossentropy"):
        model.compile(optimizer="sgd", loss="mse")


def test_weight_names():
    names = set(cpu_model(40, 8, "onehot", widths=(16,))[0].weights())
    assert "prediction/embeddings" in names and "prediction/bias" in names
    assert "body/input/embeddings/item_id/embeddings" in names and "body/input/embeddings/user_id/embeddings" in names
    assert sum(n.startswith("body/bottom/") for n in names) == 4  # two Dense layers: kernel and bias each


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam", "lazyadam"])
def test_dense_update_rule_of_the_tied_table(opt):
    """The restatement's Keras rules on a dense gradient (LazyAdam on a dense gradient is Adam), which
    test_gpu_catalog_model.py::test_tied_table_update_rule holds the trainer's tied table to."""
    rng = np.random.default_rng(3)
    w, g = rng.standard_normal((5, 4)), rng.standard_normal((5, 4))
    kind = "adam" if opt == "lazyadam" else opt
    w1, s1, s2 = O.dense_update(kind, w, g, np.full_like(w, 0.1 if kind == "adagrad" else 0.0), np.zeros_like(w), 0.01, 1)
    assert np.all(w1 != w)
    if kind == "sgd":
        np.testing.assert_allclose(w1, w - 0.01 * g)
    elif kind == "adagrad":
        np.testing.assert_allclose(w1, w - 0.01 * g / (np.sqrt(0.1 + g * g) + 1e-7))
    else:  # the first Adam step moves every element by about lr
        np.testing.assert_allclose(np.abs(w1 - w), 0.01, rtol=1e-3)
    assert isinstance(mm.train.get_optimizer(opt), mm.train.Optimizer)
