"""CPU checks of WideAndDeepModel: constructor semantics and the configurations it refuses, the wide kernel's layout,
CategoryEncoding's modes against a numpy bincount, and the float64 restatement (tests/wide_deep_train_oracle.py) tied to
its numpy forward and to the closed-form gradient of the wide kernel."""
import warnings

import numpy as np
import pytest

import models_b200 as mm
from models_b200.models import WideAndDeepBody
from models_b200.schema import ColumnSchema, Schema, Tags
from tests.wide_deep_train_oracle import BCE, MSE, bags_of, encode, encode_sparse, wide_deep_forward, wide_deep_loss_and_grads

CATS = [("C1", 30), ("C3", 3), ("C5", 400), ("C7", 7)]
LISTS = [("L2", 50), ("L4", 9)]
CONTS = ["I1", "I2"]


def schema(cats=CATS, lists=LISTS, conts=CONTS, ragged=True):
    cols = [ColumnSchema(n, tags=(Tags.CATEGORICAL,), dtype="int64", properties={"domain": {"min": 0, "max": mx, "name": n}})
            for n, mx in cats]
    cols += [ColumnSchema(n, tags=(Tags.CATEGORICAL,), dtype="int64", is_list=True, is_ragged=ragged,
                          properties={"domain": {"min": 0, "max": mx, "name": n}}) for n, mx in lists]
    cols += [ColumnSchema(n, tags=(Tags.CONTINUOUS,), dtype="float32") for n in conts]
    cols.append(ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"))
    return Schema(cols)


def test_reference_example_builds_both_branches():
    s = schema()
    wide_schema = s.select_by_name(["C1", "C3", "I1"])
    m = mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([32, 16]), wide_schema=wide_schema, deep_schema=s,
                            prediction_tasks=mm.BinaryOutput("click"))
    body = m.body
    assert isinstance(body, WideAndDeepBody)
    # the continuous column of wide_schema adds no wide rows; blocks in sorted-name order
    assert body.wide.names == ["C1", "C3"]
    assert body.wide.offsets == {"C1": 0, "C3": 31}
    assert body.wide.width == 31 + 4
    assert body.wide.mode == "one_hot"
    assert [l.units for l in body.deep.dense_layers] == [32, 16]
    logit = body.deep_logit.dense_layers
    assert len(logit) == 1 and logit[0].units == 1 and logit[0].activation == "linear" and logit[0].use_bias
    # the deep input block covers every input feature of deep_schema (target excluded) at inferred widths
    assert sorted(body.input_block.embeddings.feature_names) == sorted(n for n, _ in CATS + LISTS)
    assert body.input_block.continuous.features == CONTS
    assert all(t.sequence_combiner == "mean" for t in body.input_block.embeddings.tables.values())


def test_multi_hot_preprocess_and_layout():
    s = schema()
    ws = s.select_by_name(["L4", "C7", "L2"])
    m = mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]), wide_schema=ws,
                            wide_preprocess=mm.CategoryEncoding(ws, output_mode="multi_hot", sparse=True))
    w = m.body.wide
    assert w.names == ["C7", "L2", "L4"] and w.mode == "multi_hot"
    assert w.offsets == {"C7": 0, "L2": 8, "L4": 59} and w.width == 69
    # the reference wraps the default encoding in a tuple; one CategoryEncoding in a tuple is accepted too
    m2 = mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]), wide_schema=ws, wide_preprocess=(mm.CategoryEncoding(ws, output_mode="count"),))
    assert m2.body.wide.mode == "count"


def test_partial_models():
    s = schema()
    with pytest.warns(UserWarning, match="NO feature would be sent to wide model"):
        m = mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]))
    assert m.body.wide is None and m.body.deep is not None
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        m = mm.WideAndDeepModel(s, deep_block=None, wide_schema=s.select_by_name(["C1"]))
    assert m.body.input_block is None and m.body.wide.names == ["C1"]
    with pytest.raises(ValueError, match="At least the deep part"):
        with pytest.warns(UserWarning):
            mm.WideAndDeepModel(s, deep_block=None)


def test_rejections():
    s = schema()
    ws = s.select_by_name(["C1"])
    with pytest.raises(NotImplementedError, match="FarmHash"):
        mm.HashedCross(ws, num_bins=10)
    with pytest.raises(NotImplementedError, match="FarmHash"):
        mm.HashedCrossAll(ws, num_bins=10)
    with pytest.raises(NotImplementedError, match="wide_input_block"):
        mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]), wide_schema=ws, wide_input_block=mm.MLPBlock([1]))
    with pytest.raises(NotImplementedError, match="pre="):
        mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]), wide_schema=ws, pre=mm.MLPBlock([1]))
    with pytest.raises(NotImplementedError, match="count_weights"):
        mm.CategoryEncoding(ws, output_mode="count", count_weights=np.ones(3))
    with pytest.raises(ValueError, match="count_weights"):
        mm.CategoryEncoding(ws, output_mode="multi_hot", count_weights=np.ones(3))
    with pytest.raises(ValueError, match="output_mode"):
        mm.CategoryEncoding(ws, output_mode="tf_idf")
    with pytest.raises(NotImplementedError, match="several outputs"):
        mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]), wide_schema=ws,
                            prediction_tasks=mm.OutputBlock(s.select_by_name(["click"]) + Schema([
                                ColumnSchema("r", tags=(Tags.TARGET, Tags.REGRESSION), dtype="float32")])))
    with pytest.raises(ValueError, match="not in wide_schema"):
        mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]), wide_schema=ws, wide_preprocess=mm.CategoryEncoding(s.select_by_name(["C3"])))
    with pytest.raises(NotImplementedError, match="512"):
        mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([1024]), wide_schema=ws)
    enc = mm.CategoryEncoding(ws)
    with pytest.raises(NotImplementedError, match="fused"):
        enc({})


@pytest.mark.parametrize("mode", ["one_hot", "multi_hot", "count"])
def test_encoding_against_bincount(mode):
    g = np.random.default_rng(3)
    card = 11
    one = g.integers(0, card, 9)
    fixed = g.integers(0, card, (9, 5))
    fixed[0] = [2, 2, 2, 5, 5]
    offs = np.array([0, 0, 3, 3, 7, 7, 8, 12, 12, 14])
    vals = g.integers(0, card + 2, 14)
    for x in (one, fixed, (vals, offs)):
        if mode == "one_hot" and not (isinstance(x, np.ndarray) and x.ndim == 1):
            continue
        e = encode(x, card, mode)
        for b, ids in enumerate(bags_of(x)):
            ids = ids[(ids >= 0) & (ids < card)]
            c = np.bincount(ids, minlength=card)
            assert np.array_equal(e[b], np.minimum(c, 1) if mode != "count" else c)
    assert encode(fixed, card, "multi_hot")[0].sum() == 2 and encode(fixed, card, "count")[0].sum() == 5
    assert encode((vals, offs), card, mode)[0].sum() == 0  # an empty bag encodes to nothing


def _state(g, mode, conts=("I1",), U=(6,)):
    cards = {"C1": 13, "L2": 9}
    wide = {"cards": cards, "mode": mode, "kernel": g.standard_normal((22, 1)) * 0.3, "bias": g.standard_normal(1) * 0.1}
    tables = {"C1": g.standard_normal((13, 4)) * 0.3, "L2": g.standard_normal((9, 4)) * 0.3}
    layers, k = [], 8 + len(conts)
    for u in U:
        layers.append({"kernel": g.standard_normal((k, u)) / np.sqrt(k), "bias": g.standard_normal(u) * 0.1, "activation": "relu"})
        k = u
    deep = {"tables": tables, "continuous": list(conts), "layers": layers,
            "logit": {"kernel": g.standard_normal((k, 1)), "bias": g.standard_normal(1) * 0.1, "activation": "linear"}}
    head = {"kernel": g.standard_normal((1, 1)), "bias": g.standard_normal(1) * 0.1, "loss": BCE, "activation": "sigmoid"}
    return wide, deep, head


def _batch(g, B, ragged):
    b = {"C1": g.integers(0, 13, B), "I1": g.standard_normal(B)}
    if ragged:
        lens = g.integers(0, 5, B)
        b["L2"] = (g.integers(0, 9, int(lens.sum())), np.concatenate([[0], np.cumsum(lens)]))
    else:
        b["L2"] = g.integers(0, 9, (B, 4))
    return b


@pytest.mark.parametrize("mode", ["multi_hot", "count"])
@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("loss", [BCE, MSE])
def test_restatement_matches_forward_and_closed_form(mode, ragged, loss):
    """The autograd restatement's z equals the numpy forward, and its wide gradients equal the closed form:
    dWk = E^T ds and dbw = sum ds, with ds = dloss/dz * w_out and E the concatenated encodings."""
    g = np.random.default_rng(7)
    wide, deep, head = _state(g, mode)
    head["loss"] = loss
    B = 23
    batch = _batch(g, B, ragged)
    y = g.integers(0, 2, B) if loss == BCE else g.standard_normal(B)
    sw = g.random(B) * 2
    L, z, grads = wide_deep_loss_and_grads(batch, wide, deep, head, y, sample_weight=sw)
    np.testing.assert_allclose(z, wide_deep_forward(batch, wide, deep, head, logits=True), rtol=1e-12, atol=1e-12)
    delta = ((1 / (1 + np.exp(-z)) - y) if loss == BCE else 2 * (z - y)) * sw / B
    ds = delta * float(head["kernel"][0, 0])
    E = np.concatenate([encode(batch[n], wide["cards"][n], mode) for n in sorted(wide["cards"])], axis=1)
    np.testing.assert_allclose(grads["wide/kernel"].reshape(-1), E.T @ ds, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(grads["wide/bias"].reshape(-1), [ds.sum()], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(grads["head/bias"].reshape(-1), [delta.sum()], rtol=1e-10, atol=1e-12)


def test_the_callers_encoding_is_not_modified():
    """A categorical target in wide_schema gets no wide rows; the CategoryEncoding passed in keeps its own cardinalities
    (another model may share it)."""
    s = Schema(list(schema()) + [ColumnSchema("cat_target", tags=(Tags.CATEGORICAL, Tags.TARGET), dtype="int64",
                                              properties={"domain": {"min": 0, "max": 4, "name": "cat_target"}})])
    ws = s.select_by_name(["C1", "cat_target"])
    enc = mm.CategoryEncoding(ws, output_mode="multi_hot")
    before = dict(enc.cardinalities)
    m = mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]), wide_schema=ws, wide_preprocess=enc, prediction_tasks=mm.BinaryOutput("click"))
    assert m.body.wide.names == ["C1"] and m.body.wide.width == 31
    assert enc.cardinalities == before == {"C1": 31, "cat_target": 5}
    m2 = mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]), wide_schema=s.select_by_name(["C1", "cat_target", "C3"]),
                             wide_preprocess=enc, prediction_tasks=mm.BinaryOutput("click"))
    assert m2.body.wide.names == ["C1"]


def test_packed_uint8_list_is_refused():
    """A uint8 (B, 3) matrix is the package's packed 24-bit id of a scalar column; for a list column it is refused before
    any kernel runs, not read as one id per sample."""
    import torch

    s = schema(ragged=False)
    ws = s.select_by_name(["C1", "L2"])
    m = mm.WideAndDeepModel(s, deep_block=None, wide_schema=ws, wide_preprocess=mm.CategoryEncoding(ws, output_mode="multi_hot"))
    x = {"C1": torch.zeros((4, 3), dtype=torch.uint8), "L2": torch.zeros((4, 3), dtype=torch.uint8)}
    with pytest.raises(ValueError, match="list feature 'L2'.*packed 24-bit"):
        m.body.wide.blocks(x)
    onehot, bags = m.body.wide.blocks({"C1": x["C1"], "L2": x["L2"].to(torch.int32)})
    assert len(onehot) == 1 and onehot[0][0].dtype == torch.uint8 and len(bags) == 1 and bags[0][0].shape == (4, 3)


@pytest.mark.parametrize("mode", ["one_hot", "multi_hot", "count"])
def test_sparse_encoding_equals_the_dense_one(mode):
    """encode_sparse against encode on one-hot ids, fixed bags with repeats and ragged bags whose offsets leave values
    uncovered, go backwards and run past the end (clamped as bags_of does); out-of-range and negative ids encode to nothing."""
    g = np.random.default_rng(5)
    card = 11
    one = g.integers(-1, card + 2, 40)
    fixed = g.integers(-1, card + 2, (40, 6))
    fixed[0] = 4
    offs = np.array([2, 2, 5, 4, 9, 9, 13, 30])
    vals = g.integers(-1, card + 2, 20)
    for x in (one, fixed, (vals, offs)):
        if mode == "one_hot" and not (isinstance(x, np.ndarray) and x.ndim == 1):
            continue
        np.testing.assert_array_equal(encode_sparse(x, card, mode).toarray(), encode(x, card, mode))


@pytest.mark.parametrize("mode", ["multi_hot", "count"])
@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("loss", [BCE, MSE])
def test_sparse_restatement_equals_the_dense_one(mode, ragged, loss):
    """wide_deep_loss_and_grads(sparse=True) (CSR encodings and mean pools, closed-form wide and pooled-table gradients)
    gives the dense path's loss, logits and every gradient."""
    g = np.random.default_rng(11)
    wide, deep, head = _state(g, mode)
    head["loss"] = loss
    B = 37
    batch = _batch(g, B, ragged)
    batch["L2"] = batch["L2"] if ragged else np.where(g.random((B, 4)) < 0.1, 12, batch["L2"])  # out-of-range ids in bags
    y = g.integers(0, 2, B) if loss == BCE else g.standard_normal(B)
    sw = g.random(B) * 2
    L, z, grads = wide_deep_loss_and_grads(batch, wide, deep, head, y, sample_weight=sw)
    Ls, zs, gs = wide_deep_loss_and_grads(batch, wide, deep, head, y, sample_weight=sw, sparse=True)
    assert abs(Ls - L) <= 1e-12 * max(1.0, abs(L))
    np.testing.assert_allclose(zs, z, rtol=1e-12, atol=1e-12)
    assert sorted(gs) == sorted(grads)
    for k in grads:
        np.testing.assert_allclose(gs[k], grads[k], rtol=1e-10, atol=1e-12, err_msg=k)
