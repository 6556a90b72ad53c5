"""CPU checks of the DeepFM training step: the float64 restatement (tests/deepfm_train_oracle.py) against the forward oracle
that tests/test_gpu_fm.py trusts (oracle.deepfm_forward) and against the closed-form backward, the wide kernel's layout, and
the configurations DeepFMTrainer refuses (all refused before any device work)."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200.schema import ColumnSchema, Schema, Tags
from oracle import oracle
from tests.deepfm_train_oracle import BCE, MSE, deepfm_loss_and_grads

CATS = [("C1", 300), ("C3", 3), ("C5", 40000), ("C7", 7)]
CONTS = ["C2", "C4", "C6"]


def schema(conts=CONTS, cats=CATS, target="click"):
    cols = [ColumnSchema(n, tags=(Tags.CATEGORICAL,), dtype="int64", properties={"domain": {"min": 0, "max": mx, "name": n}})
            for n, mx in cats]
    cols += [ColumnSchema(n, tags=(Tags.CONTINUOUS,), dtype="float32") for n in conts]
    if target == "rating":
        cols.append(ColumnSchema(target, tags=(Tags.TARGET, Tags.REGRESSION), dtype="float32"))
    else:
        cols.append(ColumnSchema(target, tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"))
    return Schema(cols)


def _random_state(g, conts, D=8, deep=(16, 8), logit=(1,)):
    card = {n: mx + 1 for n, mx in CATS}
    tables = {n: g.standard_normal((c, D)) * 0.3 for n, c in card.items()}
    off, offsets = 0, {}
    for n in sorted(list(card) + list(conts)):
        offsets[n] = off
        off += card.get(n, 1)
    wide_k, wide_b = g.standard_normal((off, 1)) * 0.2, g.standard_normal(1) * 0.1
    d = len(card) * D + len(conts)
    layers, k = [], d
    for u in deep:
        layers.append({"kernel": g.standard_normal((k, u)) / np.sqrt(k), "bias": g.standard_normal(u) * 0.1, "activation": "relu"})
        k = u
    logit_layers = []
    for i, u in enumerate(logit):
        logit_layers.append({"kernel": g.standard_normal((k, u)) / np.sqrt(k), "bias": g.standard_normal(u) * 0.1,
                             "activation": "linear" if i == len(logit) - 1 else "relu"})
        k = u
    head = {"kernel": g.standard_normal((1, 1)), "bias": g.standard_normal(1) * 0.1, "loss": BCE, "activation": "sigmoid"}
    return card, tables, offsets, wide_k, wide_b, layers, logit_layers, head


def _batch(g, B, conts, card):
    f = {n: g.integers(0, c, B).astype(np.int64) for n, c in card.items()}
    f.update({n: g.standard_normal(B).astype(np.float32) for n in conts})
    return f


@pytest.mark.parametrize("conts", [CONTS, []])
def test_restatement_forward_equals_the_forward_oracle(conts):
    """The restated z, through the output layer's sigmoid, equals oracle.deepfm_forward on random inputs to 1e-6."""
    g = np.random.default_rng(len(conts))
    card, tables, offsets, wk, wb, deep, logit, head = _random_state(g, conts, logit=(4, 1))
    batch = _batch(g, 257, conts, card)
    y = (g.random(257) < 0.5).astype(np.int64)
    _, z, _ = deepfm_loss_and_grads(batch, tables, conts, offsets, wk, wb, deep, logit, head, y)
    f32 = lambda ls: [{k: (v.astype(np.float32) if isinstance(v, np.ndarray) else v) for k, v in l.items()} for l in ls]  # noqa: E731
    want = oracle.deepfm_forward(batch, {n: t.astype(np.float32) for n, t in tables.items()}, {n: n for n in tables}, conts, card,
                                 wk.astype(np.float32), wb.astype(np.float32), f32(deep), f32(logit), f32([head])[0]).reshape(-1)
    got = 1.0 / (1.0 + np.exp(-z))
    assert np.max(np.abs(got - want)) < 1e-6, float(np.max(np.abs(got - want)))


@pytest.mark.parametrize("loss", [BCE, MSE])
def test_restatement_backward_equals_the_closed_form(loss):
    """Autograd of the restatement equals the backward the kernels compute: ds = delta w_out, d e_f = ds (S_f - e_f) summed over
    the samples of each row (plus the deep tower's part, zero here: the deep logit's kernel is zeroed), dWk rows = sums of ds."""
    g = np.random.default_rng(5)
    card, tables, offsets, wk, wb, deep, logit, head = _random_state(g, CONTS)
    logit[0]["kernel"] = np.zeros_like(logit[0]["kernel"])
    head["loss"] = loss
    B = 300
    batch = _batch(g, B, CONTS, card)
    y = g.random(B) * (3.0 if loss == MSE else 1.0)
    sw = g.random(B)
    _, z, grads = deepfm_loss_and_grads(batch, tables, CONTS, offsets, wk, wb, deep, logit, head, y, sample_weight=sw)
    if loss == BCE:
        delta = (1.0 / (1.0 + np.exp(-z)) - y) * sw / B
    else:
        delta = 2.0 * (z - y) * sw / B
    ds = delta * head["kernel"][0, 0]
    wide = np.zeros(wk.shape[0])
    for n in tables:
        e = tables[n][batch[n]]
        ge = ds[:, None] * (e.sum(1, keepdims=True) - e)
        want = np.zeros_like(tables[n])
        np.add.at(want, batch[n], ge)
        np.testing.assert_allclose(grads[f"table/{n}"], want, rtol=1e-9, atol=1e-12)
        np.add.at(wide, batch[n] + offsets[n], ds)
    for c in CONTS:
        wide[offsets[c]] = float(np.sum(ds * batch[c]))
    np.testing.assert_allclose(grads["wide/kernel"].reshape(-1), wide, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(grads["wide/bias"], [ds.sum()], rtol=1e-9)
    np.testing.assert_allclose(grads["head/bias"], [delta.sum()], rtol=1e-9)


def test_wide_offsets_follow_the_sorted_names():
    """The wide kernel's rows: one block of int_domain.max + 1 rows per categorical feature and one row per continuous column,
    in sorted-name order over all of them; the trainer's block and dense-row offsets are these."""
    mm.set_seed(1)
    m = mm.DeepFMModel(schema(), embedding_dim=8, deep_block=mm.MLPBlock([16]))
    fm = m.body.fm
    assert fm.wide_offsets == {"C1": 0, "C2": 301, "C3": 302, "C4": 306, "C5": 307, "C6": 40308, "C7": 40309}
    assert fm.wide_width == 40317
    cols, _, d = m.body.input_block.layout()
    assert d == 4 * 8 + 3 and cols["C3"] == 9 and cols["C3"] % 4  # feature rows at columns that are not multiples of 4


def _model(**kw):
    mm.set_seed(2)
    deep = kw.pop("deep", mm.MLPBlock([16]))
    return mm.DeepFMModel(schema(), embedding_dim=kw.pop("dim", 8), deep_block=deep, **kw)


def rejections(device):
    """(model, match, group) of every configuration DeepFMTrainer refuses."""
    out = [(_model(), "process group", object())]
    m = _model()
    m.build(device)
    m.body.input_block.embeddings.sharded = object()
    out.append((m, "row-sharded", None))
    m = _model()
    m.build(device)
    m.body.input_block.embeddings.feature_to_table["C7"].trainable = False
    out.append((m, "'C7'.*frozen", None))
    m = _model()
    m.build(device)
    emb = m.body.input_block.embeddings
    emb.feature_to_table["C7"] = emb.feature_to_table["C3"]
    out.append((m, "'C7'.*shared", None))
    out.append((_model(dim=6), "width 6", None))
    out.append((_model(dim=132), "width 132", None))
    out.append((_model(deep=mm.MLPBlock([16], activation="tanh")), "relu / linear", None))
    out.append((_model(deep_logit_block=mm.MLPBlock([1], activation="sigmoid")), "relu / linear", None))
    out.append((_model(deep=mm.MLPBlock([16], dropout=0.2)), "dropout", None))
    return out


def test_unsupported_configurations_name_their_cause():
    from models_b200.blocks import set_dense_engine
    from models_b200.train import SGD, DeepFMTrainer, trainer_for

    dev = torch.device("cpu")
    with pytest.raises(NotImplementedError, match="DeepFMModel with a process group"):  # trainer_for picks DeepFMTrainer
        trainer_for(_model(), SGD(0.1), 64, group=object())
    for model, match, group in rejections(dev):
        with pytest.raises(NotImplementedError, match=match):
            DeepFMTrainer(model, SGD(0.1), 64, device=dev, group=group)
    set_dense_engine("fp32")
    try:
        with pytest.raises(NotImplementedError, match="fp32"):
            DeepFMTrainer(_model(), SGD(0.1), 64, device=dev)
    finally:
        set_dense_engine("auto")
