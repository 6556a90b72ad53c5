"""Learning-rate schedules and per-block optimizers without a GPU: each schedule's float64 evaluation against an
independent restatement of the Keras formulas, argument checks, config round trips, the K25 device array, and how a
MultiOptimizer resolves a model's variables to its optimizers."""
import math
import warnings

import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import _cabi, ops, train
from models_b200.optimizer import block_variables
from models_b200.schedules import (CosineDecay, ExponentialDecay, InverseTimeDecay, LearningRateSchedule,
                                   PiecewiseConstantDecay, PolynomialDecay, deserialize, serialize)
from tests.test_mmoe_host import mmoe_model, schema


# ---- an independent restatement of tf.keras.optimizers.schedules (TF 2.9-2.12) -------------------------------------
def keras_lr(kind: str, cfg: dict, s: int) -> float:
    s = np.float64(s)
    if kind == "ExponentialDecay":
        p = s / cfg["decay_steps"]
        p = np.floor(p) if cfg.get("staircase") else p
        return cfg["initial_learning_rate"] * np.power(cfg["decay_rate"], p)
    if kind == "InverseTimeDecay":
        p = s / cfg["decay_steps"]
        p = np.floor(p) if cfg.get("staircase") else p
        return cfg["initial_learning_rate"] / (1 + cfg["decay_rate"] * p)
    if kind == "PiecewiseConstantDecay":
        b, v = cfg["boundaries"], cfg["values"]
        if s <= b[0]:
            return v[0]
        for i in range(1, len(b)):
            if b[i - 1] < s <= b[i]:
                return v[i]
        return v[-1]
    if kind == "PolynomialDecay":
        ds, end = cfg["decay_steps"], cfg.get("end_learning_rate", 1e-4)
        if cfg.get("cycle"):
            D = ds * (1.0 if s == 0 else np.ceil(s / ds))
            sp = s
        else:
            D, sp = ds, min(s, ds)
        return (cfg["initial_learning_rate"] - end) * (1 - sp / D) ** cfg.get("power", 1.0) + end
    if kind == "CosineDecay":
        ds, a = cfg["decay_steps"], cfg.get("alpha", 0.0)
        return cfg["initial_learning_rate"] * ((1 - a) * 0.5 * (1 + np.cos(np.pi * min(s, ds) / ds)) + a)
    raise AssertionError(kind)


CASES = [
    ("ExponentialDecay", dict(initial_learning_rate=0.1, decay_steps=10, decay_rate=0.96)),
    ("ExponentialDecay", dict(initial_learning_rate=0.1, decay_steps=10, decay_rate=0.5, staircase=True)),
    ("InverseTimeDecay", dict(initial_learning_rate=0.2, decay_steps=7, decay_rate=0.5)),
    ("InverseTimeDecay", dict(initial_learning_rate=0.2, decay_steps=7, decay_rate=0.5, staircase=True)),
    ("PiecewiseConstantDecay", dict(boundaries=[5, 12, 30], values=[1.0, 0.5, 0.1, 0.01])),
    ("PolynomialDecay", dict(initial_learning_rate=0.1, decay_steps=10)),
    ("PolynomialDecay", dict(initial_learning_rate=0.1, decay_steps=10, end_learning_rate=0.01, power=2.0)),
    ("PolynomialDecay", dict(initial_learning_rate=0.1, decay_steps=10, end_learning_rate=0.01, power=0.5, cycle=True)),
    ("CosineDecay", dict(initial_learning_rate=0.1, decay_steps=10)),
    ("CosineDecay", dict(initial_learning_rate=0.1, decay_steps=10, alpha=0.2)),
]


def _make(kind, cfg):
    return getattr(mm.schedules, kind)(**cfg)


def _steps(kind, cfg):
    if kind == "PiecewiseConstantDecay":
        return sorted({0} | {b + d for b in cfg["boundaries"] for d in (-1, 0, 1)} | {100})
    ds = cfg["decay_steps"]
    # 0, decay_steps +- 1, and two more periods (cycle, the clamp of cosine and polynomial decay)
    return [0, 1, ds - 1, ds, ds + 1, 2 * ds - 1, 2 * ds, 2 * ds + 1, 3 * ds, 5 * ds + 3]


@pytest.mark.parametrize("kind,cfg", CASES, ids=[f"{k}-{i}" for i, (k, _) in enumerate(CASES)])
def test_schedule_matches_the_keras_formula(kind, cfg):
    sch = _make(kind, cfg)
    for s in _steps(kind, cfg):
        assert sch(s) == pytest.approx(keras_lr(kind, cfg, s), rel=1e-15, abs=0), (kind, s)


def test_clamps_and_cycles():
    assert CosineDecay(0.1, 10, alpha=0.2)(10) == pytest.approx(0.02) and CosineDecay(0.1, 10, alpha=0.2)(50) == pytest.approx(0.02)
    p = PolynomialDecay(0.1, 10, end_learning_rate=0.01)
    assert p(10) == pytest.approx(0.01) and p(25) == pytest.approx(0.01)
    c = PolynomialDecay(0.1, 10, end_learning_rate=0.0, cycle=True)
    assert c(0) == pytest.approx(0.1) and c(10) == pytest.approx(0.0) and c(11) == pytest.approx(0.1 * 9 / 20)
    assert c(20) == pytest.approx(0.0) and c(21) == pytest.approx(0.1 * 9 / 30)
    e = ExponentialDecay(1.0, 2, 0.5, staircase=True)
    assert [e(s) for s in range(5)] == [1.0, 1.0, 0.5, 0.5, 0.25]


def test_argument_validation():
    with pytest.raises(ValueError, match="1 less than the length of values"):
        PiecewiseConstantDecay([1, 2], [1.0, 2.0])
    with pytest.raises(ValueError, match="increasing"):
        PiecewiseConstantDecay([5, 2], [1.0, 2.0, 3.0])
    n = _cabi.SCHED_MAX_BOUNDARIES
    PiecewiseConstantDecay(list(range(1, n + 1)), [0.1] * (n + 1))
    with pytest.raises(NotImplementedError, match=f"1..{n}"):
        PiecewiseConstantDecay(list(range(1, n + 2)), [0.1] * (n + 2))
    for cls, kw in ((ExponentialDecay, dict(decay_rate=0.5)), (InverseTimeDecay, dict(decay_rate=0.5)),
                    (PolynomialDecay, {}), (CosineDecay, {})):
        with pytest.raises(ValueError, match="decay_steps"):
            cls(0.1, 0, **kw)


@pytest.mark.parametrize("kind,cfg", CASES, ids=[f"{k}-{i}" for i, (k, _) in enumerate(CASES)])
def test_config_round_trip(kind, cfg):
    sch = _make(kind, cfg)
    c = sch.get_config()
    assert {k: c[k] for k in cfg} == cfg and "name" in c
    assert type(sch).from_config(c) == sch
    ser = serialize(sch)
    assert ser == {"class_name": kind, "config": c}
    assert deserialize(ser) == sch
    for opt in (mm.SGD(sch), mm.Adagrad(sch), mm.Adam(sch), mm.LazyAdam(sch)):
        assert opt.learning_rate is sch and opt.schedule is sch
        oc = opt.get_config()
        assert oc["learning_rate"] == ser and deserialize(oc["learning_rate"]) == sch
        h = opt.hyper()
        assert h.shape == (_cabi.HYPER_COUNT,) and h[_cabi.HYPER_LR] == np.float32(sch(0)) and h[_cabi.HYPER_STEP] == 0


def test_device_array_layout():
    a = ExponentialDecay(0.1, 100000, 0.96, staircase=True).device_params()
    assert a.shape == (_cabi.SCHED_COUNT,) and a.dtype == np.float32
    assert a[_cabi.SCHED_KIND] == _cabi.SCHED_KINDS["ExponentialDecay"]
    assert (a[_cabi.SCHED_INIT], a[_cabi.SCHED_DECAY_STEPS], a[_cabi.SCHED_RATE], a[_cabi.SCHED_FLAG]) == (
        np.float32(0.1), 100000, np.float32(0.96), 1)
    p = PiecewiseConstantDecay([3, 9], [0.3, 0.2, 0.1]).device_params()
    assert p[_cabi.SCHED_NB] == 2 and list(p[_cabi.SCHED_BOUNDARIES:_cabi.SCHED_BOUNDARIES + 2]) == [3, 9]
    assert np.allclose(p[_cabi.SCHED_VALUES:_cabi.SCHED_VALUES + 3], [0.3, 0.2, 0.1])
    with pytest.raises(ValueError, match="unknown learning-rate schedule"):
        ops.schedule_params("WarmUp")
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.opt_tick_schedule(torch.zeros(_cabi.HYPER_COUNT), torch.zeros(_cabi.SCHED_COUNT))


def test_float_learning_rate_unchanged_and_other_callables_refused():
    assert mm.Adam(0.5).learning_rate == 0.5 and mm.Adam(0.5).schedule is None
    assert mm.Adam(0.5).get_config()["learning_rate"] == 0.5

    class Custom(LearningRateSchedule):
        def __call__(self, step):
            return 0.1

    class MyDecay(ExponentialDecay):
        pass

    for lr in (lambda s: 0.1, Custom(), MyDecay(0.1, 10, 0.5)):
        with pytest.raises(NotImplementedError, match="built-in schedules"):
            mm.Adam(lr)


# ---- MultiOptimizer ------------------------------------------------------------------------------------------------
def _model():
    s = schema()
    m = mmoe_model(s, bottom=[32])
    return s, m


def _resolved(multi, model):
    g = train._OptGroups(multi, model, torch.device("cpu"))
    return g


def test_multi_optimizer_resolution():
    s, m = _model()
    emb = m.body.input_block.embeddings
    large, small = mm.split_embeddings_on_size(emb, 100)
    assert {t.table_name for t in large} == {"C1", "C3"} and {t.table_name for t in small} == {"C0", "C2"}
    ada, sgd = mm.Adagrad(0.05), mm.SGD(0.1)
    multi = mm.MultiOptimizer([mm.OptimizerBlocks(ada, large), mm.OptimizerBlocks(sgd, m.body.bottom)],
                              default_optimizer="adam")
    g = _resolved(multi, m)
    for t in large:
        assert g.of(t).opt is ada
    for l in m.body.bottom.dense_layers:
        assert g.of(l).opt is sgd
    rest = [g.of(t).opt for t in small] + [g.of(m.body.mmoe.experts).opt, g.of(m.prediction.to_call).opt]
    assert all(o is multi.default_optimizer for o in rest) and multi.default_optimizer.kind == "adam"
    assert len(g.groups) == 3
    # add(): another disjoint entry
    adam2 = mm.Adam(0.01)
    multi.add(mm.OptimizerBlocks(adam2, small[0]))
    assert _resolved(multi, m).of(small[0]).opt is adam2
    # update(): overrides without the disjointness check
    multi.update(mm.OptimizerBlocks("sgd", large[0]))
    g = _resolved(multi, m)
    assert g.of(large[0]).kind == "sgd" and g.of(large[1]).opt is ada
    cfg = multi.get_config()
    assert set(cfg) == {"default_optimizer", "name", "optimizers_and_blocks", "update_optimizers_and_blocks"}
    assert cfg["name"] == "MultiOptimizer" and len(cfg["optimizers_and_blocks"]) == 3
    assert len(cfg["update_optimizers_and_blocks"]) == 1
    oc, blocks = cfg["optimizers_and_blocks"][0]
    assert oc["class_name"] == "Adagrad" and oc["config"]["learning_rate"] == 0.05
    assert [b["config"]["name"] for b in blocks] == [t.name for t in large]


def test_multi_optimizer_refusals():
    s, m = _model()
    emb = m.body.input_block.embeddings
    with pytest.raises(ValueError, match="can't be empty"):
        mm.MultiOptimizer([])
    with pytest.raises(ValueError, match="Unknown optimizer"):
        mm.MultiOptimizer([mm.OptimizerBlocks("ftrl", emb)])
    with pytest.raises(TypeError):
        train.get_optimizer(3)
    # a variable reachable from two entries: named, with both optimizers
    multi = mm.MultiOptimizer([mm.OptimizerBlocks(mm.Adagrad(0.05), emb), mm.OptimizerBlocks(mm.SGD(0.2), emb.tables["C2"])],
                              default_optimizer="adam")
    with pytest.raises(ValueError, match=r"'C2/embeddings'.*Adagrad\(learning_rate=0.05\).*SGD\(learning_rate=0.2\)"):
        _resolved(multi, m)
    # part of a stacked layer under another optimizer than the rest
    mo = m.body.mmoe
    part = mm.MultiOptimizer([mm.OptimizerBlocks("sgd", mo.expert_blocks["expert_0"])], default_optimizer="adam")
    with pytest.raises(NotImplementedError, match=mo.experts.name):
        _resolved(part, m)
    gate = mm.MultiOptimizer([mm.OptimizerBlocks("sgd", mo.gate_finals["click/binary_output"])], default_optimizer="adam")
    with pytest.raises(NotImplementedError, match=mo.gates.name):
        _resolved(gate, m)
    head = mm.MultiOptimizer([mm.OptimizerBlocks("sgd", m.prediction.outputs[0])], default_optimizer="adam")
    with pytest.raises(NotImplementedError, match=m.prediction.to_call.name):
        _resolved(head, m)
    # every part under one optimizer is the whole layer
    whole = mm.MultiOptimizer([mm.OptimizerBlocks("sgd", list(mo.expert_blocks.values()))], default_optimizer="adam")
    assert _resolved(whole, m).of(mo.experts).kind == "sgd"


def test_rmsprop_default_refused_only_when_used():
    s, m = _model()
    multi = mm.MultiOptimizer([mm.OptimizerBlocks("adagrad", m.body.input_block.embeddings)])
    assert multi.default_optimizer == "rmsprop" and multi.get_config()["default_optimizer"] == "rmsprop"
    g = _resolved(multi, m)
    g.of(m.body.input_block.embeddings.tables["C0"])
    with pytest.raises(NotImplementedError, match="rmsprop"):
        g.of(m.body.bottom.dense_layers[0])
    covering = mm.MultiOptimizer([mm.OptimizerBlocks("adagrad", m)])
    g = _resolved(covering, m)
    assert all(g.of(v).kind == "adagrad" for v in block_variables(m) if getattr(v, "kernel", 0) is not None)
    with pytest.raises(ValueError, match="Unknown optimizer"):
        m.compile(optimizer="rmsprop")
    m.compile(optimizer=covering)
    assert m.optimizer is covering


def test_block_variables_cover_every_family_part():
    s = schema(targets=(("click", "bin"),))
    dcn = mm.DCNModel(s, depth=2, deep_block=mm.MLPBlock([16]), prediction_tasks=mm.BinaryOutput("click"))
    vs = block_variables(dcn)
    assert sum(isinstance(v, mm.EmbeddingTable) for v in vs) == 4
    wd = mm.WideAndDeepModel(s, wide_schema=s.select_by_name(["C0", "C1"]), deep_schema=s.select_by_tag(mm.Tags.CATEGORICAL),
                             deep_block=mm.MLPBlock([8]), prediction_tasks=mm.BinaryOutput("click"))
    assert any(v is wd.body.wide.dense for v in block_variables(wd.body.wide))


def test_split_embeddings_on_size_threshold_and_warning():
    s = schema(rows=(50, 300, 7, 1200))
    emb = mm.InputBlockV2(s).embeddings
    at = mm.split_embeddings_on_size(emb, 301)  # C1 has 301 rows: at the threshold counts as large
    assert [t.table_name for t in at[0]] == ["C1", "C3"]
    above = mm.split_embeddings_on_size(emb, 302)
    assert [t.table_name for t in above[0]] == ["C3"] and len(above[1]) == 3
    below = mm.split_embeddings_on_size(emb, 1)
    assert len(below[0]) == 4 and below[1] == []
    with pytest.warns(UserWarning, match="smaller input dim than threshold 5000"):
        large, small = mm.split_embeddings_on_size(emb, 5000)
    assert large == [] and len(small) == 4
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        mm.split_embeddings_on_size(emb, 100)
    with pytest.raises(TypeError):
        mm.split_embeddings_on_size([], 10)


def test_single_optimizer_arena_is_one_run():
    from models_b200.blocks import _Dense

    layers = [_Dense(8), _Dense(3)]
    w = 5
    for l in layers:
        l.kernel, l.bias, l.input_dim, l.built = torch.randn(w, l.units), torch.randn(l.units), w, True
        w = l.units
    a = train.DenseArena(layers, mm.Adagrad(0.1), torch.device("cpu"))
    assert [(s, e) for s, e, _ in a.runs] == [(0, a.size)]
    sgd, ada = mm.SGD(0.1), mm.Adagrad(0.1, initial_accumulator_value=0.3)
    b = train.DenseArena(layers, [sgd, ada], torch.device("cpu"))
    assert [(s, e, o) for s, e, o in b.runs] == [(0, b.kernel_off[1], sgd), (b.kernel_off[1], b.size, ada)]
    assert float(b.state1[:b.kernel_off[1]].abs().max()) == 0 and float(b.state1[b.kernel_off[1]:].min()) == pytest.approx(0.3)
    assert b.state2 is None
