"""The multi-task Model(InputBlockV2, [MLPBlock], [MMOEBlock], output) without a GPU: constructor semantics and refusals,
the sorted-name expert order, independent expert and gate copies, weight names, and the restatement's gate backward
against central finite differences."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200.models import MMoEBody, ParallelOutputs, RankingModel
from models_b200.schema import ColumnSchema, Schema, Tags
from tests.mmoe_oracle import BCE, MSE, gate_mix, heads_loss


def schema(lists=(), targets=(("click", "bin"), ("conversion", "bin"), ("rating", "reg")), rows=(50, 300, 7, 1200)):
    """C0.. categorical columns (inferred widths), three continuous columns, optional list columns (name, rows, ragged)
    and the targets."""
    cols = [ColumnSchema(f"C{i}", tags=(Tags.CATEGORICAL,), dtype="int64", properties={"domain": {"min": 0, "max": r}})
            for i, r in enumerate(rows)]
    cols += [ColumnSchema(f"I{i}", tags=(Tags.CONTINUOUS,), dtype="float32") for i in range(3)]
    for name, r, ragged in lists:
        cols.append(ColumnSchema(name, tags=(Tags.CATEGORICAL,), dtype="int64", is_list=True, is_ragged=ragged,
                                 properties={"domain": {"min": 0, "max": r}, **({} if ragged else {"value_count": {"min": 3, "max": 3}})}))
    for name, kind in targets:
        tags = (Tags.TARGET, Tags.BINARY_CLASSIFICATION) if kind == "bin" else (Tags.TARGET, Tags.REGRESSION)
        cols.append(ColumnSchema(name, tags=tags, dtype="int64" if kind == "bin" else "float32"))
    return Schema(cols)


def mmoe_model(s=None, E=4, U=16, bottom=None, T=1.0, outputs=None, towers=None, gate=None):
    s = s or schema()
    out = outputs or mm.OutputBlock(s, task_blocks=None if towers is None else mm.MLPBlock(towers))
    blocks = [mm.InputBlockV2(s)]
    if bottom:
        blocks.append(mm.MLPBlock(bottom))
    if E:
        blocks.append(mm.MMOEBlock(out, expert_block=mm.MLPBlock([U]), num_experts=E, gate_softmax_temperature=T,
                                   gate_block=None if gate is None else mm.MLPBlock(gate)))
    return mm.Model(*blocks, out)


def test_sequential_model_is_a_ranking_model():
    s = schema()
    m = mmoe_model(s, bottom=[32])
    assert isinstance(m, RankingModel) and isinstance(m.body, MMoEBody)
    assert m.schema is s and m.body.bottom is not None and m.body.mmoe.num_gates == 3
    assert [o.name for o in m.output_blocks()] == ["click/binary_output", "conversion/binary_output", "rating/regression_output"]
    assert m.body.mmoe.output_names == m.prediction.names
    shared = mm.Model(mm.InputBlockV2(s), mm.MLPBlock([32, 16]), mm.OutputBlock(s))
    assert isinstance(shared, RankingModel) and shared.body.mmoe is None
    # the three-argument form is unchanged
    body = mm.MLPBlock([8])
    old = mm.Model(body, mm.BinaryOutput("click"), s)
    assert type(old) is mm.Model and old.body is body and old.schema is s


def test_mmoe_outputs_given_as_names_and_order_follows_the_output_block():
    s = schema()
    out = mm.OutputBlock(s)
    mo = mm.MMOEBlock(["rating/regression_output", "click/binary_output", "conversion/binary_output"], mm.MLPBlock([8]), 2)
    m = mm.Model(mm.InputBlockV2(s), mo, out)
    assert mo.output_names == out.names
    with pytest.raises(ValueError, match="differ"):
        mm.Model(mm.InputBlockV2(s), mm.MMOEBlock(["click/binary_output"], mm.MLPBlock([8]), 2), out)
    single = mm.BinaryOutput("click")
    m1 = mm.Model(mm.InputBlockV2(s), mm.MMOEBlock(single, mm.MLPBlock([8]), 3), single)
    assert m1.body.mmoe.output_names == [single.name] and m1.output_blocks() == [single]
    assert isinstance(m.prediction, ParallelOutputs)


def test_refusals():
    s = schema()
    out = mm.OutputBlock(s)
    ib = mm.InputBlockV2(s)
    with pytest.raises(NotImplementedError, match="CGCBlock"):
        mm.CGCBlock(out, mm.MLPBlock([8]), 2)
    with pytest.raises(NotImplementedError, match="PLEBlock"):
        mm.PLEBlock(out, mm.MLPBlock([8]), 2)
    with pytest.raises(NotImplementedError, match="gate-weight metrics"):
        mm.MMOEBlock(out, mm.MLPBlock([8]), 2, enable_gate_weights_metrics=True)
    with pytest.raises(NotImplementedError, match="gate_block"):
        mm.MMOEBlock(out, mm.MLPBlock([8]), 2, gate_block=mm.MLPBlock([4], normalization="batch_norm"))
    with pytest.raises(NotImplementedError, match="one Dense layer"):
        mm.MMOEBlock(out, mm.MLPBlock([8, 4]), 2)
    with pytest.raises(NotImplementedError, match="1..16 experts"):
        mm.MMOEBlock(out, mm.MLPBlock([8]), 17)
    with pytest.raises(NotImplementedError, match="at most 256 units"):
        mm.MMOEBlock(out, mm.MLPBlock([257]), 2)
    with pytest.raises(ValueError, match="temperature"):
        mm.MMOEBlock(out, mm.MLPBlock([8]), 2, gate_softmax_temperature=0.0)
    with pytest.raises(NotImplementedError, match="same width"):
        mm.OutputBlock(s, task_blocks={"click": mm.MLPBlock([8]), "conversion": mm.MLPBlock([8]), "rating": mm.MLPBlock([4])})
    with pytest.raises(NotImplementedError, match="every output"):
        mm.OutputBlock(s, task_blocks={"click": mm.MLPBlock([8])})
    with pytest.raises(ValueError, match="unknown"):
        mm.OutputBlock(s, task_blocks={"clicks": mm.MLPBlock([8])})
    towered = mm.OutputBlock(s, task_blocks=mm.MLPBlock([8]))
    for factory in (lambda: mm.DLRMModel(s, embedding_dim=16, bottom_block=mm.MLPBlock([16]), top_block=mm.MLPBlock([8]),
                                         prediction_tasks=towered),
                    lambda: mm.DCNModel(s, depth=1, deep_block=mm.MLPBlock([8]), prediction_tasks=towered),
                    lambda: mm.DeepFMModel(s, embedding_dim=8, prediction_tasks=towered),
                    lambda: mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]), prediction_tasks=towered)):
        with pytest.raises(NotImplementedError, match="per-task towers"):
            factory()
    with pytest.raises(TypeError):  # the three-argument form keeps its signature
        mm.Model(mm.MLPBlock([8]), out)
    mo = mm.MMOEBlock(out, mm.MLPBlock([8]), 2)
    with pytest.raises(NotImplementedError, match="optionally one MMOEBlock"):  # MMoE before the bottom
        mm.Model(ib, mo, mm.MLPBlock([8]), out)
    with pytest.raises(NotImplementedError, match="optionally one MMOEBlock"):  # two bottoms
        mm.Model(ib, mm.MLPBlock([8]), mm.MLPBlock([8]), out)
    with pytest.raises(NotImplementedError, match="output"):
        mm.Model(ib, mm.MLPBlock([8]), mo)
    with pytest.raises(NotImplementedError, match="are needed"):
        mm.Model(ib, out)
    with pytest.raises(NotImplementedError, match="concatenate"):
        mm.Model(mm.InputBlockV2(s, aggregation=None), mm.MLPBlock([8]), out)
    with pytest.raises(NotImplementedError, match="MMOEBlock runs inside"):
        mo({"x": None})


def test_sorted_name_expert_order_at_12_experts():
    mo = mm.MMOEBlock(["a"], mm.MLPBlock([4]), 12)
    assert mo.expert_names == ["expert_0", "expert_1", "expert_10", "expert_11"] + [f"expert_{i}" for i in range(2, 10)]
    mo.build(5, "cpu")
    U = 4
    w = mo.weights()
    # stacked column block e is the expert with the e-th sorted name
    for e, n in enumerate(mo.expert_names):
        k = [v for key, v in w.items() if key.startswith(f"{n}/") and key.endswith("/kernel")]
        assert len(k) == 1 and k[0].data_ptr() == mo.experts.kernel[:, e * U:(e + 1) * U].data_ptr()


def test_independent_copies_and_weight_names():
    s = schema()
    m = mmoe_model(s, E=3, U=8, bottom=[16])
    m.body.build("cpu")
    mo = m.body.mmoe
    w = m.body.weights()
    names = sorted(k for k in w if k.startswith("mmoe/"))
    expert_keys = [k for k in names if k.startswith("mmoe/expert_")]
    assert len(expert_keys) == 6 and {k.split("/")[1] for k in expert_keys} == {"expert_0", "expert_1", "expert_2"}
    assert all(k.split("/")[-1] in ("kernel", "bias") for k in expert_keys)
    gate_keys = [k for k in names if k.startswith("mmoe/gate_")]
    assert gate_keys == sorted(f"mmoe/gate_{n}/gate_final/kernel" for n in m.prediction.names)
    # every expert and gate kernel is its own initialisation: no two are equal, no tensor is shared between blocks
    ks = [w[k] for k in names if k.endswith("kernel")]
    for i in range(len(ks)):
        for j in range(i + 1, len(ks)):
            assert not torch.equal(ks[i], ks[j])
    assert len({id(b) for b in mo.expert_blocks.values()}) == 3
    layers = [b.dense_layers[0] for b in mo.expert_blocks.values()]
    assert len({l.name for l in layers}) == 3
    # glorot-uniform limits of each expert's own (K, U) kernel and each gate's own (K, E) kernel
    K = 16
    assert float(mo.experts.kernel.abs().max()) <= np.sqrt(6.0 / (K + 8)) + 1e-6
    assert float(mo.gates.kernel.abs().max()) <= np.sqrt(6.0 / (K + 3)) + 1e-6
    assert mo.gates.bias is None


def test_gate_backward_of_the_restatement_against_finite_differences():
    g = torch.Generator().manual_seed(3)
    B, E, U, T = 5, 3, 4, 0.7
    X = torch.randn((B, E * U), generator=g, dtype=torch.float64)
    L = torch.randn((B, E), generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn((U,), generator=g, dtype=torch.float64)
    y = np.array([0, 1, 1, 0, 1])

    def f(L_):
        z = gate_mix(X, L_, E, T) @ w
        return heads_loss([z], [BCE], [y])[0]

    f(L).backward()
    num = torch.zeros_like(L)
    eps = 1e-6
    for i in range(B):
        for e in range(E):
            Lp, Lm = L.detach().clone(), L.detach().clone()
            Lp[i, e] += eps
            Lm[i, e] -= eps
            num[i, e] = (f(Lp) - f(Lm)) / (2 * eps)
    assert torch.allclose(L.grad, num, rtol=1e-6, atol=1e-9)
    # and the closed form the kernel evaluates: dL = p (dg - <p, dg>) / T with dg_e = dz <w, X_e>
    with torch.no_grad():
        p = torch.softmax(L / T, dim=1)
        z = gate_mix(X, L, E, T) @ w
        dz = (torch.sigmoid(z) - torch.as_tensor(y, dtype=torch.float64)) / B
        dg = dz.unsqueeze(1) * (X.reshape(B, E, U) @ w)
        closed = p * (dg - (p * dg).sum(1, keepdim=True)) / T
    assert torch.allclose(closed, num, rtol=1e-6, atol=1e-9)
    assert MSE == "mse"


def test_task_blocks_as_a_layer_and_as_dicts_by_name_and_by_column():
    s = schema()
    tower = mm.MLPBlock([8])
    out = mm.OutputBlock(s, task_blocks=tower)
    tw = out.task_blocks
    assert sorted(tw) == out.names and len({id(t) for t in tw.values()}) == 3 and tower not in tw.values()
    by_name = {n: mm.MLPBlock([8]) for n in out.names}
    assert mm.OutputBlock(s, task_blocks=by_name).task_blocks == by_name
    by_col = {"click": mm.MLPBlock([8]), "conversion": mm.MLPBlock([8]), "rating": mm.MLPBlock([8])}
    o2 = mm.OutputBlock(s, task_blocks=by_col)
    assert o2.task_blocks["rating/regression_output"] is by_col["rating"]
    m = mm.Model(mm.InputBlockV2(s), mm.MMOEBlock(o2, mm.MLPBlock([16]), 2, gate_block=mm.MLPBlock([4])), o2)
    m.build("cpu")
    w = m.weights()
    for n in o2.names:
        assert f"prediction/{n}/dense/kernel" in w and any(k.startswith(f"prediction/{n}/task_block/") for k in w)
        assert any(k.startswith(f"body/mmoe/gate_{n}/gate_block/") for k in w)
        assert w[f"body/mmoe/gate_{n}/gate_final/kernel"].shape == (4, 2)
    assert w[f"prediction/{o2.names[0]}/dense/kernel"].shape == (8, 1)
    # towers on the shared bottom, without an MMOEBlock
    o3 = mm.OutputBlock(s, task_blocks=mm.MLPBlock([8]))
    shared = mm.Model(mm.InputBlockV2(s), mm.MLPBlock([16]), o3)
    assert shared.body.mmoe is None and shared.prediction.task_blocks


def test_kernel_cases_reach_every_instantiation():
    """tests/test_gpu_mmoe_kernels.py's CASES reach every (tasks rounded up to a power of two, columns per lane) pair the
    MMoE mixture and task-head kernels are compiled for."""
    from tests.test_gpu_mmoe_kernels import CASES, _dispatch

    assert sorted({_dispatch(c[0], c[1]) for c in CASES}) == [(nh, c) for nh in (1, 2, 4, 8) for c in (1, 2, 4, 8)]
