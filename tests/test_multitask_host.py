"""Multi-output ranking models without a GPU: OutputBlock construction, the default outputs of parse_prediction_blocks and
Keras `compile(loss=..., loss_weights=...)` parsing."""
import pytest

import models_b200 as mm
from models_b200 import datasets
from models_b200.models import ParallelOutputs, parse_prediction_blocks, resolve_loss_weights
from models_b200.schema import ColumnSchema, Schema, Tags


def _schema(*targets):
    cols = [ColumnSchema("C1", tags=(Tags.CATEGORICAL,), dtype="int64", properties={"domain": {"min": 0, "max": 9}}),
            ColumnSchema("I1", tags=(Tags.CONTINUOUS,), dtype="float32")]
    for name, kind in targets:
        if kind == "bin":
            cols.append(ColumnSchema(name, tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"))
        elif kind == "reg":
            cols.append(ColumnSchema(name, tags=(Tags.TARGET, Tags.REGRESSION), dtype="float32"))
        else:
            cols.append(ColumnSchema(name, tags=(Tags.TARGET, Tags.CATEGORICAL), dtype="int64",
                                     properties={"domain": {"min": 0, "max": kind}}))
    return Schema(cols)


def test_output_block_single_target_is_the_output_itself():
    assert type(mm.OutputBlock(_schema(("click", "bin")))) is mm.BinaryOutput
    out = mm.OutputBlock(_schema(("rating", "reg")))
    assert type(out) is mm.RegressionOutput and out.name == "rating/regression_output"
    assert out.to_call.activation == "linear" and out.loss == "mse"


def test_output_block_several_targets_names_and_order():
    out = mm.OutputBlock(_schema(("rating", "reg"), ("click", "bin"), ("conversion", "bin")))
    assert isinstance(out, ParallelOutputs)
    assert out.names == ["click/binary_output", "conversion/binary_output", "rating/regression_output"]
    assert out.losses == ["binary_crossentropy", "binary_crossentropy", "mse"]
    assert out.activations == ["sigmoid", "sigmoid", "linear"]
    assert out.to_call.units == 3


def test_output_block_categorical_targets():
    # a categorical target with int_domain.max == 1 is binary; more classes are not implemented
    out = mm.OutputBlock(_schema(("click", 1), ("rating", "reg")))
    assert out.names == ["click/binary_output", "rating/regression_output"]
    with pytest.raises(NotImplementedError, match="CategoricalOutput"):
        mm.OutputBlock(_schema(("genre", 17), ("rating", "reg")))
    with pytest.raises(ValueError, match="No targets"):
        mm.OutputBlock(_schema())


def test_output_block_model_outputs_replace_defaults():
    mine = mm.BinaryOutput("click")
    out = mm.OutputBlock(_schema(("click", "bin"), ("rating", "reg")), model_outputs=[mine])
    assert out.outputs[0] is mine


def test_parse_prediction_blocks_defaults():
    # unchanged: exactly one binary target among several keeps that one BinaryOutput
    p = parse_prediction_blocks(datasets.movielens_1m_schema())
    assert type(p) is mm.BinaryOutput and p.target == "rating_binary"
    assert type(parse_prediction_blocks(_schema(("click", "bin")))) is mm.BinaryOutput
    # several binary targets, or several targets none of them binary: OutputBlock(schema)
    p = parse_prediction_blocks(_schema(("click", "bin"), ("conversion", "bin"), ("rating", "reg")))
    assert p.names == ["click/binary_output", "conversion/binary_output", "rating/regression_output"]
    p = parse_prediction_blocks(_schema(("rating", "reg"), ("watch_time", "reg")))
    assert p.names == ["rating/regression_output", "watch_time/regression_output"]
    # a list of several outputs or v1 tasks
    p = parse_prediction_blocks(None, [mm.BinaryClassificationTask("click"), mm.RegressionOutput("rating")])
    assert isinstance(p, ParallelOutputs) and len(p.outputs) == 2
    one = mm.RegressionOutput("rating")
    assert parse_prediction_blocks(None, [one]) is one


def test_multi_output_deepfm_is_rejected():
    s = _schema(("click", "bin"), ("conversion", "bin"))
    with pytest.raises(NotImplementedError, match="several outputs"):
        mm.DeepFMModel(s, embedding_dim=8)


def test_loss_and_loss_weights_parsing():
    outs = mm.OutputBlock(_schema(("click", "bin"), ("rating", "reg"))).outputs
    assert resolve_loss_weights(outs) == [1.0, 1.0]
    assert resolve_loss_weights(outs, {"click/binary_output": "binary_crossentropy", "rating/regression_output": "mean_squared_error"},
                                [0.5, 2.0]) == [0.5, 2.0]
    assert resolve_loss_weights(outs, None, {"rating/regression_output": 3.0}) == [1.0, 3.0]
    with pytest.raises(NotImplementedError, match="mse"):
        resolve_loss_weights(outs, "mse")  # not valid for the binary output
    with pytest.raises(NotImplementedError):
        resolve_loss_weights(outs, "hinge")
    with pytest.raises(ValueError, match="unknown outputs"):
        resolve_loss_weights(outs, {"nope": "mse"})
    with pytest.raises(ValueError, match="unknown outputs"):
        resolve_loss_weights(outs, None, {"nope": 1.0})
    with pytest.raises(ValueError, match="2 outputs"):
        resolve_loss_weights(outs, None, [1.0])
    assert resolve_loss_weights([mm.RegressionOutput("r")], "mse") == [1.0]
    with pytest.raises(NotImplementedError):
        resolve_loss_weights([mm.BinaryOutput("c")], "mse")


# ---------------------------------------------------------------------------------------------------------------
# the restated multi-output step (tests/multitask_oracle.py)
# ---------------------------------------------------------------------------------------------------------------
GOLDEN = __import__("pathlib").Path(__file__).parent / "golden" / "multitask" / "ref_torch_dlrm_train_multitask.npz"


def test_one_binary_output_restatement_is_bit_identical_to_oracle_train():
    import numpy as np

    from oracle import oracle_train
    from tests import multitask_oracle as MT

    rng = np.random.default_rng(3)
    B = 11
    batch = {"a": rng.integers(0, 7, B), "b": rng.integers(0, 5, B), "I1": rng.random(B), "I2": rng.random(B)}
    tables = {"a": rng.standard_normal((7, 4)), "b": rng.standard_normal((5, 4))}
    bottom = [{"kernel": rng.standard_normal((2, 4)), "bias": rng.standard_normal(4), "activation": "relu"}]
    top = [{"kernel": rng.standard_normal((4 + 3, 3)), "bias": rng.standard_normal(3), "activation": "relu"}]
    head = {"kernel": rng.standard_normal((3, 1)), "bias": rng.standard_normal(1)}
    y = (rng.random(B) < 0.5).astype(np.float64)
    sw = rng.random(B)
    f2t = {"a": "a", "b": "b"}
    for w in (None, sw):
        want = oracle_train.dlrm_loss_and_grads(batch, tables, f2t, ["I1", "I2"], bottom, top, head, y, sample_weight=w)
        got = MT.dlrm_multitask_loss_and_grads(batch, tables, f2t, ["I1", "I2"], bottom, top,
                                               [dict(head, name="click/binary_output", loss=MT.BCE)], [y], sample_weight=w)
        assert got[0] == want[0] and got[1] == [want[0]]
        np.testing.assert_array_equal(got[2][0], want[1])
        for k, v in want[2].items():
            key = k.replace("head/", "head/click/binary_output/") if k.startswith("head/") else k
            np.testing.assert_array_equal(got[3][key], v)


def test_restatement_matches_the_reference_torch_backend_multitask():
    """Loss, per-output predictions and every gradient of one step of the reference's torch DLRMModel with its default
    output block over click / conversion (binary) and rating (regression) targets (tests/golden/make_golden_multitask.py),
    at 2e-4.  The torch backend's compute_loss AVERAGES the per-output losses; the Keras semantics restated here SUM them
    weighted by loss_weights, so the fixture is reproduced with loss_weights = 1/H for every output."""
    import numpy as np

    from tests import multitask_oracle as MT
    from tests.golden import replay

    z = replay.load(GOLDEN)
    batch, tables, f2t, cont, bottom, top, heads, ys = MT.golden_inputs(z)
    H_ = len(heads)
    assert H_ == 3 and [h["loss"] for h in heads] == [MT.BCE, MT.BCE, MT.MSE]
    loss, per, logits, grads = MT.dlrm_multitask_loss_and_grads(batch, tables, f2t, cont, bottom, top, heads, ys,
                                                                loss_weights=[1.0 / H_] * H_)
    np.testing.assert_allclose(loss, float(z["loss"]), rtol=2e-4)
    for hd, lg in zip(heads, logits):
        t = hd["target"]
        pred = 1.0 / (1.0 + np.exp(-lg)) if hd["loss"] == MT.BCE else lg
        np.testing.assert_allclose(pred, z[f"out_{t}"].reshape(-1), rtol=2e-4, atol=1e-6, err_msg=t)
        np.testing.assert_allclose(grads[f"head/{hd['name']}/kernel"], z[f"grad_head_{t}_kernel"], rtol=2e-4, atol=1e-7, err_msg=t)
        np.testing.assert_allclose(grads[f"head/{hd['name']}/bias"], z[f"grad_head_{t}_bias"], rtol=2e-4, atol=1e-7, err_msg=t)
    for tag in ("bottom", "top"):
        for i in range(len(bottom if tag == "bottom" else top)):
            for what in ("kernel", "bias"):
                np.testing.assert_allclose(grads[f"{tag}/{what}_{i}"], z[f"grad_{tag}_{what}_{i}"], rtol=2e-4, atol=1e-7,
                                           err_msg=f"{tag} {what} {i}")
    for n in z["cat_names"]:
        np.testing.assert_allclose(grads[f"table/{n}"], z[f"grad_table_{n}"], rtol=2e-4, atol=1e-7, err_msg=str(n))
    assert np.abs(z["targets_rating"]).max() > 30  # regression targets far from the prediction


def test_output_block_matches_given_outputs_by_target():
    mine = mm.BinaryOutput("click", name="ctr_head")
    out = mm.OutputBlock(_schema(("click", "bin"), ("rating", "reg")), model_outputs=[mine])
    assert len(out.outputs) == 2 and mine in out.outputs
    assert out.names == ["ctr_head", "rating/regression_output"]


def test_parallel_outputs_weights_before_build_and_width_limit():
    out = mm.OutputBlock(_schema(("click", "bin"), ("rating", "reg")))
    assert out.weights() == {}
    with pytest.raises(NotImplementedError, match="at most 256"):
        out.build(300)


def test_nine_outputs_are_refused():
    with pytest.raises(NotImplementedError, match=r"2\.\.8 outputs are supported, got 9"):
        mm.OutputBlock(_schema(*[(f"t{i}", "bin" if i % 2 else "reg") for i in range(9)]))


def test_heads_kernel_cases_reach_every_instantiation():
    """tests/test_gpu_heads_kernels.py's CASES reach all 96 kernels mm_heads_fwd_bwd is compiled for: H = 1..8 heads x
    {scalar, G2, G4, G8, G16, G32} x {training, forward only}, by heads_variant, the restatement of run_heads /
    launch_heads (train_dense.cu).  Prints the H x variant table (T: training, F: forward only)."""
    from tests.test_gpu_heads_kernels import CASES, VARIANTS, case_variants, heads_variant

    # the restatement itself, on the deciding inputs: K, the row strides, 16-byte alignment of x / dx and of w for H = 1
    assert [heads_variant(2, k, k, 0, 0) for k in (4, 8, 12, 16, 20, 32, 36, 64, 68, 128)] == \
        ["G2", "G2", "G4", "G4", "G8", "G8", "G16", "G16", "G32", "G32"]
    assert {heads_variant(2, k, k, 0, 0) for k in (1, 7, 130, 132, 256)} == {"scalar"}
    assert heads_variant(1, 32, 32, 0, 4) == "scalar" and heads_variant(2, 32, 32, 0, 4) == "G8"
    assert heads_variant(2, 32, 33, 0, 0) == "scalar" and heads_variant(2, 32, 40, 4, 0) == "scalar"
    assert heads_variant(2, 32, 40, 16, 0, 36, 16) == "G8" and heads_variant(2, 32, 40, 16, 0, 34, 16) == "scalar"
    assert heads_variant(2, 32, 40, 16, 0, 36, 20) == "scalar"
    seen = {}
    for c in CASES:
        train, fwd = case_variants(c)
        seen.setdefault((c[0], train), set()).add("T")
        seen.setdefault((c[0], fwd), set()).add("F")
    rows = ["H  " + "".join(f"{v:>8}" for v in VARIANTS)]
    rows += [f"{h:<3}" + "".join(f"{''.join(sorted(seen.get((h, v), ()), reverse=True)):>8}" for v in VARIANTS) for h in range(1, 9)]
    print("\n".join(rows))
    triples = {(h, v, t) for (h, v), ts in seen.items() for t in ts}
    assert triples == {(h, v, t) for h in range(1, 9) for v in VARIANTS for t in "TF"}, "missing: " + str(
        sorted({(h, v, t) for h in range(1, 9) for v in VARIANTS for t in "TF"} - triples))
