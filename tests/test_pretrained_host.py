"""PretrainedEmbeddings, EmbeddingOperator and the input block's pretrained slots without a GPU: constructor semantics and
refusals, the sorted-name layout and weight names, the operator's output schema, and the restatement's projection and
l2-norm backward against central finite differences."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200.schema import ColumnSchema, Schema, Tags
from tests import pretrained_oracle as PO


def _schema():
    return Schema([
        ColumnSchema("item", tags=(Tags.CATEGORICAL, Tags.ITEM_ID), dtype="int64", properties={"domain": {"min": 0, "max": 99}}),
        ColumnSchema("user_age", tags=(Tags.CONTINUOUS,)),
        ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"),
    ])


def _with_pretrained(dims=(("pre_b", 12), ("pre_a", 300))):
    cols = list(_schema())
    for name, d in dims:
        op = mm.EmbeddingOperator(np.zeros((100, d), np.float32), lookup_key="item", embedding_name=name, device="cpu")
        cols.append(op.column_schema())
    return Schema(cols)


def test_embedding_operator_output_schema():
    op = mm.EmbeddingOperator(np.ones((7, 5)), lookup_key="item", embedding_name="vecs", device="cpu")
    assert op.embeddings.dtype == torch.float32 and tuple(op.embeddings.shape) == (7, 5)
    out = op.compute_output_schema(_schema())
    col = out["vecs"]
    assert col.has_tag(Tags.EMBEDDING) and col.dtype == "float32"
    assert col.value_count.min == col.value_count.max == 5
    assert out.column_names == ["item", "user_age", "click", "vecs"]
    assert out.select_by_tag(Tags.EMBEDDING).column_names == ["vecs"]
    with pytest.raises(ValueError):
        mm.EmbeddingOperator(np.ones(5), device="cpu")


def test_constructor_output_dims_and_normalizer():
    s = _with_pretrained().select_by_tag(Tags.EMBEDDING)
    pe = mm.PretrainedEmbeddings(s)
    assert pe.output_dims() == {"pre_b": 12, "pre_a": 300}
    assert all(br.projection is None and not br.l2 for br in pe.branches.values())
    pe = mm.PretrainedEmbeddings(s, output_dims=16, normalizer="l2-norm")
    assert pe.output_dims() == {"pre_b": 16, "pre_a": 16}
    assert all(br.l2 and br.projection.activation == "linear" and br.projection.use_bias for br in pe.branches.values())
    pe = mm.PretrainedEmbeddings(s, output_dims={"pre_a": 64})
    assert pe.output_dims() == {"pre_b": 12, "pre_a": 64}
    assert pe.branches["pre_b"].projection is None
    assert pe.branches["pre_a"].lookup_key == "item"


@pytest.mark.parametrize("kwargs,match", [
    (dict(pre=object()), "pre"),
    (dict(post=object()), "post"),
    (dict(aggregation="concat"), "aggregation"),
    (dict(normalizer="batch_norm"), "normalizer"),
    (dict(id_lookup_table=object()), "id_lookup_table"),
    (dict(output_dims=257), "output_dims"),
])
def test_refusals(kwargs, match):
    with pytest.raises(NotImplementedError, match=match):
        mm.PretrainedEmbeddings(_with_pretrained().select_by_tag(Tags.EMBEDDING), **kwargs)


def test_refuses_sequence_and_too_wide_inputs():
    seq = Schema([ColumnSchema("s", tags=(Tags.EMBEDDING,), is_list=True, is_ragged=True)])
    with pytest.raises(NotImplementedError, match="sequence"):
        mm.PretrainedEmbeddings(seq)
    wide = Schema([ColumnSchema("w", tags=(Tags.EMBEDDING,), is_list=True, properties={"value_count": {"min": 1025, "max": 1025}})])
    with pytest.raises(NotImplementedError, match="1024"):
        mm.PretrainedEmbeddings(wide)


def test_input_block_layout_and_weight_names():
    s = _with_pretrained()
    pe = mm.PretrainedEmbeddings(s.select_by_tag(Tags.EMBEDDING), output_dims={"pre_a": 64}, normalizer="l2-norm")
    ib = mm.InputBlockV2(s, pretrained_embeddings=pe)
    cols, widths, total = ib.layout()
    assert list(cols) == sorted(widths) == ["item", "pre_a", "pre_b", "user_age"]
    assert widths["pre_a"] == 64 and widths["pre_b"] == 12 and total == widths["item"] + 64 + 12 + 1
    ib.build(torch.device("cpu"))
    names = sorted(ib.weights())
    dense = pe.branches["pre_a"].projection.name
    assert names == sorted(["embeddings/item/embeddings", f"pretrained_embeddings/pre_a/{dense}/kernel",
                            f"pretrained_embeddings/pre_a/{dense}/bias"])
    assert tuple(ib.weights()[f"pretrained_embeddings/pre_a/{dense}/kernel"].shape) == (300, 64)
    # the tag default picks up the EMBEDDING columns unprojected
    _, widths, _ = mm.InputBlockV2(s).layout()
    assert widths["pre_a"] == 300 and widths["pre_b"] == 12


def test_schema_without_pretrained_columns_is_unchanged():
    mm.set_seed(3)
    a = mm.InputBlockV2(_schema())
    assert a.pretrained is None
    cols, widths, total = a.layout()
    assert list(cols) == ["item", "user_age"] and total == widths["item"] + 1
    a.build(torch.device("cpu"))
    assert list(a.weights()) == ["embeddings/item/embeddings"]


def test_loader_transforms_keep_ids_and_extend_the_schema():
    data = {"item": np.arange(10, dtype=np.int64) % 7, "user_age": np.ones(10, np.float32), "click": np.zeros(10, np.int64)}
    op = mm.EmbeddingOperator(np.random.rand(7, 4), lookup_key="item", embedding_name="vecs", device="cpu")
    ld = mm.Loader(data, batch_size=4, schema=_schema(), shuffle=False, device="cpu", transforms=[op])
    assert ld.output_schema.select_by_tag(Tags.EMBEDDING).column_names == ["vecs"]
    x, y = ld.peek()
    assert "vecs" not in x and "item" in x
    plain = mm.Loader(data, batch_size=4, schema=_schema(), shuffle=False, device="cpu")
    assert plain.output_schema.column_names == ["item", "user_age", "click"]


def test_tensor_initializer_loads_the_table():
    w = np.arange(12, dtype=np.float32).reshape(4, 3)
    s = Schema([ColumnSchema("c", tags=(Tags.CATEGORICAL,), dtype="int64", properties={"domain": {"min": 0, "max": 3}})])
    emb = mm.Embeddings(s, dim=3, embeddings_initializer=mm.TensorInitializer(w))
    emb.build(torch.device("cpu"))
    assert np.array_equal(emb.tables["c"].embeddings.numpy(), w)


@pytest.mark.parametrize("l2", [False, True])
def test_restatement_projection_backward_against_finite_differences(l2):
    rng = np.random.default_rng(5 + l2)
    P, ids = rng.standard_normal((9, 6)), rng.integers(0, 9, 5)
    W, b = rng.standard_normal((6, 4)) * 0.3, rng.standard_normal(4) * 0.1
    R = rng.standard_normal((5, 4))

    def f(W_, b_):
        return float((PO.slot(P, ids, {"name": "p", "kernel": W_, "bias": b_}, l2) * torch.as_tensor(R)).sum())

    V = {}

    def var(k, a):
        V[k] = torch.tensor(np.asarray(a, dtype=np.float64), requires_grad=True)
        return V[k]

    (PO.slot(P, ids, {"name": "p", "kernel": W, "bias": b}, l2, var) * torch.as_tensor(R)).sum().backward()
    eps = 1e-6
    for key, arr in (("p/kernel", W), ("p/bias", b)):
        num = np.zeros_like(arr)
        for i in np.ndindex(arr.shape):
            hi, lo = arr.copy(), arr.copy()
            hi[i] += eps
            lo[i] -= eps
            num[i] = ((f(hi, b) - f(lo, b)) if key == "p/kernel" else (f(W, hi) - f(W, lo))) / (2 * eps)
        np.testing.assert_allclose(V[key].grad.numpy(), num, rtol=1e-6, atol=1e-8)


def test_kernel_cases_reach_every_instantiation():
    """The GPU kernel tests cover every compiled instantiation: the gather's 16-byte and scalar paths (Dp % 4 == 0 and not),
    int32 and int64 ids for the gather, the projection and its backward, the dense-input path, and the limits."""
    from tests import test_gpu_pretrained_kernels as K

    assert any(d % 4 for d in K.DPS) and any(d % 4 == 0 for d in K.DPS)
    assert min(K.DPS) == 1 and max(K.DPS) == 1024 and min(K.OUTS) == 1 and max(K.OUTS) == 256
    kinds = K.test_project_backward_matches_float64_and_repeats.pytestmark
    params = {m.args[0]: m.args[1] for m in kinds if m.name == "parametrize"}
    assert set(params["kind"]) == {"i32", "i64", "dense"} and set(params["l2"]) == {False, True}
    # the grid formula gives one lap below 64 K samples, several and a ragged last one at the benchmark's batch sizes
    sms = 132
    laps = lambda B: -(-B // 64) * 4 / min(-(-B // 64) * 4, sms * 8)  # noqa: E731
    assert laps(1001) == 1 and laps(65536) > 1 and (-(-65573 // 64) * 4) % (sms * 8) != 0
