"""Host side of the ranking metrics: the NumPy restatement against scikit-learn, the finalisation of the device state
(models_b200.metrics.MetricsState.result on a state filled on the host), metric names and compile() parsing."""
import ast
from pathlib import Path

import numpy as np
import pytest
from sklearn.metrics import accuracy_score, precision_score, recall_score, roc_auc_score

import models_b200 as mm
from models_b200 import _cabi
from models_b200 import metrics as M
from models_b200.schema import ColumnSchema, Schema, Tags
from tests import metrics_oracle as O

REPO = Path(__file__).resolve().parents[1]


def test_product_does_not_import_the_oracle():
    for f in (REPO / "models_b200").rglob("*.py"):
        tree = ast.parse(f.read_text())
        for node in ast.walk(tree):
            names = [a.name for a in node.names] if isinstance(node, (ast.Import, ast.ImportFrom)) else []
            mod = node.module or "" if isinstance(node, ast.ImportFrom) else ""
            assert "metrics_oracle" not in mod and not any("metrics_oracle" in n for n in names), f


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_threshold_counts_match_sklearn(seed):
    r = np.random.default_rng(seed)
    y = (r.random(5000) < 0.3).astype(np.int64)
    p = np.clip(r.random(5000).astype(np.float32) * 0.6 + 0.4 * y, 0, 1).astype(np.float32)
    p[:50] = np.float32(0.5)  # p == t is predicted negative
    pred = (p > 0.5).astype(np.int64)
    assert O.precision(p, y) == precision_score(y, pred)
    assert O.recall(p, y) == recall_score(y, pred)
    assert O.binary_accuracy(p, y) == accuracy_score(y, pred)


@pytest.mark.parametrize("T", [200, 1024])
def test_auc_at_bucket_centres_equals_sklearn(T):
    r = np.random.default_rng(T)
    j = r.integers(0, T - 1, 20000)
    p = ((j + 0.5) / (T - 1)).astype(np.float32)
    y = (r.random(20000) < 0.2 + 0.6 * j / T).astype(np.int64)
    pos, neg = O.histogram(p, y, None, T)
    assert abs(O.auc(pos, neg) - roc_auc_score(y, p)) < 1e-12


@pytest.mark.parametrize("T", [200, 1024])
def test_auc_on_continuous_predictions_within_bucket_bound(T):
    r = np.random.default_rng(7)
    y = (r.random(20000) < 0.4).astype(np.int64)
    p = (1 / (1 + np.exp(-(r.normal(size=20000) + 1.2 * y)))).astype(np.float32)
    pos, neg = O.histogram(p, y, None, T)
    # ties inside one bucket move the trapezoid by at most the bucket's share of positive x negative pairs
    bound = float(np.sum(pos * neg)) / (pos.sum() * neg.sum())
    assert abs(O.auc(pos, neg) - roc_auc_score(y, p)) <= bound + 1e-12


def _state(spec, heads):
    """A device-layout state filled on the host from per-head (kind, p, z, y, sw)."""
    T = spec.num_buckets
    st = np.zeros((len(heads), _cabi.METRICS_SCALARS + 4 * T))
    for h, (kind, p, z, y, sw) in enumerate(heads):
        st[h, _cabi.METRICS_LOSS] = O.loss_sum(z, y, kind, sw)
        st[h, _cabi.METRICS_COUNT] = len(y)
        for s, w in enumerate([None, sw][:len(spec.sets)]):
            a = _cabi.METRICS_SET0 + s * _cabi.METRICS_SET_STRIDE
            ww = np.ones(len(y)) if w is None else w
            if kind == "mse":
                st[h, a + _cabi.METRICS_SQ_ERR] = np.sum(ww * (np.float64(z) - y) ** 2)
                st[h, a + _cabi.METRICS_W_SUM] = np.sum(ww)
                continue
            st[h, a + _cabi.METRICS_POS] = np.sum(ww[y == 1])
            st[h, a + _cabi.METRICS_NEG] = np.sum(ww[y == 0])
            for i, t in enumerate(spec.thresholds[h]):
                tp, fp, _, _ = O.confusion(p, y, w, t)
                st[h, a + _cabi.METRICS_TP + i], st[h, a + _cabi.METRICS_FP + i] = tp, fp
            pos, neg = O.histogram(p, y, w, T)
            base = _cabi.METRICS_SCALARS + s * 2 * T
            st[h, base:base + T], st[h, base + T:base + 2 * T] = pos, neg
    return st


class _HostState(M.MetricsState):
    def __init__(self, spec, st):
        import torch

        self.spec = spec
        self.state = torch.from_numpy(st)
        self.before_last = torch.zeros((st.shape[0], 2), dtype=torch.float64)


def _binary(n=3000, seed=0):
    r = np.random.default_rng(seed)
    y = (r.random(n) < 0.35).astype(np.float64)
    z = (r.normal(size=n) + 1.5 * y).astype(np.float32)
    p = (1 / (1 + np.exp(-z.astype(np.float64)))).astype(np.float32)
    return ("binary_crossentropy", p, z, y, r.random(n).astype(np.float32))


def _regression(n=3000, seed=1):
    r = np.random.default_rng(seed)
    y = r.normal(size=n) * 2
    z = (y + r.normal(size=n)).astype(np.float32)
    return ("mse", z, z, y, r.random(n).astype(np.float32))


def test_result_follows_the_formulas_single_and_multi_output():
    b = mm.BinaryOutput("click")
    spec = M.MetricsSpec([b], [1.0], None, ["auc", "precision"])
    head = _binary()
    got = _HostState(spec, _state(spec, [head])).result()
    want = O.evaluate(["click/binary_output"], [[head]], weighted=False)
    kind, p, z, y, sw = head
    want["weighted_auc"] = O.auc(*O.histogram(p, y, sw, 200))
    want["weighted_precision"] = O.precision(p, y, sw)
    want["loss_batch"] = want["loss"]
    assert set(got) == set(want)
    for k in want:
        assert abs(got[k] - want[k]) <= 1e-12 * max(1.0, abs(want[k])), k

    outs = [mm.BinaryOutput("click"), mm.RegressionOutput("rating")]
    spec = M.MetricsSpec(outs, [0.5, 2.0])
    heads = [_binary(seed=3), _regression()]
    got = _HostState(spec, _state(spec, heads)).result()
    want = O.evaluate([o.name for o in outs], [heads], loss_weights=[0.5, 2.0])
    want["loss_batch"] = want["loss"]
    assert set(got) == set(want)
    for k in want:
        assert abs(got[k] - want[k]) <= 1e-12 * max(1.0, abs(want[k])), k


@pytest.mark.parametrize("labels", ["ones", "zeros"])
def test_degenerate_labels_give_div_no_nan_zeros(labels):
    spec = M.MetricsSpec([mm.BinaryOutput("click")], [1.0])
    kind, p, z, y, sw = _binary()
    y = np.ones_like(y) if labels == "ones" else np.zeros_like(y)
    got = _HostState(spec, _state(spec, [(kind, p, z, y, None)])).result()
    assert got["auc"] == 0.0  # one of tpr / fpr is 0 everywhere
    if labels == "zeros":
        assert got["precision"] == 0.0 or got["precision"] == O.precision(p, y)
        assert got["recall"] == 0.0
    else:
        assert got["recall"] == O.recall(p, y)
    empty = _HostState(spec, np.zeros((1, _cabi.METRICS_SCALARS + 800))).result()
    assert all(v == 0.0 for v in empty.values())


def _features():
    base = mm.datasets.criteo_schema({k: min(v, 100) for k, v in mm.datasets.CRITEO_MAX.items()})
    return [c for c in base if not c.has_tag(Tags.TARGET)]


def _reference_schema():
    return Schema(_features() + [ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64")])


def test_names_match_the_reference_single_output():
    model = mm.DLRMModel(_reference_schema(), embedding_dim=4, bottom_block=mm.MLPBlock([4]))
    model.compile(optimizer="adam")
    assert set(model.metrics_names) == {"loss", "loss_batch", "regularization_loss", "precision", "recall", "binary_accuracy", "auc"}
    model.compile(optimizer="adam", weighted_metrics=(mm.metrics.Precision(name="precision"), mm.metrics.Recall(name="recall"),
                                                      mm.metrics.BinaryAccuracy(name="binary_accuracy"), mm.metrics.AUC(name="auc")))
    assert set(model.metrics_names) == {"loss", "loss_batch", "regularization_loss", "binary_accuracy", "recall", "precision", "auc",
                                        "weighted_binary_accuracy", "weighted_recall", "weighted_precision", "weighted_auc"}


def test_names_match_the_reference_multi_task():
    cols = _features()
    for t in ("click", "follow", "like", "share"):
        cols.append(ColumnSchema(t, tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"))
    cols.append(ColumnSchema("watching_times", tags=(Tags.TARGET, Tags.REGRESSION), dtype="float32"))
    schema = Schema(cols)
    model = mm.DLRMModel(schema, embedding_dim=4, bottom_block=mm.MLPBlock([4]), prediction_tasks=mm.OutputBlock(schema))
    model.compile(optimizer="adam")
    want = {"loss", "regularization_loss", "loss_batch", "watching_times/regression_output_loss",
            "watching_times/regression_output/root_mean_squared_error"}
    for t in ("click", "follow", "like", "share"):
        want |= {f"{t}/binary_output_loss", f"{t}/binary_output/precision", f"{t}/binary_output/recall",
                 f"{t}/binary_output/binary_accuracy", f"{t}/binary_output/auc"}
    assert set(model.metrics_names) == want


def test_compile_parses_metric_specs():
    b, r = mm.BinaryOutput("click"), mm.RegressionOutput("rating")
    spec = M.MetricsSpec([b, r], [1, 1], {"click/binary_output": ["AUC", mm.metrics.Precision(0.7)]},
                         {"rating/regression_output": "root_mean_squared_error"})
    assert spec.metric_keys() == ["click/binary_output/auc", "click/binary_output/precision",
                                  "rating/regression_output/weighted_root_mean_squared_error"]
    assert spec.thresholds == [[0.7], []]
    spec = M.MetricsSpec([b], [1], [mm.metrics.AUC(num_thresholds=1024), mm.metrics.BinaryAccuracy(threshold=0.3), "recall"])
    assert spec.num_buckets == 1024 and spec.thresholds == [[0.3, 0.5]]
    assert M.MetricsSpec([b], [1], []).metric_keys() == []


@pytest.mark.parametrize("bad, exc", [
    (lambda: mm.metrics.AUC(curve="PR"), NotImplementedError),
    (lambda: mm.metrics.AUC(from_logits=True), NotImplementedError),
    (lambda: mm.metrics.AUC(multi_label=True), NotImplementedError),
    (lambda: mm.metrics.AUC(num_thresholds=1), ValueError),
    (lambda: mm.metrics.AUC(num_thresholds=2000), ValueError),
    (lambda: mm.metrics.Precision(thresholds=[0.3, 0.5]), NotImplementedError),
    (lambda: mm.metrics.Recall(top_k=5), NotImplementedError),
    (lambda: M.get("mean_absolute_error"), NotImplementedError),
    (lambda: M.get(mm.RecallAt(10)), NotImplementedError),
    (lambda: M.MetricsSpec([mm.RegressionOutput("r")], [1], ["auc"]), NotImplementedError),
    (lambda: M.MetricsSpec([mm.BinaryOutput("c")], [1], ["rmse"]), NotImplementedError),
    (lambda: M.MetricsSpec([mm.BinaryOutput("c")], [1], {"nope": "auc"}), ValueError),
    (lambda: M.MetricsSpec([mm.BinaryOutput("c")], [1], ["auc", "auc"]), ValueError),
    (lambda: M.MetricsSpec([mm.BinaryOutput("c")], [1], [mm.metrics.AUC(100)], [mm.metrics.AUC(200)]), NotImplementedError),
    (lambda: M.MetricsSpec([mm.BinaryOutput("c")], [1], [mm.metrics.Precision(t / 10, name=f"p{t}") for t in range(1, 6)]),
     NotImplementedError),
])
def test_compile_rejections(bad, exc):
    with pytest.raises(exc):
        bad()


def test_evaluate_needs_compile_and_out_of_scope_calls_raise():
    model = mm.DLRMModel(_reference_schema(), embedding_dim=4, bottom_block=mm.MLPBlock([4]))
    with pytest.raises(RuntimeError, match="compile"):
        model.evaluate([])
    with pytest.raises(NotImplementedError):
        model.predict({})
    model.compile(optimizer="adam")
    with pytest.raises(NotImplementedError):
        model.evaluate([], callbacks=[object()])
    with pytest.raises(NotImplementedError):
        model.fit([], callbacks=[object()])
