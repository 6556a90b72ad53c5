"""Keras metrics of the ranking outputs, accumulated on the device.

Reference: BinaryOutput's default metrics Precision, Recall, BinaryAccuracy and AUC (outputs/classification.py:37-50),
RegressionOutput's RootMeanSquaredError (outputs/regression.py:42-44), reported by BaseModel.test_step / compute_metrics
(models/base.py:1176-1310).  One launch of mm_metrics_update per batch adds the batch into an fp64 state that stays on the
device; `MetricsState.result()` reads it once (one device-to-host copy) and applies the Keras formulas:

    loss_h = sum sw l / N,  loss = sum_h lambda_h loss_h       (per-batch sum_over_batch_size, batch-size weighted mean)
    tp_i = sum_{j>=i} pos_j, fp_i = sum_{j>=i} neg_j, fn_i = P - tp_i, tn_i = Nn - fp_i        (AUC thresholds i < T)
    auc = sum_{i<T-1} (fpr_i - fpr_{i+1}) (tpr_i + tpr_{i+1}) / 2                          (curve="ROC", interpolation)
    precision = tp / (tp + fp), recall = tp / (tp + fn), binary_accuracy = (tp + tn) / (tp + fp + tn + fn)   (p > t)
    root_mean_squared_error = sqrt(sum w (z - y)^2 / sum w)

with 0/0 = 0 (div_no_nan).  Only these metrics exist: anything else raises NotImplementedError naming it.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _cabi, ops


class Metric:
    """A metric of one output: its Keras name and what the kernel has to count for it."""

    binary = True  # BinaryOutput metric (else RegressionOutput)
    threshold: Optional[float] = None

    def __init__(self, name: str):
        self.name = name

    def __repr__(self):
        return f"{type(self).__name__}(name={self.name!r})"


def _one_threshold(thresholds, what: str) -> float:
    if thresholds is None:
        return 0.5
    if isinstance(thresholds, (list, tuple, np.ndarray)):
        raise NotImplementedError(f"{what}: a list of thresholds is not implemented (one value, one metric)")
    return float(thresholds)


class AUC(Metric):
    """tf.keras.metrics.AUC: ROC curve, interpolated summation, `num_thresholds` evenly spaced thresholds (2..1024)."""

    def __init__(self, num_thresholds: int = 200, curve: str = "ROC", summation_method: str = "interpolation",
                 name: Optional[str] = None, thresholds=None, multi_label: bool = False, num_labels=None, label_weights=None,
                 from_logits: bool = False, **kwargs):
        super().__init__(name or "auc")
        if curve != "ROC":
            raise NotImplementedError(f"AUC(curve={curve!r}): only curve='ROC' is implemented")
        if summation_method != "interpolation":
            raise NotImplementedError(f"AUC(summation_method={summation_method!r}): only 'interpolation' is implemented")
        for arg, v in (("thresholds", thresholds), ("num_labels", num_labels), ("label_weights", label_weights)):
            if v is not None:
                raise NotImplementedError(f"AUC({arg}=...) is not implemented")
        if multi_label:
            raise NotImplementedError("AUC(multi_label=True) is not implemented")
        if from_logits:
            raise NotImplementedError("AUC(from_logits=True) is not implemented: the outputs are probabilities")
        if kwargs:
            raise NotImplementedError(f"AUC arguments {sorted(kwargs)} are not implemented")
        self.num_thresholds = int(num_thresholds)
        if not 2 <= self.num_thresholds <= _cabi.METRICS_MAX_BUCKETS:
            raise ValueError(f"AUC num_thresholds must lie in [2, {_cabi.METRICS_MAX_BUCKETS}], got {num_thresholds}")


class Precision(Metric):
    """tf.keras.metrics.Precision at one threshold (default 0.5): predicted positive when p > threshold."""

    def __init__(self, thresholds=None, top_k=None, class_id=None, name: Optional[str] = None, **kwargs):
        super().__init__(name or "precision")
        if top_k is not None or class_id is not None:
            raise NotImplementedError(f"{type(self).__name__}(top_k / class_id) is not implemented")
        if kwargs:
            raise NotImplementedError(f"{type(self).__name__} arguments {sorted(kwargs)} are not implemented")
        self.threshold = _one_threshold(thresholds, type(self).__name__)


class Recall(Precision):
    """tf.keras.metrics.Recall at one threshold (default 0.5)."""

    def __init__(self, thresholds=None, top_k=None, class_id=None, name: Optional[str] = None, **kwargs):
        super().__init__(thresholds, top_k, class_id, name=name or "recall", **kwargs)


class BinaryAccuracy(Metric):
    """tf.keras.metrics.BinaryAccuracy(threshold=0.5): the fraction of samples with (p > threshold) == y."""

    def __init__(self, name: Optional[str] = None, threshold: float = 0.5, **kwargs):
        super().__init__(name or "binary_accuracy")
        if kwargs:
            raise NotImplementedError(f"BinaryAccuracy arguments {sorted(kwargs)} are not implemented")
        self.threshold = _one_threshold(threshold, "BinaryAccuracy")


class RootMeanSquaredError(Metric):
    """tf.keras.metrics.RootMeanSquaredError."""

    binary = False

    def __init__(self, name: Optional[str] = None, **kwargs):
        super().__init__(name or "root_mean_squared_error")
        if kwargs:
            raise NotImplementedError(f"RootMeanSquaredError arguments {sorted(kwargs)} are not implemented")


_BY_NAME = {"auc": AUC, "precision": Precision, "recall": Recall, "binary_accuracy": BinaryAccuracy,
            "root_mean_squared_error": RootMeanSquaredError, "rmse": RootMeanSquaredError}
_CLASS_NAMES = {"AUC": "auc", "Precision": "precision", "Recall": "recall", "BinaryAccuracy": "binary_accuracy",
                "RootMeanSquaredError": "root_mean_squared_error"}


def get(spec) -> Metric:
    """A Metric from an instance or a Keras name ("auc", "AUC", "precision", "binary_accuracy", ...)."""
    if isinstance(spec, Metric):
        return spec
    if isinstance(spec, str):
        key = _CLASS_NAMES.get(spec, spec.lower())
        if key in _BY_NAME:
            return _BY_NAME[key]()
    raise NotImplementedError(f"metric {spec!r} is not implemented for ranking models; implemented: AUC, Precision, Recall, "
                              "BinaryAccuracy, RootMeanSquaredError")


def default_metrics(output) -> List[Metric]:
    """The reference's defaults: BinaryOutput -> Precision, Recall, BinaryAccuracy, AUC; RegressionOutput -> RMSE."""
    if output.loss == "mse":
        return [RootMeanSquaredError()]
    return [Precision(), Recall(), BinaryAccuracy(), AUC()]


def _per_output(spec, outputs, what: str, defaults: bool) -> List[List[Metric]]:
    names = [o.name for o in outputs]
    if spec is None:
        return [default_metrics(o) if defaults else [] for o in outputs]
    if isinstance(spec, dict):
        unknown = sorted(set(spec) - set(names))
        if unknown:
            raise ValueError(f"{what} names unknown outputs {unknown}; outputs are {names}")
        per = [spec.get(n, []) for n in names]
    elif isinstance(spec, (list, tuple)):
        per = [spec] * len(outputs)
    else:
        per = [[spec]] * len(outputs)
    out = []
    for o, ms in zip(outputs, per):
        ms = [get(m) for m in (ms if isinstance(ms, (list, tuple)) else [ms])]
        for m in ms:
            if m.binary != (o.loss != "mse"):
                raise NotImplementedError(f"{what}: {m!r} on the output {o.name!r} ({o.loss} loss) is not implemented")
        seen = [m.name for m in ms]
        if len(set(seen)) != len(seen):
            raise ValueError(f"{what} of output {o.name!r}: metric names must be unique, got {seen}")
        out.append(ms)
    return out


class MetricsSpec:
    """`compile(metrics=..., weighted_metrics=...)` resolved over the model's outputs: `metrics` None gives every output
    the reference's defaults, a list applies to every output, a dict maps output names to a metric or a list (outputs
    it omits get none); `weighted_metrics` likewise, without defaults, reported as `weighted_<name>`."""

    def __init__(self, outputs: Sequence, loss_weights: Sequence[float], metrics=None, weighted_metrics=None):
        self.outputs = list(outputs)
        if len(self.outputs) > _cabi.METRICS_MAX_HEADS:
            raise NotImplementedError(f"metrics of more than {_cabi.METRICS_MAX_HEADS} outputs are not implemented")
        self.names = [o.name for o in self.outputs]
        self.losses = [o.loss for o in self.outputs]
        self.loss_weights = [float(v) for v in loss_weights]
        self.sets = [_per_output(metrics, self.outputs, "metrics", True),
                     _per_output(weighted_metrics, self.outputs, "weighted_metrics", False)]
        if not any(self.sets[1]):
            self.sets = self.sets[:1]
        aucs = {m.num_thresholds for s in self.sets for ms in s for m in ms if isinstance(m, AUC)}
        if len(aucs) > 1:
            raise NotImplementedError(f"AUC metrics with different num_thresholds {sorted(aucs)} in one model are not implemented")
        self.num_buckets = aucs.pop() if aucs else 200
        self.thresholds: List[List[float]] = []
        for h, o in enumerate(self.outputs):
            thr = []
            for s in self.sets:
                for m in s[h]:
                    if m.threshold is not None and m.threshold not in thr:
                        thr.append(m.threshold)
            if len(thr) > _cabi.METRICS_MAX_THRESHOLDS:
                raise NotImplementedError(f"output {o.name!r}: more than {_cabi.METRICS_MAX_THRESHOLDS} distinct decision thresholds "
                                          f"{thr} are not implemented")
            self.thresholds.append(thr)

    @property
    def single(self) -> bool:
        return len(self.outputs) == 1

    def metric_keys(self) -> List[str]:
        """Names of the metrics alone (no losses), in result order."""
        keys = []
        for h, n in enumerate(self.names):
            for s, prefix in zip(self.sets, ("", "weighted_")):
                for m in s[h]:
                    keys.append(prefix + m.name if self.single else f"{n}/{prefix}{m.name}")
        return keys

    def result_names(self) -> List[str]:
        """`model.metrics_names` of evaluate: loss, the per-output losses (several outputs), the metrics,
        regularization_loss, loss_batch."""
        losses = [] if self.single else [f"{n}_loss" for n in self.names]
        return ["loss"] + losses + self.metric_keys() + ["regularization_loss", "loss_batch"]


def _div(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.divide(a, b, out=np.zeros(np.broadcast(a, b).shape), where=b != 0)


def auc_from_histogram(pos: np.ndarray, neg: np.ndarray) -> float:
    """Keras AUC (ROC, interpolation) from the bucket weights of the positives and the negatives."""
    tp = np.cumsum(pos[::-1])[::-1]
    fp = np.cumsum(neg[::-1])[::-1]
    P, Nn = tp[0], fp[0]
    tpr, fpr = _div(tp, P), _div(fp, Nn)
    return float(np.sum((fpr[:-1] - fpr[1:]) * (tpr[:-1] + tpr[1:]) / 2.0))


class MetricsState:
    """The device state of one evaluation (or one epoch of training metrics) of a model's outputs: `update` per batch,
    `result` once at the end."""

    def __init__(self, spec: MetricsSpec, device):
        self.spec = spec
        self.device = device
        H, T = len(spec.outputs), spec.num_buckets
        self.state = torch.zeros((H, _cabi.METRICS_SCALARS + 4 * T), dtype=torch.float64, device=device)
        self.before_last = torch.zeros((H, 2), dtype=torch.float64, device=device)  # loss sum / count before the last batch
        self.workspace = torch.empty(0, dtype=torch.uint8, device=device)

    # the embeddings' L2 term of a model that has one, created by its first update: [sum_k b_k reg_k, sum_k b_k, last reg_k]
    reg: Optional[torch.Tensor] = None

    def reset(self) -> None:
        self.state.zero_()
        self.before_last.zero_()
        if self.reg is not None:
            self.reg.zero_()

    def reserve(self, M: int) -> None:
        need = ops.metrics_workspace_bytes(M, len(self.spec.outputs))
        if self.workspace.numel() < need:
            self.workspace = torch.empty(need, dtype=torch.uint8, device=self.device)

    def update(self, z: torch.Tensor, targets: Sequence[torch.Tensor], pred_form: int, sample_weight=None,
               regularization: Optional[torch.Tensor] = None) -> None:
        """z (H, b) logits; targets one (b,) tensor per output; sample_weight None, one (b,) tensor or one per output (the
        loss and the weighted metrics use it, the plain metrics do not); regularization: one device float, the batch's
        embeddings L2 term, added to the loss batch-size weighted as the batch losses are."""
        if regularization is not None:
            if self.reg is None:
                self.reg = torch.zeros(3, dtype=torch.float64, device=self.device)
            b = z.shape[1]
            r = regularization.reshape(-1)[:1].to(torch.float64)
            self.reg[:1].add_(r, alpha=float(b))
            self.reg[1:2].add_(float(b))
            self.reg[2:].copy_(r)
        H = len(self.spec.outputs)
        sws = list(sample_weight) if isinstance(sample_weight, (list, tuple)) else [sample_weight] * H
        sws = [None if w is None else w.reshape(-1).to(torch.float32).contiguous() for w in sws]
        sets = [[None] * H] + ([sws] if len(self.spec.sets) > 1 else [])
        self.reserve(z.shape[1])
        self.before_last.copy_(self.state[:, :2])
        ops.metrics_update(z, self.spec.losses, [t.reshape(-1) for t in targets], self.state, self.workspace,
                           self.spec.num_buckets, [pred_form] * H, self.spec.thresholds, sample_weight=sws, metric_weights=sets)

    def result(self) -> Dict[str, float]:
        """One device-to-host copy of the state -> {name: value} in `spec.result_names()` order.  Raises ValueError naming
        the outputs that saw invalid samples (a binary target outside {0, 1}, a NaN target or logit)."""
        spec = self.spec
        reg = self.reg if self.reg is not None else torch.zeros(3, dtype=torch.float64, device=self.state.device)
        host = torch.cat([self.state.reshape(-1), self.before_last.reshape(-1), reg]).cpu().numpy()
        reg_sum, reg_n, reg_last = host[-3:]
        H, T = len(spec.outputs), spec.num_buckets
        st = host[:self.state.numel()].reshape(H, -1)
        prev = host[self.state.numel():-3].reshape(H, 2)
        bad = [f"{n} ({int(st[h, _cabi.METRICS_INVALID])} samples)" for h, n in enumerate(spec.names) if st[h, _cabi.METRICS_INVALID]]
        if bad:
            raise ValueError(f"invalid targets or predictions for {', '.join(bad)}: binary targets must be 0 or 1, and no "
                             "target or prediction may be NaN")
        L, N = st[:, _cabi.METRICS_LOSS], st[:, _cabi.METRICS_COUNT]
        per = _div(L, N)
        last = _div(L - prev[:, 0], N - prev[:, 1])
        out = {"loss": float(np.dot(spec.loss_weights, per)) + (float(reg_sum / reg_n) if reg_n else 0.0)}
        if not spec.single:
            out.update({f"{n}_loss": float(per[h]) for h, n in enumerate(spec.names)})
        S = _cabi.METRICS_SCALARS
        for h, n in enumerate(spec.names):
            for s, (ms, prefix) in enumerate(zip(spec.sets, ("", "weighted_"))):
                a = st[h, _cabi.METRICS_SET0 + s * _cabi.METRICS_SET_STRIDE:]
                P, Nn = a[_cabi.METRICS_POS], a[_cabi.METRICS_NEG]
                for m in ms[h]:
                    if isinstance(m, AUC):
                        hist = st[h, S + s * 2 * T: S + (s + 1) * 2 * T]
                        v = auc_from_histogram(hist[:T], hist[T:])
                    elif isinstance(m, RootMeanSquaredError):
                        v = float(np.sqrt(_div(a[_cabi.METRICS_SQ_ERR], a[_cabi.METRICS_W_SUM])))
                    else:
                        i = spec.thresholds[h].index(m.threshold)
                        tp, fp = a[_cabi.METRICS_TP + i], a[_cabi.METRICS_FP + i]
                        fn, tn = P - tp, Nn - fp
                        if isinstance(m, BinaryAccuracy):
                            v = float(_div(tp + tn, P + Nn))
                        elif isinstance(m, Recall):
                            v = float(_div(tp, tp + fn))
                        else:
                            v = float(_div(tp, tp + fp))
                    out[prefix + m.name if spec.single else f"{n}/{prefix}{m.name}"] = v
        out["regularization_loss"] = float(reg_last)
        out["loss_batch"] = float(np.dot(spec.loss_weights, last)) + float(reg_last)
        return out
