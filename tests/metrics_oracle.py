"""float64 NumPy restatement of the ranking metrics (Keras 2.9-2.12, restated, not executed):

    loss_h = sum sw l / N  (BCE l = max(z,0) - z y + log1p(exp(-|z|)), MSE l = (z - y)^2);  loss = sum_h lambda_h loss_h
    AUC: bucket(p) = max(ceil(fp32(p) * fp32(T - 1)) - 1, 0) in fp32 (metrics_utils._update_confusion_matrix_variables_
         optimized, thresholds [-1e-7, 1/(T-1), ..., (T-2)/(T-1), 1 + 1e-7]); tp_i = sum_{j>=i} pos_j, fp_i = sum_{j>=i} neg_j,
         tpr_i = tp_i / P, fpr_i = fp_i / Nn, auc = sum_{i<T-1} (fpr_i - fpr_{i+1}) (tpr_i + tpr_{i+1}) / 2
    Precision / Recall / BinaryAccuracy at t: predicted positive <=> p > t
    RootMeanSquaredError = sqrt(sum w (z - y)^2 / sum w)
with div_no_nan (0/0 = 0).  The product must not import this module.
"""
import numpy as np


def div(a, b):
    return float(a) / float(b) if b != 0 else 0.0


def bucket(p, T):
    p32 = np.asarray(p, dtype=np.float32)
    return np.maximum(np.ceil(p32 * np.float32(T - 1)).astype(np.int64) - 1, 0)


def histogram(p, y, w, T):
    pos, neg = np.zeros(T), np.zeros(T)
    b = bucket(p, T)
    w = np.ones(len(b)) if w is None else np.asarray(w, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    np.add.at(pos, b[y == 1], w[y == 1])
    np.add.at(neg, b[y == 0], w[y == 0])
    return pos, neg


def auc(pos, neg):
    tp = np.cumsum(pos[::-1])[::-1]
    fp = np.cumsum(neg[::-1])[::-1]
    tpr = np.array([div(t, tp[0]) for t in tp])
    fpr = np.array([div(f, fp[0]) for f in fp])
    return float(np.sum((fpr[:-1] - fpr[1:]) * (tpr[:-1] + tpr[1:]) / 2.0))


def confusion(p, y, w, t):
    w = np.ones(len(y)) if w is None else np.asarray(w, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    pred = np.asarray(p, dtype=np.float32) > np.float32(t)
    tp = float(np.sum(w[pred & (y == 1)]))
    fp = float(np.sum(w[pred & (y == 0)]))
    fn = float(np.sum(w[~pred & (y == 1)]))
    tn = float(np.sum(w[~pred & (y == 0)]))
    return tp, fp, tn, fn


def precision(p, y, w=None, t=0.5):
    tp, fp, _, _ = confusion(p, y, w, t)
    return div(tp, tp + fp)


def recall(p, y, w=None, t=0.5):
    tp, _, _, fn = confusion(p, y, w, t)
    return div(tp, tp + fn)


def binary_accuracy(p, y, w=None, t=0.5):
    tp, fp, tn, fn = confusion(p, y, w, t)
    return div(tp + tn, tp + fp + tn + fn)


def rmse(z, y, w=None):
    z, y = np.asarray(z, dtype=np.float64), np.asarray(y, dtype=np.float64)
    w = np.ones(len(z)) if w is None else np.asarray(w, dtype=np.float64)
    return float(np.sqrt(div(np.sum(w * (z - y) ** 2), np.sum(w))))


def loss_sum(z, y, kind, sw=None):
    z, y = np.asarray(z, dtype=np.float64), np.asarray(y, dtype=np.float64)
    l = np.maximum(z, 0) - z * y + np.log1p(np.exp(-np.abs(z))) if kind == "binary_crossentropy" else (z - y) ** 2
    return float(np.sum(l if sw is None else l * np.asarray(sw, dtype=np.float64)))


def head_metrics(kind, p, z, y, w=None, T=200, names=None):
    """{name: value} of one output's default metrics (BinaryOutput / RegressionOutput), weights w (None: unweighted)."""
    if kind == "mse":
        return {"root_mean_squared_error": rmse(z, y, w)}
    pos, neg = histogram(p, y, w, T)
    return {"precision": precision(p, y, w), "recall": recall(p, y, w), "binary_accuracy": binary_accuracy(p, y, w),
            "auc": auc(pos, neg)}


def evaluate(outputs, batches, loss_weights=None, T=200, weighted=False):
    """Keras evaluate over batches of per-output (kind, p, z, y, sw) with default metrics: outputs = names in order;
    batches = [[(kind, p, z, y, sw) per output] per batch]; weighted: also `weighted_<name>` with sw."""
    H = len(outputs)
    lw = loss_weights or [1.0] * H
    cat = [[np.concatenate([np.asarray(b[h][i]) for b in batches]) if batches[0][h][i] is not None else None
            for i in range(1, 5)] for h in range(H)]
    N = sum(len(b[0][3]) for b in batches)
    out = {}
    per = [loss_sum(c[1], c[2], batches[0][h][0], c[3]) / N for h, c in enumerate(cat)]
    out["loss"] = float(np.dot(lw, per))
    if H > 1:
        out.update({f"{n}_loss": per[h] for h, n in enumerate(outputs)})
    for h, n in enumerate(outputs):
        p, z, y, sw = cat[h]
        kind = batches[0][h][0]
        sets = [("", None)] + ([("weighted_", sw)] if weighted else [])
        for prefix, w in sets:
            for k, v in head_metrics(kind, p, z, y, w, T).items():
                out[prefix + k if H == 1 else f"{n}/{prefix}{k}"] = v
    last = batches[-1]
    nb = len(last[0][3])
    out["regularization_loss"] = 0.0
    out["loss_batch"] = float(np.dot(lw, [loss_sum(last[h][2], last[h][3], last[h][0], last[h][4]) / nb for h in range(H)]))
    return out


def state(heads, T, n_sets, thresholds):
    """The mm_metrics_update state (H, 27 + 4T) restated: heads = [(kind, p, z, y, sw, mw)] with p the fp32 predictions the
    kernel computes, mw the weights of metric set 1 (set 0 is unweighted)."""
    from models_b200 import _cabi as C

    st = np.zeros((len(heads), C.METRICS_SCALARS + 4 * T))
    for h, (kind, p, z, y, sw, mw) in enumerate(heads):
        y = np.asarray(y, dtype=np.float64)
        st[h, C.METRICS_LOSS] = loss_sum(z, y, kind, sw)
        st[h, C.METRICS_COUNT] = len(y)
        for s, w in enumerate([None, mw][:n_sets]):
            a = C.METRICS_SET0 + s * C.METRICS_SET_STRIDE
            ww = np.ones(len(y)) if w is None else np.asarray(w, dtype=np.float64)
            if kind == "mse":
                st[h, a + C.METRICS_SQ_ERR] = np.sum(ww * (np.asarray(z, dtype=np.float64) - y) ** 2)
                st[h, a + C.METRICS_W_SUM] = np.sum(ww)
                continue
            st[h, a + C.METRICS_POS] = np.sum(ww[y == 1])
            st[h, a + C.METRICS_NEG] = np.sum(ww[y == 0])
            for i, t in enumerate(thresholds[h]):
                tp, fp, _, _ = confusion(p, y, w, t)
                st[h, a + C.METRICS_TP + i], st[h, a + C.METRICS_FP + i] = tp, fp
            pos, neg = histogram(p, y, w, T)
            base = C.METRICS_SCALARS + s * 2 * T
            st[h, base:base + T], st[h, base + T:base + 2 * T] = pos, neg
    return st
