"""Float64 restatement of the label-smoothed full-catalog soft-max cross-entropy (Keras CategoricalCrossentropy(
from_logits=True, label_smoothing=eps)) of a CategoricalOutput over a weight-tied table: the target is
(1 - eps) onehot(y) + eps / N on z = (x E^T + b) / T, with per-row weights c = sample_weight / B."""
import numpy as np


def smoothed_catalog_ce(x, E, b, labels, T: float = 1.0, eps: float = 0.0, sample_weight=None, lse=None):
    """(loss, dx, dE, db) in float64, written as the kernels compute them: with s_E = sum_j E_j and beta = sum_j b_j,
    loss_b = lse_b - (1 - eps) z_b[y_b] - (eps / N) (x_b . s_E + beta) / T;  G = c (softmax - (1 - eps) onehot);
    dx = G E / T - c (eps / N) s_E / T;  dE = G^T x / T - (eps / N T) sum_b c_b x_b;  db = sum_b G / T - (eps / N T) sum_b c_b.
    A label outside [0, N) takes no one-hot term (its loss entry is NaN, as the kernel's target logit) but keeps its
    uniform term.  lse: the rows' log-sum-exp to use instead of recomputing it."""
    x, E = np.asarray(x, np.float64), np.asarray(E, np.float64)
    B, N = x.shape[0], E.shape[0]
    labels = np.asarray(labels).reshape(-1).astype(np.int64)
    bias = np.zeros(N) if b is None else np.asarray(b, np.float64)
    z = (x @ E.T + bias[None, :]) / T
    if lse is None:
        m = z.max(axis=1, keepdims=True)
        lse = (m + np.log(np.exp(z - m).sum(axis=1, keepdims=True)))[:, 0]
    p = np.exp(z - np.asarray(lse, np.float64)[:, None])
    c = (np.ones(B) if sample_weight is None else np.asarray(sample_weight, np.float64).reshape(-1)) / B
    ok = (labels >= 0) & (labels < N)
    onehot = np.zeros((B, N))
    onehot[np.nonzero(ok)[0], labels[ok]] = 1.0
    G = c[:, None] * (p - (1.0 - eps) * onehot)
    s_E, beta = E.sum(axis=0), bias.sum()
    tl = np.where(ok, z[np.arange(B), np.clip(labels, 0, N - 1)], np.nan)
    loss = float(np.sum(c * (lse - (1.0 - eps) * tl - (eps / N) * (x @ s_E + beta) / T)))
    dx = G @ E / T - np.outer(c, s_E) * (eps / N) / T
    dE = G.T @ x / T - (eps / (N * T)) * (c @ x)[None, :]
    db = G.sum(axis=0) / T - (eps / (N * T)) * c.sum()
    return loss, dx, dE, db


def smoothed_by_autograd(x, E, b, labels, T: float = 1.0, eps: float = 0.0, sample_weight=None):
    """The same quantities from torch autograd of F.cross_entropy(z, y, label_smoothing=eps, reduction="none") weighted by
    c (float64, CPU): torch's label smoothing is Keras' ((1 - eps) onehot + eps / N)."""
    import torch

    xt = torch.tensor(np.asarray(x, np.float64), requires_grad=True)
    Et = torch.tensor(np.asarray(E, np.float64), requires_grad=True)
    bt = torch.tensor(np.asarray(b, np.float64) if b is not None else np.zeros(E.shape[0]), requires_grad=True)
    y = torch.tensor(np.asarray(labels).reshape(-1).astype(np.int64))
    z = (xt @ Et.T + bt) / T
    per = torch.nn.functional.cross_entropy(z, y, label_smoothing=eps, reduction="none")
    w = torch.ones(x.shape[0], dtype=torch.float64) if sample_weight is None else torch.tensor(np.asarray(sample_weight, np.float64))
    loss = (per * w).sum() / x.shape[0]
    loss.backward()
    return loss.item(), xt.grad.numpy(), Et.grad.numpy(), bt.grad.numpy()


def smoothed_restated_step(model, feats, labels, eps: float, sample_weight=None, drop=None):
    """catalog_model_oracle.restated_step with the label-smoothed target: (loss, grads by variable name, x) in float64.
    drop: per MLP layer None or a (B, units) multiplier (0 where dropped, 1 / (1 - rate) where kept) applied after the
    layer's activation, as Keras Dropout in training."""
    import torch

    from tests.catalog_model_oracle import _forward

    out = model.prediction
    leaves = {}
    B = len(labels)
    if drop is None:
        h, leaf = _forward(model, feats, leaves)
    else:  # the input block from _forward with the MLP run here
        layers = model.mlp.layers
        model.mlp.layers = []
        try:
            h, leaf = _forward(model, feats, leaves)
        finally:
            model.mlp.layers = layers
        for i, l in enumerate(model.mlp.dense_layers):
            h = h @ leaf(f"mlp/{i}/kernel", l.kernel) + leaf(f"mlp/{i}/bias", l.bias)
            if l.activation == "relu":
                h = torch.relu(h)
            if drop[i] is not None:
                h = h * torch.from_numpy(np.asarray(drop[i], np.float64))
    E = leaf(f"tables/{out.table.table_name}", out.table.table)
    z = h @ E.T
    if out.bias is not None:
        z = z + leaf("bias", out.bias)
    z = z / out.logits_temperature
    y = torch.from_numpy(np.asarray(labels).astype(np.int64))
    per = torch.nn.functional.cross_entropy(z, y, label_smoothing=eps, reduction="none")
    w = torch.ones(B, dtype=torch.float64) if sample_weight is None else torch.from_numpy(np.asarray(sample_weight, np.float64))
    loss = (per * w).sum() / B
    loss.backward()
    return float(loss.item()), {k: v.grad.numpy() for k, v in leaves.items()}, h.detach().numpy()
