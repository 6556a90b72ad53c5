"""Float64 restatement of the full-catalog soft-max cross-entropy step of CategoricalOutput over a weight-tied table:
Keras CategoricalCrossentropy(from_logits=True) on z = (x E^T + b) / T (the reference's LogitsTemperatureScaler), mean over
the batch with per-row weights, and its gradients with respect to x, E and b."""
import numpy as np


def catalog_ce(x, E, b, labels, T: float = 1.0, sample_weight=None, lse=None):
    """(loss, dx, dE, db) in float64.  c[b] = sample_weight[b] / B (1 / B without weights); G = c (softmax(z) - onehot);
    dx = G E / T, dE = G^T x / T, db = sum_b G / T.  A label outside [0, N) takes no one-hot term (and no loss term: its
    loss entry is NaN, as the kernel's target logit).  lse: the rows' log-sum-exp to use instead of recomputing it."""
    x, E = np.asarray(x, np.float64), np.asarray(E, np.float64)
    B, N = x.shape[0], E.shape[0]
    labels = np.asarray(labels).reshape(-1).astype(np.int64)
    z = x @ E.T
    if b is not None:
        z = z + np.asarray(b, np.float64)[None, :]
    z = z / T
    if lse is None:
        m = z.max(axis=1, keepdims=True)
        lse = (m + np.log(np.exp(z - m).sum(axis=1, keepdims=True)))[:, 0]
    p = np.exp(z - np.asarray(lse, np.float64)[:, None])
    c = (np.ones(B) if sample_weight is None else np.asarray(sample_weight, np.float64).reshape(-1)) / B
    ok = (labels >= 0) & (labels < N)
    onehot = np.zeros((B, N))
    onehot[np.nonzero(ok)[0], labels[ok]] = 1.0
    G = c[:, None] * (p - onehot)
    tl = np.where(ok, z[np.arange(B), np.clip(labels, 0, N - 1)], np.nan)
    loss = float(np.sum(c * (lse - tl)))
    return loss, G @ E / T, G.T @ x / T, G.sum(axis=0) / T


def closed_form_grads_by_autograd(x, E, b, labels, T: float = 1.0, sample_weight=None):
    """The same quantities from torch autograd of torch.nn.functional.cross_entropy (float64, CPU): the check that
    catalog_ce's closed form G = c (softmax - onehot) / T is the derivative of the loss."""
    import torch

    xt = torch.tensor(np.asarray(x, np.float64), requires_grad=True)
    Et = torch.tensor(np.asarray(E, np.float64), requires_grad=True)
    bt = torch.tensor(np.asarray(b, np.float64) if b is not None else np.zeros(E.shape[0]), requires_grad=True)
    y = torch.tensor(np.asarray(labels).reshape(-1).astype(np.int64))
    z = (xt @ Et.T + bt) / T
    per = torch.nn.functional.cross_entropy(z, y, reduction="none")
    w = torch.ones(x.shape[0], dtype=torch.float64) if sample_weight is None else torch.tensor(np.asarray(sample_weight, np.float64))
    loss = (per * w).sum() / x.shape[0]
    loss.backward()
    return loss.item(), xt.grad.numpy(), Et.grad.numpy(), bt.grad.numpy()
