"""CPU restatement of WideAndDeepModel — test infrastructure.

Forward of WideAndDeepModel (models/ranking.py:504-570, CategoryEncoding transforms/features.py:473-612) in numpy
(`wide_deep_forward`) and the same forward in float64 torch with autograd (`wide_deep_loss_and_grads`):
  wide = sum_f encode(ids_f) . Wk[off_f : off_f + card_f] + bw, features in sorted-name order, encode = one_hot / multi_hot
         (1 at every distinct id of the sample) / count (occurrences); ids outside [0, card) encode to nothing
  deep = act_dl(deep(x0) . w_dl + b_dl), x0 = [embedding rows (lists: mean over the bag) | continuous] in sorted-name order
  s = wide + deep;  z = s w_out + b_out
and the loss of the one output: BCE on the logit or squared error, times the sample weight, summed and divided by B.
A feature is given as (B,) ids, a (B, L) id matrix, or a ragged (values, offsets) pair (only the bag's own ids count).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import scipy.sparse as sp
import torch

from oracle.oracle_train import _act

BCE, MSE = "binary_crossentropy", "mse"


def bags_of(x) -> List[np.ndarray]:
    """Per sample, the ids of a feature given as (B,), (B, L) or (values, offsets)."""
    if isinstance(x, tuple):
        v, o = np.asarray(x[0]).reshape(-1), np.asarray(x[1]).reshape(-1)
        n = v.shape[0]
        out = []
        for b in range(o.shape[0] - 1):
            s, e = min(max(int(o[b]), 0), n), min(max(int(o[b + 1]), 0), n)
            out.append(v[s:max(e, s)].astype(np.int64))
        return out
    x = np.asarray(x)
    return [r.reshape(-1).astype(np.int64) for r in x.reshape(x.shape[0], -1)]


def encode(x, card: int, mode: str) -> np.ndarray:
    """CategoryEncoding of one feature as a dense (B, card) float64 matrix (numpy bincount per sample)."""
    bags = bags_of(x)
    out = np.zeros((len(bags), card))
    for b, ids in enumerate(bags):
        ids = ids[(ids >= 0) & (ids < card)]
        c = np.bincount(ids, minlength=card).astype(np.float64)
        out[b] = np.minimum(c, 1.0) if mode in ("one_hot", "multi_hot") else c
    return out


def _positions(x):
    """(sample, id, bag length) of every position of a feature given as (B,), (B, L) or (values, offsets), vectorised:
    positions outside [offsets[b], offsets[b + 1]) (clamped as bags_of does) belong to no sample and are dropped."""
    if isinstance(x, tuple):
        v, o = np.asarray(x[0]).reshape(-1).astype(np.int64), np.asarray(x[1]).reshape(-1).astype(np.int64)
        n = v.shape[0]
        s = np.clip(o[:-1], 0, n)
        e = np.maximum(np.clip(o[1:], 0, n), s)
        lens = e - s
        b = np.repeat(np.arange(lens.shape[0]), lens)
        pos = np.arange(int(lens.sum())) - np.repeat(np.cumsum(lens) - lens, lens) + np.repeat(s, lens)
        return b, v[pos], lens
    x = np.asarray(x)
    x = x.reshape(x.shape[0], -1)
    B, L = x.shape
    return np.repeat(np.arange(B), L), x.reshape(-1).astype(np.int64), np.full(B, L)


def encode_sparse(x, card: int, mode: str) -> sp.csr_matrix:
    """encode() as a (B, card) CSR matrix, built without a per-sample loop."""
    b, ids, lens = _positions(x)
    ok = (ids >= 0) & (ids < card)
    m = sp.csr_matrix((np.ones(int(ok.sum())), (b[ok], ids[ok])), shape=(lens.shape[0], card))
    m.sum_duplicates()
    if mode in ("one_hot", "multi_hot"):
        m.data = np.minimum(m.data, 1.0)
    return m


def _mean_pool_sparse(x, rows: int, ragged: bool) -> sp.csr_matrix:
    """The (B, rows) weights of the deep mean over a bag: 1 / L per in-range position for fixed bags, 1 / (in-range count)
    for ragged ones, as _pooled."""
    b, ids, lens = _positions(x)
    ok = (ids >= 0) & (ids < rows)
    if ragged:
        n = np.maximum(np.bincount(b[ok], minlength=lens.shape[0]), 1)
    else:
        n = np.maximum(lens, 1)
    m = sp.csr_matrix((1.0 / n[b[ok]], (b[ok], ids[ok])), shape=(lens.shape[0], rows))
    m.sum_duplicates()
    return m


def _pooled(x, table: np.ndarray) -> np.ndarray:
    """Embedding input of one deep feature: the row (one id) or the mean of the bag's in-range rows ((B, L): over L)."""
    if not isinstance(x, tuple) and (np.asarray(x).ndim == 1 or np.asarray(x).shape[1] == 1):
        ids = np.asarray(x).reshape(-1).astype(np.int64)
        ok = (ids >= 0) & (ids < table.shape[0])
        return table[np.where(ok, ids, 0)] * ok[:, None]
    out = []
    for ids in bags_of(x):
        ok = (ids >= 0) & (ids < table.shape[0])
        n = len(ids) if not isinstance(x, tuple) else max(int(ok.sum()), 1)
        out.append((table[ids[ok]].sum(0) if ok.any() else np.zeros(table.shape[1])) / max(n, 1))
    return np.stack(out)


def wide_deep_forward(batch: Dict[str, object], wide: Optional[dict], deep: Optional[dict], head: dict, logits: bool = False):
    """numpy forward.  wide: {"cards": {name: card}, "mode", "kernel" (W, 1), "bias" (1,)}; deep: {"tables": {name: (rows,
    D)}, "continuous": [names], "layers": [{"kernel", "bias", "activation"}], "logit": {"kernel" (U, 1), "bias", "activation"}};
    head: {"kernel" (1, 1), "bias", "activation"}.  Returns (B,) predictions (logits=True: z)."""
    s = 0.0
    if wide is not None:
        off, w = 0, np.zeros(len(bags_of(batch[sorted(wide["cards"])[0]])))
        for n in sorted(wide["cards"]):
            c = wide["cards"][n]
            w = w + encode(batch[n], c, wide["mode"]) @ np.asarray(wide["kernel"], np.float64)[off:off + c, 0]
            off += c
        s = w + float(np.asarray(wide["bias"]).reshape(-1)[0])
    if deep is not None:
        cols = {n: _pooled(batch[n], np.asarray(t, np.float64)) for n, t in deep["tables"].items()}
        cols.update({n: np.asarray(batch[n], np.float64).reshape(-1, 1) for n in deep["continuous"]})
        h = np.concatenate([cols[n] for n in sorted(cols)], axis=1)
        for l in deep["layers"] + [deep["logit"]]:
            h = h @ np.asarray(l["kernel"], np.float64) + (0.0 if l.get("bias") is None else np.asarray(l["bias"], np.float64))
            h = np.maximum(h, 0.0) if l.get("activation") == "relu" else h
        s = s + h.reshape(-1)
    z = s * float(np.asarray(head["kernel"]).reshape(-1)[0]) + float(np.asarray(head["bias"]).reshape(-1)[0])
    if logits or head.get("activation") in (None, "linear"):
        return z
    return 1.0 / (1.0 + np.exp(-z))


def wide_deep_loss_and_grads(batch: Dict[str, object], wide: Optional[dict], deep: Optional[dict], head: dict, targets: np.ndarray,
                             sample_weight=None, sparse: bool = False, masks: Optional[Dict[str, np.ndarray]] = None):
    """The forward of wide_deep_forward in float64 torch, the loss of head["loss"] and autograd.  Returns (loss, z (B,), grads)
    with grads keyed "wide/kernel", "wide/bias", "table/<f>", "deep/kernel_i", "deep/bias_i", "deep_logit/kernel",
    "deep_logit/bias", "head/kernel", "head/bias".

    sparse: the encodings and the multi-hot mean pools as scipy CSR matrices built without a per-sample loop (sizes where
    a dense (B, card) matrix does not fit): the wide term enc @ wk and each pooled input enter autograd as leaves, and
    their parameters' gradients are the closed forms enc^T ds and pool^T d(pooled).

    masks {"deep_i": (B, units)} (optional): where deep layer i's relu passes its input, as the device decided it.  A
    pre-activation within float32 rounding of 0 can take either side of the kink; with the device's decisions the
    restatement's gradients follow the same branch (relu(y) and y * mask differ only at such values)."""

    def var(x):
        return torch.tensor(np.asarray(x, dtype=np.float64), requires_grad=True)

    P = {"head/kernel": var(head["kernel"]), "head/bias": var(head["bias"])}
    leaves = {}  # name: (leaf tensor, CSR matrix, parameter key) for the sparse path
    s = 0.0
    if wide is not None:
        P["wide/kernel"], P["wide/bias"] = var(wide["kernel"]), var(wide["bias"])
        if sparse:
            enc = sp.hstack([encode_sparse(batch[n], wide["cards"][n], wide["mode"]) for n in sorted(wide["cards"])], format="csr")
            t = torch.tensor(enc @ np.asarray(wide["kernel"], np.float64).reshape(-1), requires_grad=True)
            leaves["wide"] = (t, enc, "wide/kernel")
            s = t + P["wide/bias"].reshape(())
        else:
            enc = np.concatenate([encode(batch[n], wide["cards"][n], wide["mode"]) for n in sorted(wide["cards"])], axis=1)
            s = torch.from_numpy(enc) @ P["wide/kernel"].reshape(-1) + P["wide/bias"].reshape(())
    if deep is not None:
        cols = {}
        for n, t in deep["tables"].items():
            P[f"table/{n}"] = var(t)
            x = batch[n]
            rows = P[f"table/{n}"].shape[0]
            if not isinstance(x, tuple) and (np.asarray(x).ndim == 1 or np.asarray(x).shape[1] == 1):
                ids = torch.from_numpy(np.asarray(x).reshape(-1).astype(np.int64))
                ok = ((ids >= 0) & (ids < rows)).double()
                cols[n] = P[f"table/{n}"][ids.clamp(0, rows - 1)] * ok[:, None]
            elif sparse:
                M = _mean_pool_sparse(x, rows, isinstance(x, tuple))
                cols[n] = torch.tensor(M @ np.asarray(t, np.float64), requires_grad=True)
                leaves[f"pool/{n}"] = (cols[n], M, f"table/{n}")
            else:  # mean over the bag as a (B, rows) weight matrix
                bags = bags_of(x)
                M = np.zeros((len(bags), rows))
                for b, ids in enumerate(bags):
                    ok = ids[(ids >= 0) & (ids < rows)]
                    n_ = len(ids) if not isinstance(x, tuple) else max(len(ok), 1)
                    np.add.at(M[b], ok, 1.0 / max(n_, 1))
                cols[n] = torch.from_numpy(M) @ P[f"table/{n}"]
        for n in deep["continuous"]:
            cols[n] = torch.from_numpy(np.asarray(batch[n], np.float64).reshape(-1, 1))
        h = torch.cat([cols[n] for n in sorted(cols)], dim=1)
        for i, l in enumerate(deep["layers"]):
            P[f"deep/kernel_{i}"], P[f"deep/bias_{i}"] = var(l["kernel"]), var(l["bias"])
            h = h @ P[f"deep/kernel_{i}"] + P[f"deep/bias_{i}"]
            if l.get("activation") == "relu" and f"deep_{i}" in (masks or {}):
                h = h * torch.from_numpy(np.asarray(masks[f"deep_{i}"], dtype=np.float64))
            else:
                h = _act(h, l.get("activation"))
        lg = deep["logit"]
        P["deep_logit/kernel"], P["deep_logit/bias"] = var(lg["kernel"]), var(lg["bias"])
        s = s + _act(h @ P["deep_logit/kernel"] + P["deep_logit/bias"], lg.get("activation")).reshape(-1)
    z = s * P["head/kernel"].reshape(()) + P["head/bias"].reshape(())
    y = torch.from_numpy(np.asarray(targets, dtype=np.float64).reshape(-1))
    if head["loss"] == BCE:
        per = torch.clamp(z, min=0) - z * y + torch.log1p(torch.exp(-z.abs()))
    else:
        per = (z - y) ** 2
    if sample_weight is not None:
        per = per * torch.from_numpy(np.asarray(sample_weight, dtype=np.float64).reshape(-1))
    loss = per.sum() / y.shape[0]
    loss.backward()
    grads = {k: (v.grad.numpy().copy() if v.grad is not None else np.zeros(tuple(v.shape))) for k, v in P.items()}
    for leaf, M, key in leaves.values():  # the sparse path's closed forms
        grads[key] = np.asarray(M.T @ leaf.grad.numpy()).reshape(grads[key].shape)
    return float(loss.item()), z.detach().numpy().copy(), grads
