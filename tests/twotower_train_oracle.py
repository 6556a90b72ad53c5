"""CPU restatement of one TwoTowerModel training step — test infrastructure.

Forward of the v1 TwoTowerModel (blocks/retrieval/two_tower.py:32-118) with its default ItemRetrievalTask
(prediction_tasks/retrieval.py:33-191) in float64 with autograd:
  per tower x0 = [table rows (one-hot; ragged or (B, L) bags pooled by their combiner) | continuous columns] in sorted-name
  order (a zero row for an id outside [0, rows)), then the MLP;  post="l2-norm": y = x / sqrt(max(sum x^2, 1e-12))
  (transforms/regularization.py:27-82);
  logits s = [q.i | masked(Q I^T)] / T with the batch's own items as negatives, masked where the item ids agree
  (utils/tf_utils.py:126-154: a constant false_negative_score, no gradient);
  loss = mean_b CategoricalCrossentropy(from_logits=True) against the one-hot on column 0 = mean_b (lse_b - s_b0).
The updates are oracle/oracle_train.py's Keras rules (dense_update, sparse_update).
"""
from __future__ import annotations

from typing import Dict, List

import numpy as np
import torch

from oracle.oracle_train import _act, dense_update, sparse_update

MIN_FLOAT = float(np.finfo(np.float16).min) / 100.0


def _pool(w, feat, combiner: str, dtype):
    """Rows of one feature: (B,) ids, (values, offsets) ragged bags or a (B, L) id matrix (padding not masked)."""
    rows = w.shape[0]
    if isinstance(feat, tuple):
        values, offsets = (np.asarray(a).reshape(-1).astype(np.int64) for a in feat)
        out = []
        for b in range(len(offsets) - 1):
            ids = values[offsets[b]:offsets[b + 1]]
            ids = ids[(ids >= 0) & (ids < rows)]
            if len(ids) == 0:
                out.append(torch.zeros(w.shape[1], dtype=dtype))
                continue
            s = w[torch.as_tensor(ids)].sum(0)
            n = float(len(ids))
            out.append(s / n if combiner == "mean" else (s / np.sqrt(n) if combiner == "sqrtn" else s))
        return torch.stack(out)
    ids = np.asarray(feat).astype(np.int64)
    if ids.ndim == 2 and ids.shape[1] == 1:
        ids = ids.reshape(-1)
    t = torch.as_tensor(ids)
    ok = ((t >= 0) & (t < rows)).to(dtype)
    r = w[t.clamp(0, rows - 1)] * ok.unsqueeze(-1)
    if ids.ndim == 1:
        return r
    return r.mean(1) if combiner == "mean" else r.sum(1)


def tower_forward(P, tag: str, tower: dict, batch, dtype):
    cols = {}
    for f in tower["tables"]:
        cols[f] = _pool(P[f"{tag}/table/{f}"], batch[f], tower.get("combiner", {}).get(f, "mean"), dtype)
    for n in tower.get("continuous", []):
        cols[n] = torch.as_tensor(np.asarray(batch[n], dtype=np.float64).reshape(-1, 1)).to(dtype)
    x = torch.cat([cols[n] for n in sorted(cols)], dim=1)
    for i, l in enumerate(tower["layers"]):
        x = x @ P[f"{tag}/kernel_{i}"]
        if f"{tag}/bias_{i}" in P:
            x = x + P[f"{tag}/bias_{i}"]
        x = _act(x, l.get("activation"))
    return x


def l2_normalize(x):
    return x / torch.sqrt(torch.clamp((x * x).sum(-1, keepdim=True), min=1e-12))


def inbatch_ce(q, it, item_ids, temperature: float = 1.0, downscore: bool = True, false_neg_score: float = MIN_FLOAT,
               row_scale=None):
    """sum_b c_b (lse_b - s_b0) of the in-batch logits (c = 1/B: the mean)."""
    B = q.shape[0]
    pos = (q * it).sum(-1, keepdim=True)
    neg = q @ it.T
    if downscore:
        ids = torch.as_tensor(np.asarray(item_ids).reshape(-1).astype(np.int64))
        neg = torch.where(ids.view(-1, 1) == ids.view(1, -1), torch.full_like(neg, false_neg_score), neg)
    s = torch.cat([pos, neg], dim=1) / temperature
    per = torch.logsumexp(s, dim=1) - s[:, 0]
    c = torch.full((B,), 1.0 / B, dtype=q.dtype) if row_scale is None else row_scale
    return (c * per).sum()


def twotower_loss_and_grads(batch: Dict[str, np.ndarray], towers: Dict[str, dict], item_id: str, temperature: float = 1.0,
                            l2: bool = False, downscore: bool = True, false_neg_score: float = MIN_FLOAT, dtype=torch.float64):
    """towers = {"query": t, "item": t}, t = {"tables": {feature: (rows, D)}, "combiner": {feature: name}, "continuous": [names],
    "layers": [{"kernel", "bias" (or None), "activation"}]}.  Returns (loss, {"query": (B, D), "item": (B, D)} outputs,
    grads keyed "<tower>/table/<f>" (dense (rows, D)), "<tower>/kernel_i", "<tower>/bias_i")."""
    P = {}
    for tag, t in towers.items():
        for f, w in t["tables"].items():
            P[f"{tag}/table/{f}"] = torch.tensor(np.asarray(w), dtype=dtype, requires_grad=True)
        for i, l in enumerate(t["layers"]):
            P[f"{tag}/kernel_{i}"] = torch.tensor(np.asarray(l["kernel"]), dtype=dtype, requires_grad=True)
            if l.get("bias") is not None:
                P[f"{tag}/bias_{i}"] = torch.tensor(np.asarray(l["bias"]), dtype=dtype, requires_grad=True)
    out = {tag: tower_forward(P, tag, t, batch, dtype) for tag, t in towers.items()}
    if l2:
        out = {k: l2_normalize(v) for k, v in out.items()}
    loss = inbatch_ce(out["query"], out["item"], batch[item_id], temperature, downscore, false_neg_score)
    loss.backward()
    grads = {k: (v.grad.numpy().copy() if v.grad is not None else np.zeros(tuple(v.shape))) for k, v in P.items()}
    return float(loss.item()), {k: v.detach().numpy().copy() for k, v in out.items()}, grads


def sparse_ids(feat) -> np.ndarray:
    """The ids a feature's IndexedSlices carry (every id of a bag)."""
    if isinstance(feat, tuple):
        values, offsets = (np.asarray(a).reshape(-1) for a in feat)
        return values[offsets[0]:offsets[-1]]
    return np.asarray(feat).reshape(-1)


def train_steps(batches: List[Dict[str, np.ndarray]], towers: Dict[str, dict], item_id: str, opt: str, lr: float,
                temperature: float = 1.0, l2: bool = False, initial_accumulator_value: float = 0.1, **hyper):
    """Several optimizer steps: dense variables take dense_update, tables sparse_update on the rows each batch touched.
    Returns (losses, towers with the trained variables)."""
    import copy

    towers = copy.deepcopy(towers)
    slots = {"sgd": [], "adagrad": ["a"], "adam": ["m", "v"]}[opt]
    init = {"a": initial_accumulator_value, "m": 0.0, "v": 0.0}
    state: Dict[str, dict] = {}
    losses = []
    for step, batch in enumerate(batches, start=1):
        loss, _, grads = twotower_loss_and_grads(batch, towers, item_id, temperature, l2)
        losses.append(loss)
        for tag, t in towers.items():
            for i, l in enumerate(t["layers"]):
                for what in ("kernel", "bias"):
                    if l.get(what) is None:
                        continue
                    key = f"{tag}/{what}_{i}"
                    st = state.setdefault(key, {s: np.full(np.shape(l[what]), init[s]) for s in slots})
                    l[what] = dense_update(opt, l[what], grads[key], st, lr, step=step, **hyper)
            for f, w in t["tables"].items():
                key = f"{tag}/table/{f}"
                st = state.setdefault(key, {s: np.full(np.shape(w), init[s]) for s in slots})
                ids = sparse_ids(batch[f])
                # the slices a step produces: d loss / d row per looked-up id; summing them per id gives the dense gradient
                # rows, so apply the dense gradient once per touched id
                uniq = np.unique(ids[(ids >= 0) & (ids < np.shape(w)[0])].astype(np.int64))
                t["tables"][f] = sparse_update(opt, w, uniq, grads[key][uniq], st, lr, step=step, **hyper)
    return losses, towers


def golden_inputs(z):
    """(batch, towers, ids) of the two-tower training fixture (tests/golden/twotower_train/ref_torch_twotower_train.npz).  The
    tables hold only the rows the batch touches: ids[(tower, f)] maps them back, and the batch's ids are remapped to row
    positions (equal ids stay equal, so the false-negative mask is unchanged)."""
    raw = {k[len("batch_"):]: z[k] for k in z.files if k.startswith("batch_")}
    towers, ids, batch = {}, {}, {}
    for tag in ("query", "item"):
        cols = [str(n) for n in z[f"{tag}_cols"]]
        tables = {f: z[f"{tag}_table_{f}_rows"] for f in cols if f"{tag}_table_{f}_rows" in z.files}
        for f in tables:
            ids[(tag, f)] = z[f"{tag}_table_{f}_ids"]
            if f + "__values" in raw:
                batch[f] = (np.searchsorted(ids[(tag, f)], raw[f + "__values"]), raw[f + "__offsets"])
            else:
                batch[f] = np.searchsorted(ids[(tag, f)], raw[f])
        for n in cols:
            if n not in tables:
                batch[n] = raw[n]
        layers, i = [], 0
        while f"{tag}_kernel_{i}" in z.files:
            layers.append({"kernel": z[f"{tag}_kernel_{i}"], "bias": z[f"{tag}_bias_{i}"], "activation": "relu"})
            i += 1
        towers[tag] = {"tables": tables, "combiner": {f: "mean" for f in tables},
                       "continuous": [n for n in cols if n not in tables], "layers": layers}
    return batch, towers, ids


def golden_variants(z):
    """[(tag, T)] of the fixture's temperature variants; tag prefixes the loss and gradient entries."""
    return [(f"T{float(t):g}".replace(".", "p"), float(t)) for t in z["temperatures"]]
