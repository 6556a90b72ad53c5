"""CPU restatement of one DLRM training step whose categorical features may be multi-hot — test infrastructure.

oracle/oracle_train.py:dlrm_loss_and_grads restates the step for one-hot features; this module restates the same step
(same staging, same orders, float64 autograd) with a feature given in any of the three forms the forward accepts:
  * one-hot (B,) ids;
  * ragged `name__values` + `name__offsets` (tf.nn.safe_embedding_lookup_sparse, inputs/embedding.py:432-441): ids < 0
    are pruned, ids >= rows contribute nothing (TF-GPU gather semantics; the GPU path counts them as out of range), the
    combiner divides by the number of ids kept (mean) or its square root (sqrtn), an empty bag gives zeros;
  * fixed-length (B, L) ids (Embedding + process_sequence_combiner, inputs/embedding.py:457-461, :1556-1587): mean or
    sum over all L positions, padding NOT masked; an id outside [0, rows) reads a zero row.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from oracle.oracle_train import _act


def pool(batch: Dict[str, np.ndarray], name: str, table: torch.Tensor, combiner: str) -> torch.Tensor:
    """The (B, D) embedding of feature `name` read from `table` (differentiable)."""
    rows, D = table.shape
    if name + "__values" in batch:
        values = np.asarray(batch[name + "__values"]).reshape(-1).astype(np.int64)
        offsets = np.asarray(batch[name + "__offsets"]).reshape(-1).astype(np.int64)
        B = offsets.shape[0] - 1
        seg = np.repeat(np.arange(B), np.diff(offsets))
        keep = (values >= 0) & (values < rows)
        emb = table[torch.as_tensor(values[keep])]
        out = torch.zeros((B, D), dtype=table.dtype).index_add(0, torch.as_tensor(seg[keep]), emb)
        cnt = np.bincount(seg[keep], minlength=B).astype(np.float64)
        if combiner == "mean":
            div = np.where(cnt > 0, cnt, 1.0)
        elif combiner == "sqrtn":
            div = np.where(cnt > 0, np.sqrt(cnt), 1.0)
        elif combiner == "sum":
            div = np.ones(B)
        else:
            raise ValueError(combiner)
        return out / torch.as_tensor(div, dtype=table.dtype).reshape(-1, 1)
    ids = np.asarray(batch[name]).astype(np.int64)
    if ids.ndim == 1 or (ids.ndim == 2 and ids.shape[1] == 1):
        return table[torch.as_tensor(ids.reshape(-1))]
    ok = torch.as_tensor((ids >= 0) & (ids < rows))
    emb = table[torch.as_tensor(np.clip(ids, 0, rows - 1))] * ok.unsqueeze(-1).to(table.dtype)
    s = emb.sum(dim=1)
    if combiner == "mean":
        return s / ids.shape[1]
    if combiner == "sum":
        return s
    raise ValueError(combiner)


def dlrm_loss_and_grads(batch: Dict[str, np.ndarray], tables: Dict[str, np.ndarray], feature_table: Dict[str, str],
                        combiners: Dict[str, str], continuous: Sequence[str], bottom: List[dict], top: List[dict], head: dict,
                        targets: np.ndarray, dtype=torch.float64):
    """oracle_train.dlrm_loss_and_grads with each feature pooled by `pool` (combiners: feature -> combiner).
    Returns (loss, logits (B,), grads) with the same keys."""
    P = {}
    for n, t in tables.items():
        P[f"table/{n}"] = torch.tensor(np.asarray(t), dtype=dtype, requires_grad=True)
    for tag, layers in (("bottom", bottom), ("top", top)):
        for i, l in enumerate(layers):
            P[f"{tag}/kernel_{i}"] = torch.tensor(np.asarray(l["kernel"]), dtype=dtype, requires_grad=True)
            if l.get("bias") is not None:
                P[f"{tag}/bias_{i}"] = torch.tensor(np.asarray(l["bias"]), dtype=dtype, requires_grad=True)
    P["head/kernel"] = torch.tensor(np.asarray(head["kernel"]), dtype=dtype, requires_grad=True)
    if head.get("bias") is not None:
        P["head/bias"] = torch.tensor(np.asarray(head["bias"]), dtype=dtype, requires_grad=True)

    def mlp(x, tag, layers):
        for i, l in enumerate(layers):
            x = x @ P[f"{tag}/kernel_{i}"]
            if f"{tag}/bias_{i}" in P:
                x = x + P[f"{tag}/bias_{i}"]
            x = _act(x, l.get("activation"))
        return x

    emb = {n: pool(batch, n, P[f"table/{t}"], combiners.get(n, "mean")) for n, t in feature_table.items()}
    x = torch.cat([torch.as_tensor(np.asarray(batch[k], dtype=np.float64).reshape(-1, 1)).to(dtype) for k in sorted(continuous)], dim=1)
    emb["bottom_block"] = mlp(x, "bottom", bottom)
    stacked = torch.stack([emb[k] for k in sorted(emb)], dim=1)
    z = torch.bmm(stacked, stacked.transpose(1, 2))
    Fn = stacked.shape[1]
    mask = torch.triu(torch.ones(Fn, Fn, dtype=torch.bool), diagonal=1)
    body = mlp(torch.cat([emb["bottom_block"], z[:, mask]], dim=1), "top", top)
    logits = (body @ P["head/kernel"]).reshape(-1)
    if "head/bias" in P:
        logits = logits + P["head/bias"].reshape(-1)
    y = torch.as_tensor(np.asarray(targets, dtype=np.float64).reshape(-1)).to(dtype)
    per = torch.clamp(logits, min=0) - logits * y + torch.log1p(torch.exp(-logits.abs()))
    loss = per.sum() / y.shape[0]
    loss.backward()
    grads = {k: (v.grad.numpy().copy() if v.grad is not None else np.zeros(tuple(v.shape))) for k, v in P.items()}
    return float(loss.item()), logits.detach().numpy().copy(), grads


def touched_rows(batch: Dict[str, np.ndarray], name: str, rows: int) -> np.ndarray:
    """Rows of the table of `name` that the batch's IndexedSlices carry (ids in [0, rows)): the rows a sparse update moves."""
    ids = np.asarray(batch[name + "__values"] if name + "__values" in batch else batch[name]).reshape(-1).astype(np.int64)
    return np.unique(ids[(ids >= 0) & (ids < rows)])
