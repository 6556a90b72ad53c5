"""CPU restatement of one DLRM training step with several output heads — test infrastructure.

oracle/oracle_train.py:dlrm_loss_and_grads restates the step for one BinaryOutput and tests/multihot_oracle.py extends
the feature side to multi-hot bags; this module keeps that forward (same staging, same orders, float64 autograd, features
pooled by tests/multihot_oracle.pool) and replaces the single head by H heads on the same top-tower output, with the Keras
semantics of compile(loss_weights=...):
  * head h: z_h = body . w_h + b_h;  BinaryOutput: BCE on the logit, RegressionOutput: (z_h - y_h)^2 (no 1/2 factor);
  * loss_h = sum_i sw_i l_h,i / B  (SUM_OVER_BATCH_SIZE; sw one array for every head, or one per head);
  * total = sum_h lambda_h loss_h.
With one BinaryOutput and lambda = 1 it computes exactly what oracle_train computes.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from oracle.oracle_train import _act
from tests.multihot_oracle import pool

BCE, MSE = "binary_crossentropy", "mse"


def dlrm_multitask_loss_and_grads(batch: Dict[str, np.ndarray], tables: Dict[str, np.ndarray], feature_table: Dict[str, str],
                                  continuous: Sequence[str], bottom: List[dict], top: List[dict], heads: List[dict],
                                  targets: Sequence[np.ndarray], loss_weights: Optional[Sequence[float]] = None,
                                  sample_weight=None, combiners: Optional[Dict[str, str]] = None, dtype=torch.float64):
    """heads[h] = {"name", "kernel" (K, 1), "bias" (1,) or None, "loss": "binary_crossentropy" | "mse"}; targets[h] (B,).
    Returns (total loss, [loss_h], [z_h (B,)], grads) with grads keyed "table/<t>", "bottom/kernel_i", ..., and
    "head/<name>/kernel", "head/<name>/bias"."""
    H = len(heads)
    lws = [1.0] * H if loss_weights is None else [float(v) for v in loss_weights]
    sws = list(sample_weight) if isinstance(sample_weight, (list, tuple)) else [sample_weight] * H
    P = {}
    for n, t in tables.items():
        P[f"table/{n}"] = torch.tensor(np.asarray(t), dtype=dtype, requires_grad=True)
    for tag, layers in (("bottom", bottom), ("top", top)):
        for i, l in enumerate(layers):
            P[f"{tag}/kernel_{i}"] = torch.tensor(np.asarray(l["kernel"]), dtype=dtype, requires_grad=True)
            if l.get("bias") is not None:
                P[f"{tag}/bias_{i}"] = torch.tensor(np.asarray(l["bias"]), dtype=dtype, requires_grad=True)
    for hd in heads:
        P[f"head/{hd['name']}/kernel"] = torch.tensor(np.asarray(hd["kernel"]), dtype=dtype, requires_grad=True)
        if hd.get("bias") is not None:
            P[f"head/{hd['name']}/bias"] = torch.tensor(np.asarray(hd["bias"]), dtype=dtype, requires_grad=True)

    def mlp(x, tag, layers):
        for i, l in enumerate(layers):
            x = x @ P[f"{tag}/kernel_{i}"]
            if f"{tag}/bias_{i}" in P:
                x = x + P[f"{tag}/bias_{i}"]
            x = _act(x, l.get("activation"))
        return x

    emb = {n: pool(batch, n, P[f"table/{t}"], (combiners or {}).get(n, "mean")) for n, t in feature_table.items()}
    x = torch.cat([torch.as_tensor(np.asarray(batch[k], dtype=np.float64).reshape(-1, 1)).to(dtype) for k in sorted(continuous)], dim=1)
    emb["bottom_block"] = mlp(x, "bottom", bottom)
    stacked = torch.stack([emb[k] for k in sorted(emb)], dim=1)
    z = torch.bmm(stacked, stacked.transpose(1, 2))
    Fn = stacked.shape[1]
    mask = torch.triu(torch.ones(Fn, Fn, dtype=torch.bool), diagonal=1)
    body = mlp(torch.cat([emb["bottom_block"], z[:, mask]], dim=1), "top", top)
    total, losses, logits = None, [], []
    for hd, y_np, sw, lw in zip(heads, targets, sws, lws):
        lg = (body @ P[f"head/{hd['name']}/kernel"]).reshape(-1)
        if f"head/{hd['name']}/bias" in P:
            lg = lg + P[f"head/{hd['name']}/bias"].reshape(-1)
        y = torch.as_tensor(np.asarray(y_np, dtype=np.float64).reshape(-1)).to(dtype)
        if hd["loss"] == BCE:
            per = torch.clamp(lg, min=0) - lg * y + torch.log1p(torch.exp(-lg.abs()))
        elif hd["loss"] == MSE:
            per = (lg - y) ** 2
        else:
            raise ValueError(hd["loss"])
        if sw is not None:
            per = per * torch.as_tensor(np.asarray(sw, dtype=np.float64).reshape(-1)).to(dtype)
        lh = per.sum() / y.shape[0]
        term = lh if lw == 1.0 else lw * lh
        total = term if total is None else total + term
        losses.append(float(lh.item()))
        logits.append(lg.detach().numpy().copy())
    total.backward()
    grads = {k: (v.grad.numpy().copy() if v.grad is not None else np.zeros(tuple(v.shape))) for k, v in P.items()}
    return float(total.item()), losses, logits, grads


def heads_ref(x, W, b, losses, ys, sws, lws, mask_relu):
    """The output heads alone (what mm_heads_fwd_bwd computes), float64 autograd on the device of x: (total loss,
    per-head losses, logits (H, M), dx, dW, db)."""
    x = x.double().clone().requires_grad_(True)
    W = W.double().clone().requires_grad_(True)
    b = b.double().clone().requires_grad_(True)
    z = x @ W + b  # (M, H)
    M = x.shape[0]
    per = []
    for h, l in enumerate(losses):
        y = ys[h].double()
        zh = z[:, h]
        term = torch.clamp(zh, min=0) - zh * y + torch.log1p(torch.exp(-zh.abs())) if l == BCE else (zh - y) ** 2
        sw = sws[h].double() if sws[h] is not None else torch.ones(M, dtype=torch.float64, device=x.device)
        per.append((term * sw).sum() / M)
    total = sum(lw * p for lw, p in zip(lws, per))
    total.backward()
    dx = x.grad
    if mask_relu:
        dx = dx * (x > 0)
    return total.detach(), torch.stack([p.detach() for p in per]), z.detach().t(), dx, W.grad, b.grad


def golden_inputs(z):
    """(batch, tables, feature_table, continuous, bottom, top, heads, targets) of the multitask fixture, heads in the
    package's output order (sorted output names)."""
    from tests.golden import replay

    cat = [str(n) for n in z["cat_names"]]
    batch = {k[len("batch_"):]: z[k] for k in z if k.startswith("batch_")}
    heads, ys = [], []
    kinds = dict(zip([str(n) for n in z["target_names"]], [str(k) for k in z["target_kinds"]]))
    names = sorted(f"{t}/{'binary_output' if k == 'binary' else 'regression_output'}" for t, k in kinds.items())
    for name in names:
        t = name.split("/")[0]
        heads.append({"name": name, "target": t, "kernel": z[f"head_{t}_kernel"], "bias": z[f"head_{t}_bias"],
                      "loss": BCE if kinds[t] == "binary" else MSE})
        ys.append(z[f"targets_{t}"])
    return (batch, {n: z[f"table_{n}"] for n in cat}, {n: n for n in cat}, [str(n) for n in z["cont_names"]],
            replay.unpack_layers(z, "bottom"), replay.unpack_layers(z, "top"), heads, ys)
