"""CPU restatement of one DCN-v2 training step — test infrastructure.

Forward of DCNModel (blocks/cross.py:113-221, torch/blocks/cross.py:131-164) in float64 with autograd:
  x0 = [table rows | continuous columns] in sorted-name order (a zero row for an id outside [0, rows));
  x_{l+1} = x0 * (x_l W_l + b_l) + x_l;  deep tower on x_L (stacked) or on x0 (parallel, head input [cross | deep] in the
  given order); H heads as tests/multitask_oracle.py (BCE on the logit / squared error, SUM_OVER_BATCH_SIZE, loss
  weights).  The updates are oracle/oracle_train.py's Keras rules (dense_update, sparse_update).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from oracle.oracle_train import _act

BCE, MSE = "binary_crossentropy", "mse"


def dcn_loss_and_grads(batch: Dict[str, np.ndarray], tables: Dict[str, np.ndarray], continuous: Sequence[str], cross: List[dict],
                       deep: List[dict], heads: List[dict], targets: Sequence[np.ndarray], stacked: bool = True,
                       order: Sequence[str] = ("cross", "deep"), loss_weights: Optional[Sequence[float]] = None,
                       sample_weight=None, dtype=torch.float64):
    """tables: feature -> (rows, D); cross[l] / deep[i] = {"kernel", "bias" (or None), "activation"}; heads[h] = {"name",
    "kernel" (K, 1), "bias", "loss"}.  Returns (total loss, [loss_h], [z_h (B,)], grads keyed "table/<f>", "cross/kernel_l",
    "cross/bias_l", "deep/kernel_i", "deep/bias_i", "head/<name>/kernel", "head/<name>/bias")."""
    H = len(heads)
    lws = [1.0] * H if loss_weights is None else [float(v) for v in loss_weights]
    sws = list(sample_weight) if isinstance(sample_weight, (list, tuple)) else [sample_weight] * H
    P = {f"table/{n}": torch.tensor(np.asarray(t), dtype=dtype, requires_grad=True) for n, t in tables.items()}
    for tag, layers in (("cross", cross), ("deep", deep)):
        for i, l in enumerate(layers):
            P[f"{tag}/kernel_{i}"] = torch.tensor(np.asarray(l["kernel"]), dtype=dtype, requires_grad=True)
            if l.get("bias") is not None:
                P[f"{tag}/bias_{i}"] = torch.tensor(np.asarray(l["bias"]), dtype=dtype, requires_grad=True)
    for hd in heads:
        P[f"head/{hd['name']}/kernel"] = torch.tensor(np.asarray(hd["kernel"]), dtype=dtype, requires_grad=True)
        if hd.get("bias") is not None:
            P[f"head/{hd['name']}/bias"] = torch.tensor(np.asarray(hd["bias"]), dtype=dtype, requires_grad=True)

    cols = {}
    for n in tables:
        w = P[f"table/{n}"]
        ids = torch.as_tensor(np.asarray(batch[n]).reshape(-1).astype(np.int64))
        ok = (ids >= 0) & (ids < w.shape[0])
        cols[n] = w[ids.clamp(0, w.shape[0] - 1)] * ok.to(dtype).unsqueeze(1)
    for n in continuous:
        cols[n] = torch.as_tensor(np.asarray(batch[n], dtype=np.float64).reshape(-1, 1)).to(dtype)
    x0 = torch.cat([cols[n] for n in sorted(cols)], dim=1)

    def dense(x, tag, i, act):
        x = x @ P[f"{tag}/kernel_{i}"]
        if f"{tag}/bias_{i}" in P:
            x = x + P[f"{tag}/bias_{i}"]
        return _act(x, act)

    x = x0
    for i in range(len(cross)):
        x = x0 * dense(x, "cross", i, "linear") + x
    h = x if stacked else x0
    for i, l in enumerate(deep):
        h = dense(h, "deep", i, l.get("activation"))
    if stacked:
        body = h
    else:
        body = torch.cat([x, h] if tuple(order) == ("cross", "deep") else [h, x], dim=1)
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


def golden_inputs(z, tag: str):
    """(batch, tables, continuous, cross, deep, heads, targets, order, ids) of one model of the DCN training fixture.  The
    tables hold only the rows the batch touches: `ids[f]` maps them back, the batch's ids are remapped to row positions."""
    cat = [str(n) for n in z["cat_names"]]
    conts = [str(n) for n in z["cont_names"]]
    batch = {k[len("batch_"):]: z[k] for k in z if k.startswith("batch_")}
    ids = {f: z[f"{tag}_table_{f}_ids"] for f in cat}
    local = dict(batch)
    for f in cat:
        local[f] = np.searchsorted(ids[f], batch[f])
    tables = {f: z[f"{tag}_table_{f}_rows"] for f in cat}

    def layers(grp):
        out, i = [], 0
        while f"{tag}_{grp}_kernel_{i}" in z:
            out.append({"kernel": z[f"{tag}_{grp}_kernel_{i}"], "bias": z[f"{tag}_{grp}_bias_{i}"],
                        "activation": str(z[f"{tag}_{grp}_act_{i}"])})
            i += 1
        return out

    hd = layers("head")[0]
    heads = [{"name": "click/binary_output", "kernel": hd["kernel"], "bias": hd["bias"], "loss": BCE}]
    order = ("cross", "deep") if str(z[f"{tag}_order"]) == "cross_deep" else ("deep", "cross")
    return local, tables, conts, layers("cross"), layers("deep"), heads, [z["targets"]], order, ids
