"""CPU restatement of an input block with pretrained features feeding the DCN and sequential bodies — test infrastructure.

float64 torch autograd over the TensorFlow semantics:
  * x0: the concat, in sorted-name order, of one-hot embedding rows, continuous columns and the pretrained slots;
    a slot is P[ids] (or the batch's own (B, Dp) vectors), then optionally Dense(new_dim) (inputs/embedding.py:770-781,
    MLPBlock([new_dim], activation=None)), then optionally L2Norm x / sqrt(max(sum x^2, 1e-12));
  * body "dcn" (stacked): x_{l+1} = x0 * (x_l W_l + b_l) + x_l, then the deep MLP; body "mlp": the MLP on x0;
    body "mmoe": the MLP, then relu experts and a stacked bias-free gate layer (tests/mmoe_oracle.gate_mix);
  * one BinaryOutput head: BCE on the logit, mean over the batch.
Nothing flows into P.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch

from oracle.oracle_train import _act
from tests.mmoe_oracle import gate_mix, heads_loss


def slot(P: np.ndarray, ids: Optional[np.ndarray], proj: Optional[dict], l2: bool, var=None) -> torch.Tensor:
    """One pretrained slot (B, width): P[ids] (ids None: P itself), projected and l2-normalised as configured; var(key,
    array) makes the projection's variables (plain tensors without it)."""
    P = np.asarray(P, dtype=np.float64)
    rows = P if ids is None else P[np.asarray(ids).reshape(-1)]
    y = torch.as_tensor(rows)
    if proj is not None:
        mk = var or (lambda k, a: torch.as_tensor(np.asarray(a, dtype=np.float64)))
        y = y @ mk(f"{proj['name']}/kernel", proj["kernel"])
        if proj.get("bias") is not None:
            y = y + mk(f"{proj['name']}/bias", proj["bias"])
    if l2:
        y = y / torch.sqrt(torch.clamp((y * y).sum(1, keepdim=True), min=1e-12))
    return y


def loss_and_grads(batch: Dict[str, np.ndarray], tables: Dict[str, np.ndarray], continuous: List[str], pretrained: List[dict],
                   body: str, layers: Dict[str, List[dict]], head: dict, targets: np.ndarray,
                   masks: Optional[Dict[str, np.ndarray]] = None):
    """pretrained: [{"name", "P", "ids" (or None), "proj" ({"name", "kernel", "bias"} or None), "l2"}]; layers: "cross",
    "deep" (dcn) / "bottom" (mlp, mmoe) / "experts" (one stacked layer, with "E") / "gates" (a (K, E) kernel); each layer
    {"kernel", "bias", "activation"}.  masks {"<chain>_i": (B, units)}: the device's relu decisions.  Returns (loss,
    logits (B,), grads keyed "<name>/kernel|bias" for the projections and "<chain>/kernel_i|bias_i", "head/kernel|bias")."""
    V: Dict[str, torch.Tensor] = {}
    masks = masks or {}

    def var(k, a):
        V[k] = torch.tensor(np.asarray(a, dtype=np.float64), requires_grad=True)
        return V[k]

    def act(y, a, key):
        if a == "relu" and key in masks:
            return y * torch.as_tensor(np.asarray(masks[key], dtype=np.float64))
        return _act(y, a)

    cols = {}
    for n, t in tables.items():
        cols[n] = torch.as_tensor(np.asarray(t, dtype=np.float64)[np.asarray(batch[n]).reshape(-1)])
    for c in continuous:
        cols[c] = torch.as_tensor(np.asarray(batch[c], dtype=np.float64).reshape(-1, 1))
    for p in pretrained:
        cols[p["name"]] = slot(p["P"], p["ids"], p["proj"], p["l2"], var)
    x0 = torch.cat([cols[k] for k in sorted(cols)], dim=1)

    def chain(x, ls, tag):
        for i, l in enumerate(ls):
            x = x @ var(f"{tag}/kernel_{i}", l["kernel"])
            if l.get("bias") is not None:
                x = x + var(f"{tag}/bias_{i}", l["bias"])
            x = act(x, l.get("activation"), f"{tag}_{i}")
        return x

    if body == "dcn":
        x = x0
        for i, l in enumerate(layers["cross"]):
            x = x0 * (x @ var(f"cross/kernel_{i}", l["kernel"]) + var(f"cross/bias_{i}", l["bias"])) + x
        h = chain(x, layers["deep"], "deep")
    else:
        h = chain(x0, layers.get("bottom", []), "bottom")
        if body == "mmoe":
            ex = layers["experts"]
            X = act(h @ var("experts/kernel", ex["kernel"]) + var("experts/bias", ex["bias"]), ex["activation"], "experts")
            h = gate_mix(X, h @ var("gates/kernel", layers["gates"]), ex["E"], 1.0)
    z = (h @ var("head/kernel", head["kernel"])).reshape(-1)
    if head.get("bias") is not None:
        z = z + var("head/bias", head["bias"]).reshape(-1)
    total, _ = heads_loss([z], ["binary_crossentropy"], [targets])
    total.backward()
    grads = {k: (v.grad.numpy().copy() if v.grad is not None else np.zeros(tuple(v.shape))) for k, v in V.items()}
    return float(total.item()), z.detach().numpy().copy(), grads
