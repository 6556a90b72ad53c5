"""CPU restatement of one DeepFM training step — test infrastructure.

Forward of DeepFMModel (models/ranking.py:171-279, blocks/interaction.py:256-332) in float64 with autograd, as
oracle.deepfm_forward computes it:
  e_f = the table row of feature f's id (a zero row for an id outside [0, rows)), S_f = sum_d e_f[d]
  pair = sum_f 0.5 (S_f^2 - sum_d e_f[d]^2)                  (the reference's axis: per feature over D, then summed)
  wide = sum_f Wk[off_f + id_f] + sum_c Wk[off_c] x_c + bw     (ids outside [0, rows) contribute nothing)
  deep = deep_logit(deep(x0)), x0 = [rows | continuous columns] in sorted-name order
  s = pair + wide + deep;  z = s w_out + b_out
and the loss of the one output: BCE on the logit (BinaryOutput) or squared error (RegressionOutput), times the sample
weight, summed over the batch and divided by B.  The updates are oracle/oracle_train.py's Keras rules.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from oracle.oracle_train import _act

BCE, MSE = "binary_crossentropy", "mse"


def deepfm_loss_and_grads(batch: Dict[str, np.ndarray], tables: Dict[str, np.ndarray], continuous: Sequence[str],
                          wide_offsets: Dict[str, int], wide_kernel: np.ndarray, wide_bias: Optional[np.ndarray], deep: List[dict],
                          deep_logit: List[dict], head: dict, targets: np.ndarray, sample_weight=None, dtype=torch.float64):
    """tables: feature -> (rows, D); wide_offsets: feature or continuous column -> first row in the wide kernel;
    deep / deep_logit: [{"kernel", "bias" (or None), "activation"}]; head: {"kernel" (1, 1), "bias", "loss"}.
    Returns (loss, z (B,), grads keyed "table/<f>", "wide/kernel", "wide/bias", "deep/kernel_i", "deep/bias_i",
    "deep_logit/kernel_i", "deep_logit/bias_i", "head/kernel", "head/bias")."""

    def var(x):
        return torch.tensor(np.asarray(x, dtype=np.float64), dtype=dtype, requires_grad=True)

    P = {f"table/{n}": var(t) for n, t in tables.items()}
    P["wide/kernel"] = var(wide_kernel)
    if wide_bias is not None:
        P["wide/bias"] = var(wide_bias)
    for tag, layers in (("deep", deep), ("deep_logit", deep_logit)):
        for i, l in enumerate(layers):
            P[f"{tag}/kernel_{i}"] = var(l["kernel"])
            if l.get("bias") is not None:
                P[f"{tag}/bias_{i}"] = var(l["bias"])
    P["head/kernel"] = var(head["kernel"])
    if head.get("bias") is not None:
        P["head/bias"] = var(head["bias"])

    wk = P["wide/kernel"].reshape(-1)
    cols, pair, wide = {}, 0.0, 0.0
    for n in tables:
        w = P[f"table/{n}"]
        ids = torch.as_tensor(np.asarray(batch[n]).reshape(-1).astype(np.int64))
        ok = (ids >= 0) & (ids < w.shape[0])
        e = w[ids.clamp(0, w.shape[0] - 1)] * ok.to(dtype).unsqueeze(1)
        cols[n] = e
        S = e.sum(1)
        pair = pair + 0.5 * (S * S - (e * e).sum(1))
        wide = wide + wk[(ids.clamp(0, w.shape[0] - 1) + int(wide_offsets[n]))] * ok.to(dtype)
    for n in continuous:
        x = torch.as_tensor(np.asarray(batch[n], dtype=np.float64).reshape(-1)).to(dtype)
        cols[n] = x.reshape(-1, 1)
        wide = wide + wk[int(wide_offsets[n])] * x
    if "wide/bias" in P:
        wide = wide + P["wide/bias"].reshape(())
    x0 = torch.cat([cols[n] for n in sorted(cols)], dim=1)

    def dense(x, tag, i, act):
        x = x @ P[f"{tag}/kernel_{i}"]
        if f"{tag}/bias_{i}" in P:
            x = x + P[f"{tag}/bias_{i}"]
        return _act(x, act)

    h = x0
    for tag, layers in (("deep", deep), ("deep_logit", deep_logit)):
        for i, l in enumerate(layers):
            h = dense(h, tag, i, l.get("activation"))
    s = pair + wide + h.reshape(-1)
    z = s * P["head/kernel"].reshape(())
    if "head/bias" in P:
        z = z + P["head/bias"].reshape(())
    y = torch.as_tensor(np.asarray(targets, dtype=np.float64).reshape(-1)).to(dtype)
    if head["loss"] == BCE:
        per = torch.clamp(z, min=0) - z * y + torch.log1p(torch.exp(-z.abs()))
    elif head["loss"] == MSE:
        per = (z - y) ** 2
    else:
        raise ValueError(head["loss"])
    if sample_weight is not None:
        per = per * torch.as_tensor(np.asarray(sample_weight, dtype=np.float64).reshape(-1)).to(dtype)
    loss = per.sum() / y.shape[0]
    loss.backward()
    grads = {k: (v.grad.numpy().copy() if v.grad is not None else np.zeros(tuple(v.shape))) for k, v in P.items()}
    return float(loss.item()), z.detach().numpy().copy(), grads
