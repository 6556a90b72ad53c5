"""CPU restatement of one NCFModel training step — test infrastructure.

In float64 with autograd, as the reference's NCFModel (models/benchmark.py:32-100) computes it:
    g = u_mf * i_mf,  h = mlp([i_mlp | u_mlp]),  z_t = [g | h] . w_t + b_t
    loss = sum_t lambda_t mean_b(sw l_t) + reg,  reg = l2 sum_b (|u_mf|^2 + |i_mf|^2 + |u_mlp|^2 + |i_mlp|^2)
The torch backend has no add_loss, so the L2 term (inputs/embedding.py:1108-1113, added to the loss through model.losses)
is restated here.  The updates are oracle/oracle_train.py's Keras rules.
"""
from __future__ import annotations

import copy
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from oracle.oracle_train import dense_update, sparse_update
from tests.mmoe_oracle import heads_loss

TABLES = ("mf/query", "mf/item", "mlp/query", "mlp/item")


def ncf_loss_and_grads(ids: Dict[str, np.ndarray], p: dict, losses: Sequence[str], targets, loss_weights=None,
                       sample_weight=None, l2: float = 0.0, dtype=torch.float64):
    """ids {"query", "item"}: (B,) row ids of both sides (shared by both branches); p: {"mf/query", "mf/item", "mlp/query",
    "mlp/item": tables, "layers": [{kernel, bias, act}], "head_kernel" (D + U, H), "head_bias" (H,)}.  An id outside a
    table reads a zero row.  Returns (loss, reg, [loss_t], z (H, B), grads keyed as p: dense (rows, D) for tables,
    "kernel_i" / "bias_i", "head_kernel", "head_bias")."""
    P = {k: torch.tensor(np.asarray(p[k], dtype=np.float64), dtype=dtype, requires_grad=True) for k in TABLES}
    for i, l in enumerate(p["layers"]):
        P[f"kernel_{i}"] = torch.tensor(np.asarray(l["kernel"], dtype=np.float64), dtype=dtype, requires_grad=True)
        P[f"bias_{i}"] = torch.tensor(np.asarray(l["bias"], dtype=np.float64), dtype=dtype, requires_grad=True)
    P["head_kernel"] = torch.tensor(np.asarray(p["head_kernel"], dtype=np.float64), dtype=dtype, requires_grad=True)
    P["head_bias"] = torch.tensor(np.asarray(p["head_bias"], dtype=np.float64), dtype=dtype, requires_grad=True)

    def rows(key, side):
        w = P[key]
        i = torch.as_tensor(np.asarray(ids[side]).reshape(-1).astype(np.int64))
        ok = (i >= 0) & (i < w.shape[0])
        return w[i.clamp(0, w.shape[0] - 1)] * ok.to(dtype).unsqueeze(1)

    e = {k: rows(k, k.split("/")[1]) for k in TABLES}
    g = e["mf/query"] * e["mf/item"]
    x = torch.cat([e["mlp/item"], e["mlp/query"]], dim=1)
    for i, l in enumerate(p["layers"]):
        x = x @ P[f"kernel_{i}"] + P[f"bias_{i}"]
        if l.get("act", "relu") == "relu":
            x = torch.relu(x)
    z = torch.cat([g, x], dim=1) @ P["head_kernel"] + P["head_bias"]
    total, per = heads_loss([z[:, t] for t in range(z.shape[1])], losses, targets, loss_weights, sample_weight)
    reg = float(l2) * sum((v * v).sum() for v in e.values())
    loss = total + reg
    loss.backward()
    grads = {k: (v.grad.numpy().copy() if v.grad is not None else np.zeros(tuple(v.shape))) for k, v in P.items()}
    return (float(loss.item()), float(reg.detach()), [float(v.detach()) for v in per], z.detach().numpy().T.copy(), grads)


def ncf_train_steps(batches: List[dict], p: dict, losses: Sequence[str], opt: str, lr: float, l2: float = 0.0,
                    loss_weights=None, initial_accumulator_value: float = 0.1, **hyper):
    """Several optimizer steps; batches: dicts with "ids" ({"query", "item"}) and "targets" (one per head).  The tables take
    sparse_update on the rows each batch touched, the Dense variables dense_update.  Returns ([loss per step], params)."""
    p = copy.deepcopy(p)
    slots = {"sgd": [], "adagrad": ["a"], "adam": ["m", "v"]}[opt]
    init = {"a": initial_accumulator_value, "m": 0.0, "v": 0.0}
    state: Dict[str, dict] = {}
    out = []
    for step, bt in enumerate(batches, start=1):
        loss, _, _, _, grads = ncf_loss_and_grads(bt["ids"], p, losses, bt["targets"], loss_weights, l2=l2)
        out.append(loss)
        for k in TABLES:
            st = state.setdefault(k, {s: np.full(np.shape(p[k]), init[s]) for s in slots})
            i = np.asarray(bt["ids"][k.split("/")[1]]).reshape(-1).astype(np.int64)
            uniq = np.unique(i[(i >= 0) & (i < np.shape(p[k])[0])])
            p[k] = sparse_update(opt, p[k], uniq, grads[k][uniq], st, lr, step=step, **hyper)
        dense = [(f"kernel_{i}", p["layers"][i], "kernel") for i in range(len(p["layers"]))]
        dense += [(f"bias_{i}", p["layers"][i], "bias") for i in range(len(p["layers"]))]
        dense += [("head_kernel", p, "head_kernel"), ("head_bias", p, "head_bias")]
        for key, holder, name in dense:
            st = state.setdefault(key, {s: np.full(np.shape(holder[name]), init[s]) for s in slots})
            holder[name] = dense_update(opt, holder[name], grads[key], st, lr, step=step, **hyper)
    return out, p


def model_params(model) -> dict:
    """The parameters of an NCFModel as ncf_loss_and_grads reads them (host float64 copies)."""
    body = model.body
    f64 = lambda t: t.detach().cpu().numpy().astype(np.float64)  # noqa: E731
    p = {f"{b}/{s}": f64(body.table(b, s).embeddings) for b in ("mf", "mlp") for s in ("query", "item")}
    p["layers"] = [dict(kernel=f64(l.kernel), bias=f64(l.bias), act=l.activation) for l in body.mlp.dense_layers]
    head = model.prediction.to_call
    p["head_kernel"], p["head_bias"] = f64(head.kernel), f64(head.bias)
    return p


def golden_inputs(z):
    """(ids, params, targets, losses) of the NCF fixture (tests/golden/ncf_train/ref_torch_ncf_train.npz): tables holding
    only the rows the batch touches, the batch's ids remapped to those rows (both branches share the remap, since they
    look up the same ids), the heads stacked in the fixture's output order."""
    q, it = str(z["query_col"]), str(z["item_col"])
    ids = {"query": np.searchsorted(z["mf_query_ids"], z[f"batch_{q}"]), "item": np.searchsorted(z["mf_item_ids"], z[f"batch_{it}"])}
    p = {f"{b}/{s}": z[f"{b}_{s}_rows"] for b in ("mf", "mlp") for s in ("query", "item")}
    p["layers"] = [dict(kernel=z[f"mlp_kernel_{i}"], bias=z[f"mlp_bias_{i}"], act="relu") for i in range(len(z["units"]))]
    outs = [str(n) for n in z["outputs"]]
    p["head_kernel"] = np.concatenate([z[f"head_{n}_kernel"] for n in outs], axis=1)
    p["head_bias"] = np.concatenate([z[f"head_{n}_bias"] for n in outs])
    losses = ["mse" if n == "rating" else "binary_crossentropy" for n in outs]
    return ids, p, [z[f"targets_{n}"] for n in outs], losses
