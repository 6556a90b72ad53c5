"""CPU restatement of one MatrixFactorizationModel training step — test infrastructure.

The step of tests/twotower_train_oracle.py (towers without layers are the concat of their pooled embeddings) plus the
embeddings' L2 term of the reference (inputs/embedding.py:1108-1113, added to the loss through model.losses):
    reg  = sum_tower l2_tower sum_f sum_b ||e_f,b||^2     (e_f,b: feature f's looked-up / pooled row of sample b)
    loss = CE + reg;   d reg / d e_f,b = 2 l2_tower e_f,b
in float64 with autograd.  The updates are oracle/oracle_train.py's Keras rules.
"""
from __future__ import annotations

import copy
from typing import Dict, List, Optional

import numpy as np
import torch

from oracle.oracle_train import sparse_update
from tests.twotower_train_oracle import MIN_FLOAT, _pool, inbatch_ce, l2_normalize, sparse_ids, tower_forward


def mf_loss_and_grads(batch: Dict[str, np.ndarray], towers: Dict[str, dict], item_id: str, temperature: float = 1.0,
                      l2: bool = False, l2_reg: Optional[Dict[str, float]] = None, downscore: bool = True,
                      false_neg_score: float = MIN_FLOAT, dtype=torch.float64):
    """towers as twotower_train_oracle.twotower_loss_and_grads; l2_reg = {"query": l2, "item": l2} (missing: 0).
    Returns (loss = CE + reg, reg, {"query", "item"} outputs, grads keyed "<tower>/table/<f>" (dense (rows, D)),
    "<tower>/kernel_i", "<tower>/bias_i")."""
    l2_reg = l2_reg or {}
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
    ce = inbatch_ce(out["query"], out["item"], batch[item_id], temperature, downscore, false_neg_score)
    reg = torch.zeros((), dtype=dtype)
    for tag, t in towers.items():
        lam = float(l2_reg.get(tag, 0.0))
        for f in t["tables"]:
            e = _pool(P[f"{tag}/table/{f}"], batch[f], t.get("combiner", {}).get(f, "mean"), dtype)
            reg = reg + lam * (e * e).sum()
    loss = ce + reg
    loss.backward()
    grads = {k: (v.grad.numpy().copy() if v.grad is not None else np.zeros(tuple(v.shape))) for k, v in P.items()}
    return float(loss.item()), float(reg.item()), {k: v.detach().numpy().copy() for k, v in out.items()}, grads


def mf_train_steps(batches: List[Dict[str, np.ndarray]], towers: Dict[str, dict], item_id: str, opt: str, lr: float,
                   temperature: float = 1.0, l2: bool = False, l2_reg: Optional[Dict[str, float]] = None,
                   initial_accumulator_value: float = 0.1, **hyper):
    """Several optimizer steps of tower-less towers: every table takes sparse_update on the rows each batch touched.
    Returns ([(loss, reg)] per step, towers with the trained tables)."""
    towers = copy.deepcopy(towers)
    slots = {"sgd": [], "adagrad": ["a"], "adam": ["m", "v"]}[opt]
    init = {"a": initial_accumulator_value, "m": 0.0, "v": 0.0}
    state: Dict[str, dict] = {}
    losses = []
    for step, batch in enumerate(batches, start=1):
        loss, reg, _, grads = mf_loss_and_grads(batch, towers, item_id, temperature, l2, l2_reg)
        losses.append((loss, reg))
        for tag, t in towers.items():
            assert not t["layers"], "mf_train_steps trains tower-less towers"
            for f, w in t["tables"].items():
                key = f"{tag}/table/{f}"
                st = state.setdefault(key, {s: np.full(np.shape(w), init[s]) for s in slots})
                ids = sparse_ids(batch[f])
                uniq = np.unique(ids[(ids >= 0) & (ids < np.shape(w)[0])].astype(np.int64))
                t["tables"][f] = sparse_update(opt, w, uniq, grads[key][uniq], st, lr, step=step, **hyper)
    return losses, towers


def golden_inputs(z):
    """(batch, towers, ids) of the matrix factorization fixture (tests/golden/mf_train/ref_torch_mf_train.npz): tables
    holding only the rows the batch touches, ids[(tower, f)] mapping them back, the batch's ids remapped to row positions."""
    raw = {k[len("batch_"):]: z[k] for k in z.files if k.startswith("batch_")}
    towers, ids, batch = {}, {}, {}
    for tag in ("query", "item"):
        f = str(z[f"{tag}_cols"][0])
        ids[(tag, f)] = z[f"{tag}_table_{f}_ids"]
        batch[f] = np.searchsorted(ids[(tag, f)], raw[f])
        towers[tag] = {"tables": {f: z[f"{tag}_table_{f}_rows"]}, "combiner": {f: "mean"}, "continuous": [], "layers": []}
    return batch, towers, ids
