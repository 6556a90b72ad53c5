"""CPU restatement of the in-batch pairwise ranking losses and of one TwoTowerModel / MatrixFactorizationModel step
trained with them — test infrastructure.

The reference computes these losses in a float32 TF graph (losses/pairwise.py:44-395): column 0 of the scores is the
positive, the other N columns the batch's items, with the row's own item (and every item with the same id) down-scored
to the constant MIN_FLOAT (utils/tf_utils.py:126-154) and then all columns divided by logits_temperature.  Per element:

    bpr       -log(eps0(sigmoid(sp - sn)))
    bpr-max   -log(eps0(sigmoid(sp - sn) w)) + reg_lambda sn^2 w,      w = softmax(sn) over the row
    top1      sigmoid(sn - sp) + sigmoid(sn^2)
    top1_v2   mean_n(sigmoid(sn - sp) + sigmoid(sn^2)) - sigmoid(sp^2) / N      (one value per row)
    top1-max  (sigmoid(sn - sp) + sigmoid(sn^2)) w
    logistic  relu(sn - sp) + log1p(eps0(exp(-|sn - sp|)))
    hinge     relu(1 + sn - sp)

eps0(x) = where(x == 0, x + 1e-24, x) (tf_utils.add_epsilon_to_zeros).  The `x == 0` test is made on the float32 value of
x, as the reference's graph makes it: a down-scored column's softmax weight exp(-655 - lse) is 0 in float32 (so its
BPR-max element is -log(1e-24) = 55.26) but 1e-285 in float64.  The loss is Keras' SUM_OVER_BATCH_SIZE: the mean over
the (B, N) elements (top1_v2: over its (B, 1) rows).  Everything else is float64 autograd.
"""
from __future__ import annotations

import copy
from typing import Dict, List, Optional

import numpy as np
import torch

from oracle.oracle_train import dense_update, sparse_update
from tests.twotower_train_oracle import MIN_FLOAT, _pool, l2_normalize, sparse_ids, tower_forward

KINDS = ("bpr", "bpr-max", "top1", "top1_v2", "top1-max", "logistic", "hinge")
EPS0_LOSS = -np.log(1e-24)  # 55.262...


def _zero32(*factors) -> torch.Tensor:
    """Whether the float32 product of the float32 values of `factors` is exactly 0 (subnormals kept)."""
    x = factors[0].detach().to(torch.float32)
    for f in factors[1:]:
        x = x * f.detach().to(torch.float32)
    return x == 0


def element_losses(sp: torch.Tensor, sn: torch.Tensor, kind: str, reg_lambda: float = 1.0) -> torch.Tensor:
    """The per-element losses (B, N) (top1_v2: (B, 1)) of the scores sp (B, 1) and sn (B, N)."""
    if kind == "bpr":
        d = sp - sn
        sig = torch.sigmoid(d)
        return torch.where(_zero32(sig), -torch.log(sig + 1e-24), torch.nn.functional.softplus(-d))
    if kind == "bpr-max":
        d = sp - sn
        sig = torch.sigmoid(d)
        w = torch.softmax(sn, dim=1)
        zero = _zero32(sig, w)
        main = torch.where(zero, -torch.log(sig * w + 1e-24), torch.nn.functional.softplus(-d) - torch.log_softmax(sn, dim=1))
        return main + reg_lambda * sn * sn * w
    if kind in ("top1", "top1_v2", "top1-max"):
        e = torch.sigmoid(sn - sp) + torch.sigmoid(sn * sn)
        if kind == "top1":
            return e
        if kind == "top1-max":
            return e * torch.softmax(sn, dim=1)
        return e.mean(dim=1, keepdim=True) - torch.sigmoid(sp * sp) / sn.shape[1]
    if kind == "logistic":
        u = sn - sp
        x = torch.exp(-torch.abs(u))
        return torch.relu(u) + torch.log1p(torch.where(_zero32(x), x + 1e-24, x))
    if kind == "hinge":
        return torch.relu(1.0 + sn - sp)
    raise ValueError(kind)


def inbatch_scores(q, pos, neg, pos_ids=None, neg_ids=None, temperature: float = 1.0, downscore: bool = True,
                   false_neg_score: float = MIN_FLOAT):
    """(sp (B, 1), sn (B, N)): the positive and the down-scored in-batch scores, divided by T after the rescoring."""
    sp = (q * pos).sum(-1, keepdim=True)
    sn = q @ neg.T
    if downscore:
        pid = torch.as_tensor(np.asarray(pos_ids).reshape(-1).astype(np.int64))
        nid = torch.as_tensor(np.asarray(neg_ids).reshape(-1).astype(np.int64))
        sn = torch.where(pid.view(-1, 1) == nid.view(1, -1), torch.full_like(sn, float(np.float32(false_neg_score))), sn)
    return sp / temperature, sn / temperature


def pairwise_loss(q, pos, neg, kind: str, pos_ids=None, neg_ids=None, temperature: float = 1.0, downscore: bool = True,
                  reg_lambda: float = 1.0, false_neg_score: float = MIN_FLOAT):
    """The mean loss of the in-batch scores of (q, pos, neg)."""
    sp, sn = inbatch_scores(q, pos, neg, pos_ids, neg_ids, temperature, downscore, false_neg_score)
    return element_losses(sp, sn, kind, reg_lambda).mean()


def loss_and_grads(batch: Dict[str, np.ndarray], towers: Dict[str, dict], item_id: str, kind: str, reg_lambda: float = 1.0,
                   temperature: float = 1.0, l2: bool = False, l2_reg: Optional[Dict[str, float]] = None,
                   downscore: bool = True, dtype=torch.float64):
    """One step of a TwoTowerModel / MatrixFactorizationModel compiled with a pairwise loss: towers as
    twotower_train_oracle.twotower_loss_and_grads, l2_reg = {"query": l2, "item": l2} the embeddings' L2 factors (the
    term of mf_train_oracle).  Returns (loss = pairwise + reg, reg, grads keyed "<tower>/table/<f>" (dense (rows, D)),
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
    ids = batch[item_id]
    loss = pairwise_loss(out["query"], out["item"], out["item"], kind, ids, ids, temperature, downscore, reg_lambda)
    reg = torch.zeros((), dtype=dtype)
    for tag, t in towers.items():
        lam = float(l2_reg.get(tag, 0.0))
        if lam:
            for f in t["tables"]:
                e = _pool(P[f"{tag}/table/{f}"], batch[f], t.get("combiner", {}).get(f, "mean"), dtype)
                reg = reg + lam * (e * e).sum()
    total = loss + reg
    total.backward()
    grads = {k: (v.grad.numpy().copy() if v.grad is not None else np.zeros(tuple(v.shape))) for k, v in P.items()}
    return float(total.item()), float(reg.item()), grads


def train_steps(batches: List[Dict[str, np.ndarray]], towers: Dict[str, dict], item_id: str, kind: str, opt: str, lr: float,
                reg_lambda: float = 1.0, temperature: float = 1.0, l2: bool = False, l2_reg: Optional[Dict[str, float]] = None,
                initial_accumulator_value: float = 0.1, **hyper):
    """Several optimizer steps with the Keras update rules (dense variables dense_update, tables sparse_update on the rows
    each batch touched).  Returns (losses, towers with the trained variables)."""
    towers = copy.deepcopy(towers)
    slots = {"sgd": [], "adagrad": ["a"], "adam": ["m", "v"]}[opt]
    init = {"a": initial_accumulator_value, "m": 0.0, "v": 0.0}
    state: Dict[str, dict] = {}
    losses = []
    for step, batch in enumerate(batches, start=1):
        loss, _, grads = loss_and_grads(batch, towers, item_id, kind, reg_lambda, temperature, l2, l2_reg)
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
                uniq = np.unique(ids[(ids >= 0) & (ids < np.shape(w)[0])].astype(np.int64))
                t["tables"][f] = sparse_update(opt, w, uniq, grads[key][uniq], st, lr, step=step, **hyper)
    return losses, towers
