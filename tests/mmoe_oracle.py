"""CPU restatement of the multi-task Model(InputBlockV2, [MLPBlock], [MMOEBlock], output) — test infrastructure.

float64 torch autograd over the TensorFlow semantics (blocks/experts.py:37-208, outputs/block.py:32-190):
  * x0: the input block's concat of embedding rows (multi-hot features pooled by tests/multihot_oracle.pool) and continuous
    columns in sorted-name order; then the shared bottom's Dense layers;
  * expert e (stacked order = sorted expert names): act(x W_e + b_e) (U wide);
  * gate t (output order): p_t = softmax(gate_t(x) / T) with gate_t = x G_t, or gate_block_t then gate_final_t;
    m_t = sum_e p_t,e expert_e;
  * tower t (optional): task_block_t(m_t) (without experts: task_block_t of the bottom's output);
  * head t: z_t = tower_t . w_t + b_t (without towers m_t, without experts the bottom's output); BinaryOutput BCE on the logit,
    RegressionOutput (z - y)^2; loss_t = sum_i sw_i l_t,i / B; total = sum_t lambda_t loss_t.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from oracle.oracle_train import _act
from tests.multihot_oracle import pool

BCE, MSE = "binary_crossentropy", "mse"


def gate_mix(X: torch.Tensor, L: torch.Tensor, E: int, T: float) -> torch.Tensor:
    """(B, U) mixture of the E experts X (B, E U) under the gate logits L (B, E)."""
    B = X.shape[0]
    p = torch.softmax(L / T, dim=1)
    return (p.unsqueeze(2) * X.reshape(B, E, -1)).sum(1)


def heads_loss(zs: Sequence[torch.Tensor], losses: Sequence[str], targets, loss_weights=None, sample_weight=None):
    """(total, [loss_t]) of the logits zs[t] (B,); targets and sample weights as numpy arrays or tensors (on any device)."""
    H = len(zs)
    lws = [1.0] * H if loss_weights is None else [float(v) for v in loss_weights]
    sws = list(sample_weight) if isinstance(sample_weight, (list, tuple)) else [sample_weight] * H
    like = lambda v, z: (v.reshape(-1).to(z) if isinstance(v, torch.Tensor)  # noqa: E731
                         else torch.as_tensor(np.asarray(v, dtype=np.float64).reshape(-1)).to(z))
    total, per = None, []
    for z, l, y_np, sw, lw in zip(zs, losses, targets, sws, lws):
        y = like(y_np, z)
        # max(z, 0) as (z + |z|) / 2: the same value, and at z = 0 (a dead tower's output times the head kernel plus a zero
        # bias) the derivative sigmoid(0) - y the kernels compute, where clamp's sub-gradient would give 1 - y
        term = (z + z.abs()) / 2 - z * y + torch.log1p(torch.exp(-z.abs())) if l == BCE else (z - y) ** 2
        if sw is not None:
            term = term * like(sw, z)
        lt = term.sum() / y.shape[0]
        total = lw * lt if total is None else total + lw * lt
        per.append(lt)
    return total, per


def mmoe_loss_and_grads(batch: Dict[str, np.ndarray], tables: Dict[str, np.ndarray], continuous: Sequence[str],
                        bottom: List[dict], experts: Optional[List[dict]], gates: Optional[List[np.ndarray]], temperature: float,
                        heads: List[dict], targets: Sequence[np.ndarray], loss_weights=None, sample_weight=None,
                        combiners: Optional[Dict[str, str]] = None, masks: Optional[Dict[str, np.ndarray]] = None,
                        towers: Optional[List[List[dict]]] = None):
    """tables {feature: (rows, D)}; bottom / experts: [{"kernel", "bias" or None, "activation"}], experts in stacked order;
    gates[t] in output order: a (K, E) kernel, or a list of layers (gate_block's, then gate_final); towers[t]: the layers of
    output t's tower; heads[t] {"kernel" (K, 1), "bias" (1,) or None, "loss"}.  Returns (total, [loss_t], [z_t (B,)], grads)
    with grads keyed "table/<f>", "bottom/kernel_i", "bottom/bias_i", "expert/kernel_e", "expert/bias_e", "gate/kernel_t"
    (or "gate_t/kernel_i", "gate_t/bias_i"), "tower_t/kernel_i", "tower_t/bias_i", "head/kernel_t", "head/bias_t".

    masks {"bottom_i": (B, units), "experts": (B, E U), "gate_t_i", "tower_t_i"} (optional): where a relu layer passes its input, as the device decided
    it.  A pre-activation within float32 rounding of 0 can take either side of the kink; with the device's decisions the
    restatement's gradients follow the same branch (relu(y) and y * mask differ only at such values)."""
    P = {}
    masks = masks or {}

    def act(y, a, key):
        if a == "relu" and key in masks:
            return y * torch.as_tensor(np.asarray(masks[key], dtype=np.float64))
        return _act(y, a)

    def var(k, a):
        P[k] = torch.tensor(np.asarray(a, dtype=np.float64), requires_grad=True)
        return P[k]

    for n, t in tables.items():
        var(f"table/{n}", t)
    cols = {n: pool(batch, n, P[f"table/{n}"], (combiners or {}).get(n, "mean")) for n in tables}
    for c in continuous:
        cols[c] = torch.as_tensor(np.asarray(batch[c], dtype=np.float64).reshape(-1, 1))
    x = torch.cat([cols[k] for k in sorted(cols)], dim=1)
    def chain(x, layers, tag, mtag):
        for i, l in enumerate(layers):
            x = x @ var(f"{tag}/kernel_{i}", l["kernel"])
            if l.get("bias") is not None:
                x = x + var(f"{tag}/bias_{i}", l["bias"])
            x = act(x, l.get("activation"), f"{mtag}_{i}")
        return x

    x = chain(x, bottom, "bottom", "bottom")
    if experts is not None:
        outs = []
        for e, l in enumerate(experts):
            y = x @ var(f"expert/kernel_{e}", l["kernel"])
            if l.get("bias") is not None:
                y = y + var(f"expert/bias_{e}", l["bias"])
            outs.append(y)
        X = act(torch.cat(outs, dim=1), experts[0].get("activation"), "experts")
        gl = [chain(x, g, f"gate_{t}", f"gate_{t}") if isinstance(g, list) else x @ var(f"gate/kernel_{t}", g)
              for t, g in enumerate(gates)]
        bodies = [gate_mix(X, L, len(experts), temperature) for L in gl]
    else:
        bodies = [x] * len(heads)
    if towers is not None:
        bodies = [chain(m, tw, f"tower_{t}", f"tower_{t}") for t, (m, tw) in enumerate(zip(bodies, towers))]
    zs = []
    for t, (hd, m) in enumerate(zip(heads, bodies)):
        z = (m @ var(f"head/kernel_{t}", hd["kernel"])).reshape(-1)
        if hd.get("bias") is not None:
            z = z + var(f"head/bias_{t}", hd["bias"]).reshape(-1)
        zs.append(z)
    total, per = heads_loss(zs, [hd["loss"] for hd in heads], targets, loss_weights, sample_weight)
    total.backward()
    grads = {k: (v.grad.numpy().copy() if v.grad is not None else np.zeros(tuple(v.shape))) for k, v in P.items()}
    return float(total.item()), [float(p.item()) for p in per], [z.detach().numpy().copy() for z in zs], grads


def model_arrays(model) -> dict:
    """The restatement's arguments (tables, continuous, bottom, experts, gates, temperature, heads) read from a built
    model: the experts and gates as the stacked layers' column blocks."""
    body, outs = model.body, model.output_blocks()
    ib = body.input_block
    emb = ib.embeddings
    np_ = lambda t: None if t is None else t.detach().cpu().numpy().astype(np.float64)
    tables = {f: np_(emb.feature_to_table[f].table) for f in emb.feature_names} if emb is not None else {}
    cont = sorted(ib.continuous.features) if ib.continuous is not None else []
    bottom = [] if body.bottom is None else [{"kernel": np_(l.kernel), "bias": np_(l.bias), "activation": l.activation}
                                             for l in body.bottom.dense_layers]
    head = model.prediction.to_call
    W, b = np_(head.kernel), np_(head.bias)
    heads = [{"kernel": W[:, t:t + 1], "bias": None if b is None else b[t:t + 1], "loss": o.loss} for t, o in enumerate(outs)]
    layers = lambda ls: [{"kernel": np_(l.kernel), "bias": np_(l.bias), "activation": l.activation} for l in ls]
    from models_b200.models import output_towers

    tw = output_towers(model.prediction)
    towers = None if tw is None else [layers(t.dense_layers) for t in tw]
    experts = gates = None
    T = 1.0
    mo = body.mmoe
    if mo is not None:
        U, E = mo.units, mo.num_experts
        K, Bx = np_(mo.experts.kernel), np_(mo.experts.bias)
        experts = [{"kernel": K[:, e * U:(e + 1) * U], "bias": None if Bx is None else Bx[e * U:(e + 1) * U],
                    "activation": mo.experts.activation} for e in range(E)]
        if mo.gates is not None:
            G = np_(mo.gates.kernel)
            gates = [G[:, t * E:(t + 1) * E] for t in range(mo.num_gates)]
        else:
            gates = [layers(mo.gate_chain(t)) for t in range(mo.num_gates)]
        T = mo.temperature
    return dict(tables=tables, continuous=cont, bottom=bottom, experts=experts, gates=gates, temperature=T, heads=heads,
                towers=towers)
