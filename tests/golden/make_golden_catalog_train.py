"""Golden vectors of ONE TRAINING STEP of a weight-tied next-item classifier built from the reference's torch modules — TEST
INFRASTRUCTURE, run in the build container where /root/reference exists:

    python tests/golden/make_golden_catalog_train.py   # writes tests/golden/catalog_train/ref_torch_catalog_train.npz

It reuses the stand-in modules of oracle/make_golden_from_reference_torch.py.  The reference's torch backend has no
model-level sequential form for this case, so the step is composed from its module files, executed unmodified, and
differentiated by torch autograd:

    inputs/embedding.py EmbeddingTable   the user table (forward_tensor) and the item table, which the fixed-length item
                                          history reads through forward_bag (F.embedding_bag, mean)
    blocks/mlp.py MLPBlock([24, 16])      its MaybeAgg(Concat()) concatenates the features in sorted-name order
    outputs/classification.py EmbeddingTablePrediction   logits = x E^T + b over the SAME item table (weight tying)
    transforms/bias.py LogitsTemperatureScaler(T)        logits / T
    torch.nn.CrossEntropyLoss(reduction="none")          per row, weighted by sample_weight, summed and divided by B
                                                          (Keras' sample-weighted mean)

The item table's gradient therefore sums its two paths (the history's lookups and the output product).  The batch repeats
item ids within and across rows, T = 0.05 and the bias is non-zero.  Stored: the batch, the labels and sample weights,
every weight (kernels in Keras (in, out) layout), the loss and every gradient.  Its own rng: nothing else moves.  Checked by
tests/test_catalog_model_host.py (the restatement) and tests/test_gpu_catalog_model.py (the CUDA step).
"""
from __future__ import annotations

import importlib
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import make_golden_from_reference_torch as G  # noqa: E402

N_ITEMS, N_USERS, D, L, B, T = 60, 50, 16, 4, 37, 0.05


def main():
    if not G.REF.exists():
        raise SystemExit("/root/reference is not present: golden vectors can only be regenerated in the build container")
    G.install_stand_ins()
    import torch

    import models_b200.schema as S

    emb = importlib.import_module("merlin.models.torch.inputs.embedding")
    mlpm = importlib.import_module("merlin.models.torch.blocks.mlp")
    clsm = importlib.import_module("merlin.models.torch.outputs.classification")
    bias_mod = importlib.import_module("merlin.models.torch.transforms.bias")
    rng = np.random.default_rng(2026)
    torch.manual_seed(31)
    item_col = S.ColumnSchema("item_id", tags=("categorical", "item_id"), dtype="int64",
                              properties={"domain": {"min": 0, "max": N_ITEMS - 1, "name": "item_id"}})
    user_col = S.ColumnSchema("user_id", tags=("categorical", "user_id"), dtype="int64",
                              properties={"domain": {"min": 0, "max": N_USERS - 1, "name": "user_id"}})
    items = emb.EmbeddingTable(D, S.Schema([item_col]), seq_combiner="mean")
    users = emb.EmbeddingTable(D, S.Schema([user_col]))
    mlp = mlpm.MLPBlock([24, D])
    pred = clsm.EmbeddingTablePrediction(items)
    scale = bias_mod.LogitsTemperatureScaler(T)
    with torch.no_grad():  # a small, non-zero start: the soft-max is not saturated at T = 0.05
        items.table.weight.copy_(torch.from_numpy((rng.standard_normal((N_ITEMS, D)) * 0.1).astype(np.float32)))
        users.table.weight.copy_(torch.from_numpy((rng.standard_normal((N_USERS, D)) * 0.3).astype(np.float32)))
        pred.bias.copy_(torch.from_numpy((rng.standard_normal(N_ITEMS) * 0.3).astype(np.float32)))

    hist = rng.integers(0, N_ITEMS, (B, L)).astype(np.int64)
    hist[rng.random((B, L)) < 0.4] = 3  # a popular item: duplicates within and across rows
    batch = {"user_id": rng.integers(0, N_USERS, B).astype(np.int64), "item_history": hist,
             "c1": rng.standard_normal(B).astype(np.float32), "c2": rng.standard_normal(B).astype(np.float32)}
    labels = rng.integers(0, N_ITEMS, B).astype(np.int64)
    labels[:3] = [3, 0, N_ITEMS - 1]
    sw = rng.uniform(0.2, 2.0, B).astype(np.float32)

    feats = {"user_id": users.forward_tensor(torch.from_numpy(batch["user_id"])),
             "item_history": items.forward_bag(torch.from_numpy(hist)),
             "c1": torch.from_numpy(batch["c1"]), "c2": torch.from_numpy(batch["c2"])}
    x = mlp(feats)
    logits = scale(pred(x))
    per = torch.nn.CrossEntropyLoss(reduction="none")(logits, torch.from_numpy(labels))
    loss = (per * torch.from_numpy(sw)).sum() / B
    loss.backward()

    lins = [m for m in mlp.modules() if isinstance(m, torch.nn.Linear)]
    acts = [type(m).__name__ for m in mlp.modules() if isinstance(m, torch.nn.ReLU)]
    assert len(lins) == 2 and len(acts) == 2, (lins, acts)
    assert pred.embeddings() is items.table.weight  # weight tying: one Parameter, both paths in its .grad
    blobs = {}
    for i, l in enumerate(lins):
        blobs[f"mlp_kernel_{i}"] = l.weight.detach().numpy().T.copy()
        blobs[f"mlp_bias_{i}"] = l.bias.detach().numpy().copy()
        blobs[f"grad_mlp_kernel_{i}"] = l.weight.grad.detach().numpy().T.copy()
        blobs[f"grad_mlp_bias_{i}"] = l.bias.grad.detach().numpy().copy()
    path = G.OUT / "catalog_train" / "ref_torch_catalog_train.npz"
    path.parent.mkdir(exist_ok=True)
    np.savez(path, kind="catalog_train", n_items=np.int64(N_ITEMS), n_users=np.int64(N_USERS), dim=np.int64(D),
             hist_len=np.int64(L), temperature=np.float32(T), labels=labels, sample_weight=sw, loss=np.float32(loss.item()),
             query=x.detach().numpy(), table_item_id=items.table.weight.detach().numpy().copy(),
             table_user_id=users.table.weight.detach().numpy().copy(), bias=pred.bias.detach().numpy().copy(),
             grad_table_item_id=items.table.weight.grad.detach().numpy().copy(),
             grad_table_user_id=users.table.weight.grad.detach().numpy().copy(), grad_bias=pred.bias.grad.detach().numpy().copy(),
             **{f"batch_{k}": v for k, v in batch.items()}, **blobs)
    print("wrote", path)


if __name__ == "__main__":
    main()
