"""Golden vectors of ONE TRAINING STEP of the reference's NCF set-up on its torch modules — TEST INFRASTRUCTURE, run in the
build container where /root/reference exists:

    python tests/golden/make_golden_ncf_train.py   # writes tests/golden/ncf_train/ref_torch_ncf_train.npz

It reuses the stand-in modules of oracle/make_golden_from_reference_torch.py, as make_golden_mf_train.py does, and
executes the reference's torch modules unmodified: four EmbeddingTable(16) (userId / movieId on the ML-1M column names,
one pair per branch), MLPBlock([24, 8]) and a BinaryOutput plus a RegressionOutput.  The torch backend has no NCFModel, so
the script composes them as the TensorFlow factory (models/benchmark.py:32-100) does: the GMF product u_mf * i_mf, the MLP
over [i_mlp | u_mlp] (item first: the sorted-key concat of {"query", "item"}), the body [mf | mlp], each output's default
loss (nn.BCELoss on the sigmoid, nn.MSELoss) summed with unit loss weights, and torch.autograd.  The torch backend has no
add_loss either, so the embeddings' L2 term is not part of this fixture (tests/ncf_train_oracle.py restates it).

Stored: the batch and targets, per table the rows the batch touches with their gradient rows (the gradient of every other
row is asserted to be zero), every dense weight and gradient in Keras layout, each output's prediction and the loss.  Its
own rng: nothing else moves.
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

B, DIM, UNITS = 37, 16, (24, 8)
OUTPUTS = ("rating", "rating_binary")  # RegressionOutput, BinaryOutput: the order of OutputBlock(movielens_1m_schema())


def main():
    if not G.REF.exists():
        raise SystemExit("/root/reference is not present: golden vectors can only be regenerated in the build container")
    G.install_stand_ins()
    import torch

    import models_b200.schema as S

    embm = importlib.import_module("merlin.models.torch.inputs.embedding")
    mlpm = importlib.import_module("merlin.models.torch.blocks.mlp")
    clsm = importlib.import_module("merlin.models.torch.outputs.classification")
    regm = importlib.import_module("merlin.models.torch.outputs.regression")

    def catc(name, mx, tags):
        return S.ColumnSchema(name, tags=("categorical",) + tuple(tags), dtype="int64",
                              properties={"domain": {"min": 0, "max": mx, "name": name}})

    cols = {"query": catc("userId", 6040, ("user", "user_id")), "item": catc("movieId", 3684, ("item", "item_id"))}
    rng = np.random.default_rng(3031)
    batch = {"userId": rng.integers(1, 6041, B).astype(np.int64), "movieId": rng.integers(1, 3685, B).astype(np.int64)}
    batch["userId"][9] = batch["userId"][4]    # duplicate user -> two slices summed into one row of each user table
    batch["movieId"][11] = batch["movieId"][2]
    targets = {"rating_binary": rng.integers(0, 2, B).astype(np.float32), "rating": (rng.random(B) * 5.0).astype(np.float32)}
    targets["rating"][[5, 20]] = [9.0, -3.0]

    tables = {}
    for branch, seed in (("mf", 71), ("mlp", 72)):
        for side in ("query", "item"):
            torch.manual_seed(seed * 10 + (side == "item"))
            tables[(branch, side)] = embm.EmbeddingTable(DIM, cols[side])
    torch.manual_seed(73)
    mlp = mlpm.MLPBlock(list(UNITS))
    heads = {"rating": regm.RegressionOutput(S.Schema([S.ColumnSchema("rating", tags=("target", "regression"), dtype="float32")])),
             "rating_binary": clsm.BinaryOutput(S.ColumnSchema("rating_binary", tags=("target", "binary_classification"),
                                                               dtype="int64"))}

    def emb(branch, side):
        return tables[(branch, side)].forward_tensor(torch.from_numpy(batch[cols[side].name]))

    g = emb("mf", "query") * emb("mf", "item")
    h = mlp(torch.cat([emb("mlp", "item"), emb("mlp", "query")], dim=1))
    x = torch.cat([g, h], dim=1)
    preds = {n: heads[n](x) for n in OUTPUTS}
    loss = sum(heads[n].loss(preds[n].reshape(-1), torch.from_numpy(targets[n])) for n in OUTPUTS)
    loss.backward()

    blobs = {"loss": np.float64(loss.item())}
    for n in OUTPUTS:
        blobs[f"pred_{n}"] = preds[n].detach().numpy().reshape(-1).copy()
        blobs[f"targets_{n}"] = targets[n]
        lin = [m for m in heads[n].modules() if isinstance(m, torch.nn.Linear)]
        assert len(lin) == 1 and lin[0].weight.shape == (1, DIM + UNITS[-1])
        blobs[f"head_{n}_kernel"] = lin[0].weight.detach().numpy().T.copy()
        blobs[f"head_{n}_bias"] = lin[0].bias.detach().numpy().copy()
        blobs[f"grad_head_{n}_kernel"] = lin[0].weight.grad.detach().numpy().T.copy()
        blobs[f"grad_head_{n}_bias"] = lin[0].bias.grad.detach().numpy().copy()
    lins = [m for m in mlp.modules() if isinstance(m, torch.nn.Linear)]
    assert len(lins) == len(UNITS)
    for i, l in enumerate(lins):
        blobs[f"mlp_kernel_{i}"] = l.weight.detach().numpy().T.copy()
        blobs[f"mlp_bias_{i}"] = l.bias.detach().numpy().copy()
        blobs[f"grad_mlp_kernel_{i}"] = l.weight.grad.detach().numpy().T.copy()
        blobs[f"grad_mlp_bias_{i}"] = l.bias.grad.detach().numpy().copy()
    for (branch, side), t in tables.items():
        f = cols[side].name
        ids = np.unique(batch[f])
        w = t.table.weight
        gr = w.grad.detach().numpy()
        assert not np.any(gr[np.setdiff1d(np.arange(gr.shape[0]), ids)]), f"{branch}/{side}: gradient outside the batch's rows"
        blobs[f"{branch}_{side}_ids"] = ids
        blobs[f"{branch}_{side}_rows"] = w.detach().numpy()[ids].copy()
        blobs[f"grad_{branch}_{side}_rows"] = gr[ids].copy()

    path = G.OUT / "ncf_train" / "ref_torch_ncf_train.npz"
    path.parent.mkdir(exist_ok=True)
    np.savez(path, kind="ncf_train", dim=np.int64(DIM), units=np.array(UNITS, dtype=np.int64), outputs=np.array(OUTPUTS),
             query_col=np.array("userId"), item_col=np.array("movieId"), **{f"batch_{k}": v for k, v in batch.items()}, **blobs)
    print("wrote", path)


if __name__ == "__main__":
    main()
