"""Golden vectors of ONE TRAINING STEP of the reference's torch matrix factorization set-up — TEST INFRASTRUCTURE, run in
the build container where /root/reference exists:

    python tests/golden/make_golden_mf_train.py   # writes tests/golden/mf_train/ref_torch_mf_train.npz

It reuses the stand-in modules of oracle/make_golden_from_reference_torch.py, as tests/golden/make_golden_twotower_train.py
does, and executes the reference's torch modules unmodified: per tower a TabularInputBlock with EmbeddingTables(16) over
one id column (userId / movieId on the ML-1M column names) and no MLP — QueryItemIdsEmbeddingsBlock's towers are the
id embeddings themselves; InBatchNegativeSampler; ContrastiveOutput.contrastive_outputs with false-negative rescoring by
movieId (a duplicated movieId puts one accidental hit off the diagonal); LogitsTemperatureScaler; F.cross_entropy against
class 0 and torch.autograd.  Two variants on the same tables and batch: T = 1 and T = 0.5.  The torch backend has no
add_loss, so the embeddings' L2 term is not part of this fixture (tests/mf_train_oracle.py restates it).

Stored: the batch, per table the rows the batch touches with their gradient rows (the gradient of every other row is
asserted to be zero), the loss and both towers' outputs.  Its own rng: nothing else moves.
"""
from __future__ import annotations

import importlib
import sys
import types
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import make_golden_from_reference_torch as G  # noqa: E402

B, DIM = 41, 16
TEMPERATURES = (1.0, 0.5)


def main():
    if not G.REF.exists():
        raise SystemExit("/root/reference is not present: golden vectors can only be regenerated in the build container")
    G.install_stand_ins()
    import torch
    import torch.nn.functional as F

    import models_b200.schema as S

    tab = importlib.import_module("merlin.models.torch.inputs.tabular")
    embm = importlib.import_module("merlin.models.torch.inputs.embedding")
    importlib.import_module("merlin.models.torch.blocks.mlp")  # registers the "concat" aggregation TabularInputBlock uses
    con = importlib.import_module("merlin.models.torch.outputs.contrastive")
    bias_mod = importlib.import_module("merlin.models.torch.transforms.bias")
    sampler = importlib.import_module("merlin.models.torch.outputs.sampling.in_batch").InBatchNegativeSampler()
    MINF = float(np.finfo(np.float16).min) / 100.0  # utils/constants.py:19 under NumPy 1.x

    def catc(name, mx, tags):
        return S.ColumnSchema(name, tags=("categorical",) + tuple(tags), dtype="int64",
                              properties={"domain": {"min": 0, "max": mx, "name": name}})

    q_cols = [catc("userId", 6040, ("user", "user_id"))]
    i_cols = [catc("movieId", 3684, ("item", "item_id"))]

    def tower_init(block):
        block.add_route(S.Tags.CATEGORICAL, embm.EmbeddingTables(DIM))

    rng = np.random.default_rng(2027)
    batch = {"userId": rng.integers(1, 6041, B).astype(np.int64), "movieId": rng.integers(1, 3685, B).astype(np.int64)}
    batch["movieId"][5] = batch["movieId"][3]  # duplicate item -> an accidental hit off the diagonal
    batch["userId"][7] = batch["userId"][2]    # duplicate user -> two slices summed into one table row

    towers = {}
    for tag, cols_t, seed in (("query", q_cols, 51), ("item", i_cols, 52)):
        torch.manual_seed(seed)
        inp = tab.TabularInputBlock(S.Schema(cols_t), init=tower_init, agg="concat")
        feed = {k: torch.from_numpy(v) for k, v in batch.items() if k == cols_t[0].name}
        inp(feed)  # lazy modules are built by the first call
        embs = [m for m in inp.modules() if isinstance(m, torch.nn.Embedding)]
        assert len(embs) == 1 and embs[0].weight.shape[1] == DIM
        towers[tag] = dict(inp=inp, feed=feed, emb=embs[0], f=cols_t[0].name)

    blobs = {}
    for tag, t in towers.items():
        ids = np.unique(batch[t["f"]])
        blobs[f"{tag}_table_{t['f']}_rows_total"] = np.int64(t["emb"].weight.shape[0])
        blobs[f"{tag}_table_{t['f']}_ids"] = ids
        blobs[f"{tag}_table_{t['f']}_rows"] = t["emb"].weight.detach().numpy()[ids].copy()

    for T in TEMPERATURES:
        vt = f"T{T:g}".replace(".", "p")
        for t in towers.values():
            t["inp"].zero_grad()
        qo = towers["query"]["inp"](towers["query"]["feed"])
        io = towers["item"]["inp"](towers["item"]["feed"])
        assert qo.shape == (B, DIM) and io.shape == (B, DIM)
        item_ids = torch.from_numpy(batch["movieId"])
        neg_e, neg_i = sampler(io, item_ids)
        fake = types.SimpleNamespace(downscore_false_negatives=True, false_negative_score=MINF)
        logits = con.ContrastiveOutput.contrastive_outputs(fake, qo, io, neg_e, positive_id=item_ids, negative_id=neg_i)
        assert (logits[:, 1:] == MINF).sum().item() > B  # the diagonal plus the duplicated item
        logits = bias_mod.LogitsTemperatureScaler(T)(logits)
        loss = F.cross_entropy(logits, torch.zeros(B, dtype=torch.long))
        loss.backward()
        blobs[f"{vt}_loss"] = np.float64(loss.item())
        blobs[f"{vt}_query_out"] = qo.detach().numpy().copy()
        blobs[f"{vt}_item_out"] = io.detach().numpy().copy()
        for tag, t in towers.items():
            ids = blobs[f"{tag}_table_{t['f']}_ids"]
            g = t["emb"].weight.grad.detach().numpy()
            assert not np.any(g[np.setdiff1d(np.arange(g.shape[0]), ids)]), f"{t['f']}: gradient outside the batch's rows"
            blobs[f"{vt}_grad_{tag}_table_{t['f']}_rows"] = g[ids].copy()

    path = G.OUT / "mf_train" / "ref_torch_mf_train.npz"
    path.parent.mkdir(exist_ok=True)
    np.savez(path, kind="mf_train", dim=np.int64(DIM), temperatures=np.array(TEMPERATURES), min_float=np.float64(MINF),
             query_cols=np.array([c.name for c in q_cols]), item_cols=np.array([c.name for c in i_cols]),
             **{f"batch_{k}": v for k, v in batch.items()}, **blobs)
    print("wrote", path)


if __name__ == "__main__":
    main()
