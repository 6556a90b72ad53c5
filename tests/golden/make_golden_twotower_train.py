"""Golden vectors of ONE TRAINING STEP of the reference's torch two-tower set-up — TEST INFRASTRUCTURE, run in the build
container where /root/reference exists:

    python tests/golden/make_golden_twotower_train.py   # writes tests/golden/twotower_train/ref_torch_twotower_train.npz

It reuses the stand-in modules of oracle/make_golden_from_reference_torch.py (that script and the fixtures it writes are
left as they are), as tests/golden/make_golden_dcn_train.py does, and executes the reference's torch modules unmodified:
the §13 towers of that script (TabularInputBlock with EmbeddingTables(16, seq_combiner="mean") and the continuous columns,
sorted-name concat, MLPBlock([24, 12])) on the ML-1M column names; InBatchNegativeSampler; then
ContrastiveOutput.contrastive_outputs with false-negative rescoring by movieId (a duplicated movieId puts one accidental
hit off the diagonal); LogitsTemperatureScaler; F.cross_entropy against class 0 (the positive column, the mean over the
batch) and torch.autograd.  Two variants on the same weights and batch: T = 1 and T = 0.5.

Stored: the batch, every tower variable and its gradient, and per table the rows the batch touches with their gradient
rows; the gradient of every other row is asserted to be zero.  Its own rng: nothing else moves.  Checked by
tests/test_twotower_train_host.py (the restatement) and tests/test_gpu_train_twotower.py (the CUDA step through
mm.TwoTowerModel).
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

B, DIM, TOWER = 41, 16, [24, 12]
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
    mlpm = importlib.import_module("merlin.models.torch.blocks.mlp")
    con = importlib.import_module("merlin.models.torch.outputs.contrastive")
    bias_mod = importlib.import_module("merlin.models.torch.transforms.bias")
    sampler = importlib.import_module("merlin.models.torch.outputs.sampling.in_batch").InBatchNegativeSampler()
    # utils/constants.py:19 under the NumPy 1.x the reference pins (see make_golden_from_reference_torch.py, section 6)
    MINF = float(np.finfo(np.float16).min) / 100.0

    def catc(name, mx, tags=(), is_list=False):
        props = {"domain": {"min": 0, "max": mx, "name": name}}
        if is_list:
            props["value_count"] = {"min": 1, "max": 4}
        return S.ColumnSchema(name, tags=("categorical",) + tuple(tags), dtype="int64", is_list=is_list, is_ragged=is_list,
                              properties=props)

    q_cols = [catc("userId", 6040, ("user", "user_id"))] + [
        S.ColumnSchema(n, tags=("continuous", "user"), dtype="float32")
        for n in ("TE_age_rating", "TE_gender_rating", "TE_occupation_rating", "TE_userId_rating", "TE_zipcode_rating")]
    i_cols = [catc("movieId", 3684, ("item", "item_id")), catc("genres", 18, ("item",), is_list=True),
              S.ColumnSchema("TE_movieId_rating", tags=("continuous", "item"), dtype="float32")]

    def tower_init(block):
        block.add_route(S.Tags.CONTINUOUS, required=False)
        block.add_route(S.Tags.CATEGORICAL, embm.EmbeddingTables(DIM, seq_combiner="mean"))

    rng = np.random.default_rng(1341)
    lens = rng.integers(1, 5, B)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    batch = {"userId": rng.integers(1, 6041, B).astype(np.int64), "movieId": rng.integers(1, 3685, B).astype(np.int64),
             "genres__values": rng.integers(1, 19, int(offs[-1])).astype(np.int64), "genres__offsets": offs,
             "TE_movieId_rating": rng.random(B).astype(np.float32)}
    batch["movieId"][5] = batch["movieId"][3]  # duplicate item -> an accidental hit off the diagonal
    batch["userId"][7] = batch["userId"][2]    # duplicate user -> two slices summed into one table row
    for c in q_cols[1:]:
        batch[c.name] = rng.random(B).astype(np.float32)

    towers = {}
    for tag, cols_t, seed in (("query", q_cols, 41), ("item", i_cols, 42)):
        torch.manual_seed(seed)
        inp = tab.TabularInputBlock(S.Schema(cols_t), init=tower_init, agg="concat")
        mlp_t = mlpm.MLPBlock(list(TOWER))
        names_t = [c.name for c in cols_t]
        feed = {k: torch.from_numpy(v) for k, v in batch.items() if any(k == n or k.startswith(n + "__") for n in names_t)}
        inp(feed)  # lazy modules are built by the first call
        mlp_t(inp(feed))
        embs = {}
        for name, m in inp.named_modules():
            if isinstance(m, torch.nn.Embedding):
                embs[[c.name for c in cols_t if f".{c.name}." in f".{name}."][0]] = m
        lins = [m for m in mlp_t.modules() if isinstance(m, torch.nn.Linear)]
        assert len(lins) == len(TOWER) and all(e.weight.shape[1] == DIM for e in embs.values())
        towers[tag] = dict(inp=inp, mlp=mlp_t, feed=feed, embs=embs, lins=lins)

    blobs = {}
    for tag, t in towers.items():
        for i, l in enumerate(t["lins"]):
            blobs[f"{tag}_kernel_{i}"] = l.weight.detach().numpy().T.copy()  # Keras layout (in, out)
            blobs[f"{tag}_bias_{i}"] = l.bias.detach().numpy().copy()
        for f, e in t["embs"].items():
            ids = np.unique(batch["genres__values"] if f == "genres" else batch[f])
            blobs[f"{tag}_table_{f}_rows_total"] = np.int64(e.weight.shape[0])
            blobs[f"{tag}_table_{f}_ids"] = ids
            blobs[f"{tag}_table_{f}_rows"] = e.weight.detach().numpy()[ids].copy()

    for T in TEMPERATURES:
        vt = f"T{T:g}".replace(".", "p")
        for t in towers.values():
            t["inp"].zero_grad()
            t["mlp"].zero_grad()
        qo = towers["query"]["mlp"](towers["query"]["inp"](towers["query"]["feed"]))
        io = towers["item"]["mlp"](towers["item"]["inp"](towers["item"]["feed"]))
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
            for i, l in enumerate(t["lins"]):
                blobs[f"{vt}_grad_{tag}_kernel_{i}"] = l.weight.grad.detach().numpy().T.copy()
                blobs[f"{vt}_grad_{tag}_bias_{i}"] = l.bias.grad.detach().numpy().copy()
            for f, e in t["embs"].items():
                ids = blobs[f"{tag}_table_{f}_ids"]
                g = e.weight.grad.detach().numpy()
                assert not np.any(g[np.setdiff1d(np.arange(g.shape[0]), ids)]), f"{f}: gradient outside the batch's rows"
                blobs[f"{vt}_grad_{tag}_table_{f}_rows"] = g[ids].copy()

    path = G.OUT / "twotower_train" / "ref_torch_twotower_train.npz"
    path.parent.mkdir(exist_ok=True)
    np.savez(path, kind="twotower_train", dim=np.int64(DIM), tower=np.array(TOWER, dtype=np.int64),
             temperatures=np.array(TEMPERATURES), min_float=np.float64(MINF), query_cols=np.array([c.name for c in q_cols]),
             item_cols=np.array([c.name for c in i_cols]), **{f"batch_{k}": v for k, v in batch.items()}, **blobs)
    print("wrote", path)


if __name__ == "__main__":
    main()
