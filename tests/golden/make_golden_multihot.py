"""Golden vectors of ONE TRAINING STEP of the reference's torch DLRMModel on a schema with a ragged multi-hot column —
TEST INFRASTRUCTURE, run in the build container where /root/reference exists:

    python tests/golden/make_golden_multihot.py      # writes tests/golden/multihot/ref_torch_dlrm_train_multihot.npz

It reuses the stand-in modules of oracle/make_golden_from_reference_torch.py (that script and the fixtures it writes are
left as they are) and executes the reference's module files unmodified: torch/models/ranking.py DLRMModel, whose
DLRMInputBlock routes the categorical columns through EmbeddingTables(dim, seq_combiner="mean") — a ragged
`name__values` + `name__offsets` column goes through F.embedding_bag(mode="mean") (torch/inputs/embedding.py:264-293,
torch/blocks/dlrm.py:47) — then the backend's default BinaryOutput loss (nn.BCELoss on the sigmoid outputs) and
torch.autograd.  Stored: the batch, every weight, the outputs, the loss and every gradient (tables included).  Its own
rng: nothing else moves.  The fixture lives in its own directory: tests/golden/*.npz are the fixtures that
tests/golden/replay.py knows how to check; this one is checked by tests/test_train_multihot_host.py (the restatement) and
tests/test_gpu_train_multihot.py (the CUDA step).
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


def main():
    if not G.REF.exists():
        raise SystemExit("/root/reference is not present: golden vectors can only be regenerated in the build container")
    G.install_stand_ins()
    import torch

    import models_b200.schema as S

    ranking = importlib.import_module("merlin.models.torch.models.ranking")
    mlpm = importlib.import_module("merlin.models.torch.blocks.mlp")
    rng = np.random.default_rng(915)
    cats = [("C1", 30), ("C10", 7), ("C2", 101), ("genres", 18)]
    conts = ["I1", "I2", "I3"]
    cols = [S.ColumnSchema(n, tags=("categorical",), dtype="int64", properties={"domain": {"min": 0, "max": mx, "name": n}})
            for n, mx in cats[:3]]
    cols.append(S.ColumnSchema("genres", tags=("categorical",), dtype="int64", is_list=True, is_ragged=True,
                               properties={"domain": {"min": 0, "max": 18, "name": "genres"}, "value_count": {"min": 0, "max": 4}}))
    cols += [S.ColumnSchema(n, tags=("continuous",), dtype="float32") for n in conts]
    cols.append(S.ColumnSchema("click", tags=("target", "binary_classification"), dtype="int64"))
    dim, Bm = 16, 37
    lens = rng.integers(0, 5, Bm)
    lens[[4, 20]] = 0  # empty bags: embedding_bag gives zeros
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    batch = {n: rng.integers(0, mx + 1, Bm).astype(np.int64) for n, mx in cats[:3]}
    batch["genres__values"] = rng.integers(0, 19, int(offs[-1])).astype(np.int64)
    batch["genres__offsets"] = offs
    batch.update({n: rng.random(Bm).astype(np.float32) for n in conts})
    y = rng.integers(0, 2, Bm).astype(np.float32)
    torch.manual_seed(21)
    dm = ranking.DLRMModel(S.Schema(cols), dim=dim, bottom_block=mlpm.MLPBlock([32, dim]), top_block=mlpm.MLPBlock([24, 8]))
    out = dm({k: torch.from_numpy(v) for k, v in batch.items()})["click"]
    combiners = {getattr(m, "seq_combiner") for _, m in dm.named_modules() if isinstance(getattr(m, "seq_combiner", None), str)}
    assert combiners == {"mean"}, combiners  # the backend's default bag combiner
    loss_mods = [m for m in dm.modules() if isinstance(m, torch.nn.BCELoss)]
    assert len(loss_mods) == 1, loss_mods
    dm.zero_grad()
    loss = loss_mods[0](out, torch.from_numpy(y).reshape(-1, 1))
    loss.backward()

    blobs = {}
    for name, m in dm.named_modules():
        if isinstance(m, torch.nn.Embedding):
            feat = [n for n, _ in cats if f".{n}." in f".{name}."][0]
            blobs[f"table_{feat}"] = m.weight.detach().numpy().copy()
            blobs[f"grad_table_{feat}"] = m.weight.grad.detach().numpy().copy()
    assert len([k for k in blobs if k.startswith("table_")]) == len(cats)
    lins = [(n, m) for n, m in dm.named_modules() if isinstance(m, torch.nn.Linear)]
    assert len(lins) == 5
    groups = {"bottom": [m for n, m in lins if ".continuous." in f".{n}."],
              "top": [m for n, m in lins if ".continuous." not in f".{n}."][:2], "head": [lins[-1][1]]}
    for tag, ls in groups.items():
        for i, l in enumerate(ls):
            blobs[f"{tag}_kernel_{i}"] = l.weight.detach().numpy().T.copy()  # Keras layout (in, out)
            blobs[f"{tag}_bias_{i}"] = l.bias.detach().numpy().copy()
            blobs[f"{tag}_act_{i}"] = np.array("sigmoid" if tag == "head" else "relu")
            blobs[f"grad_{tag}_kernel_{i}"] = l.weight.grad.detach().numpy().T.copy()
            blobs[f"grad_{tag}_bias_{i}"] = l.bias.grad.detach().numpy().copy()
    path = G.OUT / "multihot" / "ref_torch_dlrm_train_multihot.npz"
    path.parent.mkdir(exist_ok=True)
    np.savez(path, kind="dlrm_train_multihot", cat_names=np.array([n for n, _ in cats]),
             cat_max=np.array([mx for _, mx in cats], dtype=np.int64), list_names=np.array(["genres"]),
             cont_names=np.array(conts), dim=np.int64(dim), combiner=np.array("mean"), out=out.detach().numpy(), targets=y,
             loss=np.float32(loss.item()), **{f"batch_{k}": v for k, v in batch.items()}, **blobs)
    print("wrote", path)


if __name__ == "__main__":
    main()
