"""Golden vectors of ONE TRAINING STEP of the reference's torch DLRMModel with several outputs — TEST INFRASTRUCTURE, run
in the build container where /root/reference exists:

    python tests/golden/make_golden_multitask.py      # writes tests/golden/multitask/ref_torch_dlrm_train_multitask.npz

It reuses the stand-in modules of oracle/make_golden_from_reference_torch.py (that script and the fixtures it writes are
left as they are) and executes the reference's module files unmodified: torch/models/ranking.py DLRMModel on a schema
with the targets `click`, `conversion` (binary) and `rating` (regression).  Its default output block builds one
BinaryOutput / RegressionOutput per target; torch/models/base.py `compute_loss` sums each output's default loss
(nn.BCELoss on the sigmoid output, nn.MSELoss on the linear one) divided by the number of outputs, and torch.autograd
differentiates it.  Stored: the batch, every weight (heads by target), the per-output predictions, the loss and every
gradient (tables included).  Some ratings are far from the prediction.  Its own rng: nothing else moves.  The fixture
lives in its own directory: tests/golden/*.npz are the fixtures that tests/golden/replay.py knows how to check; this one is
checked by tests/test_multitask_host.py (the restatement) and tests/test_gpu_multitask.py (the CUDA step).
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

TARGETS = [("click", "binary"), ("conversion", "binary"), ("rating", "regression")]


def main():
    if not G.REF.exists():
        raise SystemExit("/root/reference is not present: golden vectors can only be regenerated in the build container")
    G.install_stand_ins()
    import torch

    import models_b200.schema as S

    ranking = importlib.import_module("merlin.models.torch.models.ranking")
    mlpm = importlib.import_module("merlin.models.torch.blocks.mlp")
    base = importlib.import_module("merlin.models.torch.models.base")
    rng = np.random.default_rng(916)
    cats = [("C1", 30), ("C10", 7), ("C2", 101)]
    conts = ["I1", "I2"]
    cols = [S.ColumnSchema(n, tags=("categorical",), dtype="int64", properties={"domain": {"min": 0, "max": mx, "name": n}})
            for n, mx in cats]
    cols += [S.ColumnSchema(n, tags=("continuous",), dtype="float32") for n in conts]
    for n, kind in TARGETS:
        if kind == "binary":
            cols.append(S.ColumnSchema(n, tags=("target", "binary_classification"), dtype="int64"))
        else:
            cols.append(S.ColumnSchema(n, tags=("target", "regression"), dtype="float32"))
    dim, Bm = 16, 41
    batch = {n: rng.integers(0, mx + 1, Bm).astype(np.int64) for n, mx in cats}
    batch.update({n: rng.random(Bm).astype(np.float32) for n in conts})
    targets = {"click": rng.integers(0, 2, Bm).astype(np.float32), "conversion": rng.integers(0, 2, Bm).astype(np.float32),
               "rating": (rng.random(Bm) * 5.0).astype(np.float32)}
    targets["rating"][[3, 17, 30]] = [40.0, -25.0, 60.0]  # far from any prediction
    torch.manual_seed(22)
    dm = ranking.DLRMModel(S.Schema(cols), dim=dim, bottom_block=mlpm.MLPBlock([32, dim]), top_block=mlpm.MLPBlock([24, 8]))
    out = dm({k: torch.from_numpy(v) for k, v in batch.items()})
    assert isinstance(out, dict) and sorted(out) == sorted(n for n, _ in TARGETS), out
    outputs = dm.model_outputs()
    assert len(outputs) == len(TARGETS)
    dm.zero_grad()
    res = base.compute_loss(out, {k: torch.from_numpy(v) for k, v in targets.items()}, outputs, compute_metrics=False)
    loss = res["loss"]
    loss.backward()

    blobs = {}
    for name, m in dm.named_modules():
        if isinstance(m, torch.nn.Embedding):
            feat = [n for n, _ in cats if f".{n}." in f".{name}."][0]
            blobs[f"table_{feat}"] = m.weight.detach().numpy().copy()
            blobs[f"grad_table_{feat}"] = m.weight.grad.detach().numpy().copy()
    lins = [(n, m) for n, m in dm.named_modules() if isinstance(m, torch.nn.Linear)]
    assert len(lins) == 4 + len(TARGETS), [n for n, _ in lins]
    heads = {}
    for mo in outputs:  # each output's Linear(1), by the target it predicts
        hl = [m for m in mo.modules() if isinstance(m, torch.nn.Linear)]
        assert len(hl) == 1
        heads[mo.output_schema.first.name] = hl[0]
    head_ids = {id(m) for m in heads.values()}
    tower = [(n, m) for n, m in lins if id(m) not in head_ids]
    groups = {"bottom": [m for n, m in tower if ".continuous." in f".{n}."],
              "top": [m for n, m in tower if ".continuous." not in f".{n}."]}
    assert len(groups["bottom"]) == 2 and len(groups["top"]) == 2
    for tag, ls in groups.items():
        for i, l in enumerate(ls):
            blobs[f"{tag}_kernel_{i}"] = l.weight.detach().numpy().T.copy()  # Keras layout (in, out)
            blobs[f"{tag}_bias_{i}"] = l.bias.detach().numpy().copy()
            blobs[f"{tag}_act_{i}"] = np.array("relu")
            blobs[f"grad_{tag}_kernel_{i}"] = l.weight.grad.detach().numpy().T.copy()
            blobs[f"grad_{tag}_bias_{i}"] = l.bias.grad.detach().numpy().copy()
    for n, kind in TARGETS:
        l = heads[n]
        blobs[f"head_{n}_kernel"] = l.weight.detach().numpy().T.copy()
        blobs[f"head_{n}_bias"] = l.bias.detach().numpy().copy()
        blobs[f"grad_head_{n}_kernel"] = l.weight.grad.detach().numpy().T.copy()
        blobs[f"grad_head_{n}_bias"] = l.bias.grad.detach().numpy().copy()
        blobs[f"out_{n}"] = out[n].detach().numpy().copy()
        blobs[f"targets_{n}"] = targets[n]
    loss_kinds = [type(mo.loss).__name__ for mo in outputs]
    assert sorted(loss_kinds) == ["BCELoss", "BCELoss", "MSELoss"], loss_kinds
    path = G.OUT / "multitask" / "ref_torch_dlrm_train_multitask.npz"
    path.parent.mkdir(exist_ok=True)
    np.savez(path, kind="dlrm_train_multitask", cat_names=np.array([n for n, _ in cats]),
             cat_max=np.array([mx for _, mx in cats], dtype=np.int64), cont_names=np.array(conts), dim=np.int64(dim),
             target_names=np.array([n for n, _ in TARGETS]), target_kinds=np.array([k for _, k in TARGETS]),
             loss=np.float32(loss.item()), **{f"batch_{k}": v for k, v in batch.items()}, **blobs)
    print("wrote", path)


if __name__ == "__main__":
    main()
