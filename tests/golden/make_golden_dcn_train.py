"""Golden vectors of ONE TRAINING STEP of the reference's torch DCNModel — TEST INFRASTRUCTURE, run in the build container
where /root/reference exists:

    python tests/golden/make_golden_dcn_train.py      # writes tests/golden/dcn_train/ref_torch_dcn_train.npz

It reuses the stand-in modules of oracle/make_golden_from_reference_torch.py (that script and the fixtures it writes are
left as they are), as tests/golden/make_golden_multitask.py does, and executes the reference's torch/models/ranking.py
DCNModel unmodified with its default input block (embedding widths inferred from the cardinalities) and default
BinaryOutput, twice: stacked with depth 2, and parallel (stacked=False) with depth 1.  nn.BCELoss on the sigmoid output and
torch.autograd give the gradients.

The schema's categorical widths include 24 (4 097 - 20 736 rows) and 48 (160 001 - 331 776 rows), which the sparse update
formerly rejected, and its sorted column names interleave categorical and continuous columns, so tables start at
unaligned column offsets of x0.  The script asserts both.  Tables are stored as the rows the batch touches (ids, rows and
gradient rows); the gradient of every other row is asserted to be zero.  x0 and the head's input are captured with
forward hooks and checked against the sorted-name concat and the branch order the package assumes.  Its own rng: nothing
else moves.  Checked by tests/test_dcn_train_host.py (the restatement) and tests/test_gpu_train_dcn.py (the CUDA step).
"""
from __future__ import annotations

import importlib
import math
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import make_golden_from_reference_torch as G  # noqa: E402

# (name, max id): widths 16, 24, 48, 8 by the reference's rule; C2 / C4 / C6 are continuous
CATS = [("C1", 300), ("C3", 5000), ("C5", 200000), ("C7", 7)]
CONTS = ["C2", "C4", "C6"]
WIDTHS = {"C1": 16, "C3": 24, "C5": 48, "C7": 8}
B = 37


def _width(card: int) -> int:
    return int(math.ceil(math.ceil(card ** 0.25 * 2.0) / 8) * 8)


def run(torch, ranking, mlpm, schema, batch, y, stacked: bool, depth: int, seed: int, tag: str) -> dict:
    torch.manual_seed(seed)
    m = ranking.DCNModel(schema, depth=depth, deep_block=mlpm.MLPBlock([16, 8]), stacked=stacked)
    feed = {k: torch.from_numpy(v) for k, v in batch.items()}
    m(feed)  # lazy modules are built by the first call
    lins = [mod for _, mod in m.named_modules() if isinstance(mod, torch.nn.Linear)]
    embs = {}
    for name, mod in m.named_modules():
        if isinstance(mod, torch.nn.Embedding):
            feat = [n for n, _ in CATS if f".{n}." in f".{name}."][0]
            embs[feat] = mod
    assert {f: e.weight.shape[1] for f, e in embs.items()} == WIDTHS, {f: e.weight.shape for f, e in embs.items()}
    d = sum(WIDTHS.values()) + len(CONTS)
    cross = [l for l in lins if l.in_features == d and l.out_features == d]
    rest = [l for l in lins if not (l.in_features == d and l.out_features == d)]
    assert len(cross) == depth and len(rest) == 3, (len(cross), len(rest))
    head = rest[2]
    seen = {}
    hooks = [cross[0].register_forward_pre_hook(lambda mod, inp: seen.__setitem__("x0", inp[0].detach().clone())),
             head.register_forward_pre_hook(lambda mod, inp: seen.__setitem__("head_in", inp[0].detach().clone()))]
    m.zero_grad()
    out = m(feed)["click"]
    for h in hooks:
        h.remove()
    loss_mods = [mod for mod in m.modules() if isinstance(mod, torch.nn.BCELoss)]
    assert len(loss_mods) == 1, loss_mods
    loss = loss_mods[0](out, torch.from_numpy(y).reshape(-1, 1))
    loss.backward()

    # x0 is the sorted-name concat the package builds
    cols = {}
    for n in sorted(list(WIDTHS) + CONTS):
        if n in WIDTHS:
            cols[n] = embs[n].weight.detach()[torch.from_numpy(batch[n])]
        else:
            cols[n] = torch.from_numpy(batch[n]).reshape(-1, 1)
    x0 = torch.cat([cols[n] for n in sorted(cols)], dim=1)
    assert torch.allclose(seen["x0"], x0), "x0 is not the sorted-name concat"
    order = "cross_deep"
    if not stacked:
        with torch.no_grad():
            x = x0
            for l in cross:
                x = x0 * l(x) + x
            h = x0
            for l in rest[:2]:
                h = torch.relu(l(h))
        if torch.allclose(seen["head_in"], torch.cat([h, x], dim=1)):
            order = "deep_cross"
        else:
            assert torch.allclose(seen["head_in"], torch.cat([x, h], dim=1)), "head input is neither [cross | deep] nor [deep | cross]"

    blobs = {f"{tag}_order": np.array(order), f"{tag}_out": out.detach().numpy().copy(), f"{tag}_loss": np.float32(loss.item())}
    for f, e in embs.items():
        ids = np.unique(batch[f])
        g = e.weight.grad.detach().numpy()
        rest_rows = np.setdiff1d(np.arange(g.shape[0]), ids)
        assert not np.any(g[rest_rows]), f"{f}: gradient outside the batch's rows"
        blobs[f"{tag}_table_{f}_ids"] = ids
        blobs[f"{tag}_table_{f}_rows"] = e.weight.detach().numpy()[ids].copy()
        blobs[f"{tag}_grad_table_{f}_rows"] = g[ids].copy()
    for grp, ls, act in (("cross", cross, "linear"), ("deep", rest[:2], "relu"), ("head", [head], "sigmoid")):
        for i, l in enumerate(ls):
            blobs[f"{tag}_{grp}_kernel_{i}"] = l.weight.detach().numpy().T.copy()  # Keras layout (in, out)
            blobs[f"{tag}_{grp}_bias_{i}"] = l.bias.detach().numpy().copy()
            blobs[f"{tag}_{grp}_act_{i}"] = np.array(act)
            blobs[f"{tag}_grad_{grp}_kernel_{i}"] = l.weight.grad.detach().numpy().T.copy()
            blobs[f"{tag}_grad_{grp}_bias_{i}"] = l.bias.grad.detach().numpy().copy()
    return blobs


def main():
    if not G.REF.exists():
        raise SystemExit("/root/reference is not present: golden vectors can only be regenerated in the build container")
    G.install_stand_ins()
    import torch

    import models_b200.schema as S

    ranking = importlib.import_module("merlin.models.torch.models.ranking")
    mlpm = importlib.import_module("merlin.models.torch.blocks.mlp")
    for n, mx in CATS:
        assert _width(mx + 1) == WIDTHS[n], (n, _width(mx + 1))
    rng = np.random.default_rng(1037)
    cols = [S.ColumnSchema(n, tags=("categorical",), dtype="int64", properties={"domain": {"min": 0, "max": mx, "name": n}})
            for n, mx in CATS]
    cols += [S.ColumnSchema(n, tags=("continuous",), dtype="float32") for n in CONTS]
    cols.append(S.ColumnSchema("click", tags=("target", "binary_classification"), dtype="int64"))
    schema = S.Schema(cols)
    batch = {n: rng.integers(0, mx + 1, B).astype(np.int64) for n, mx in CATS}
    batch["C7"][:10] = 3  # duplicate ids in one batch
    batch.update({n: rng.standard_normal(B).astype(np.float32) for n in CONTS})
    y = rng.integers(0, 2, B).astype(np.float32)
    blobs = {}
    blobs.update(run(torch, ranking, mlpm, schema, batch, y, stacked=True, depth=2, seed=31, tag="stacked"))
    blobs.update(run(torch, ranking, mlpm, schema, batch, y, stacked=False, depth=1, seed=32, tag="parallel"))
    path = G.OUT / "dcn_train" / "ref_torch_dcn_train.npz"
    path.parent.mkdir(exist_ok=True)
    np.savez(path, kind="dcn_train", cat_names=np.array([n for n, _ in CATS]), cat_max=np.array([mx for _, mx in CATS], dtype=np.int64),
             cont_names=np.array(CONTS), targets=y, **{f"batch_{k}": v for k, v in batch.items()}, **blobs)
    print("wrote", path)


if __name__ == "__main__":
    main()
