"""Cost of learning-rate schedules and per-block optimizers in a DLRM training step: the Criteo schema (26 tables, 13
continuous columns), embedding_dim 64, bottom [512, 256, 64], top [1024, 1024, 512, 256, 1], B = 65 536, every step one
CUDA-graph replay.

Legs, timed in alternating blocks in one process with CUDA events:
  adagrad     Adagrad(0.01)
  schedule    Adagrad(ExponentialDecay(0.01, 100000, 0.96, staircase=True)): mm_opt_tick_schedule instead of mm_opt_tick
  multi       MultiOptimizer: Adagrad on the tables with >= 100 000 rows, Adam on the smaller tables and (by default) on
              the dense layers: one tick and one sparse apply per width for each group
Prints one JSON line: ms per step per leg (median, min, max over the blocks), launches per graph, the card's name and
power limit read in the same run.

    python tools/train_optimizer_bench.py [--batch 65536] [--steps 20] [--blocks 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import models_b200 as mm  # noqa: E402
from models_b200 import datasets  # noqa: E402
from train_pretrained_bench import card, timed  # noqa: E402

THRESHOLD = 100_000


def build_leg(leg: str, schema, B: int, dev, x, y):
    mm.set_seed(0)
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([512, 256, 64]),
                         top_block=mm.MLPBlock([1024, 1024, 512, 256]))
    model.build(dev)
    if leg == "adagrad":
        opt = mm.Adagrad(0.01)
    elif leg == "schedule":
        opt = mm.Adagrad(mm.schedules.ExponentialDecay(0.01, decay_steps=100000, decay_rate=0.96, staircase=True))
    else:
        large, small = mm.split_embeddings_on_size(model.body.embeddings, THRESHOLD)
        opt = mm.MultiOptimizer([mm.OptimizerBlocks(mm.Adagrad(0.01), large), mm.OptimizerBlocks(mm.Adam(0.001), small)],
                                default_optimizer="adam")
    model.compile(optimizer=opt)
    tr = model.trainer(B)
    tr.capture(x, y)
    return tr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_optimizer_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B = args.batch
    schema = datasets.criteo_schema({k: min(v, 1_000_000) for k, v in datasets.CRITEO_MAX.items()})
    feats, targs = datasets.split_targets(schema, datasets.generate_batch(schema, B, seed=7, index_law="uniform"))
    x = {k: torch.from_numpy(np.asarray(v)).to(dev) for k, v in feats.items()}
    y = torch.from_numpy(np.asarray(targs["label"], dtype=np.float32)).to(dev)

    legs = {leg: build_leg(leg, schema, B, dev, x, y) for leg in ("adagrad", "schedule", "multi")}
    for tr in legs.values():  # warm every graph
        tr.replay()
    torch.cuda.synchronize()
    times = {leg: [] for leg in legs}
    for _ in range(args.blocks):
        for leg, tr in legs.items():
            times[leg].append(timed(tr.replay, args.steps) / 1e3)
    for tr in legs.values():
        tr.check_indices()
    res = {"tool": "train_optimizer_bench", "card": card(), "batch": B, "steps_per_block": args.steps, "blocks": args.blocks,
           "step_ms": {leg: {"median": float(np.median(t)), "min": float(np.min(t)), "max": float(np.max(t))}
                       for leg, t in times.items()},
           "launches_per_graph": {leg: tr.launches_per_step for leg, tr in legs.items()},
           "optimizer_groups": {leg: [g.kind for g in tr._groups.groups] for leg, tr in legs.items()}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
