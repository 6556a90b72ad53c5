"""DLRM training step with three outputs (two binary heads + one regression head) against the same model with one
BinaryOutput, at the Criteo shape, each captured as one CUDA graph, timed in alternating blocks in one process.

    python tools/train_multitask_bench.py [--batch 65536] [--blocks 6] [--steps 20] [--max-rows 4000000]

26 tables at the bundled Criteo cardinalities capped at --max-rows rows (two models, each with Adagrad slots and operand
mirrors, must fit on one card), D = 64, bottom [128, 64], top [128, 64, 32], Adagrad(0.01).  Prints the card's name and
power limit read in the same run, and each model's median ms per step over the blocks (CUDA events around --steps graph
replays per block).
"""
import argparse
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import models_b200 as mm  # noqa: E402
from models_b200 import datasets  # noqa: E402
from models_b200.schema import ColumnSchema, Schema, Tags  # noqa: E402


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--max-rows", type=int, default=4_000_000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_multitask_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card()}")
    B = args.batch
    base = datasets.criteo_schema({k: min(v, args.max_rows - 1) for k, v in datasets.CRITEO_MAX.items()})
    feats_cols = [c for c in base if not c.has_tag(Tags.TARGET)]
    targets = [ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"),
               ColumnSchema("conversion", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"),
               ColumnSchema("rating", tags=(Tags.TARGET, Tags.REGRESSION), dtype="float32")]
    schema = Schema(feats_cols + targets)
    g = torch.Generator(device=dev).manual_seed(7)
    batches = []
    for _ in range(4):
        x = {c.name: torch.randint(0, c.int_domain.max + 1, (B,), generator=g, device=dev, dtype=torch.int32)
             for c in feats_cols if c.has_tag(Tags.CATEGORICAL)}
        x.update({c.name: torch.rand(B, generator=g, device=dev) for c in feats_cols if c.has_tag(Tags.CONTINUOUS)})
        ys = {"click": (torch.rand(B, generator=g, device=dev) < 0.3).float(),
              "conversion": (torch.rand(B, generator=g, device=dev) < 0.05).float(),
              "rating": torch.rand(B, generator=g, device=dev) * 5.0}
        batches.append((x, ys))
    runs = {}
    for name, outputs in (("one BinaryOutput", mm.BinaryOutput("click")), ("3 outputs (2 binary + 1 regression)", mm.OutputBlock(schema))):
        mm.set_seed(1)
        model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([128, 64]), top_block=mm.MLPBlock([128, 64, 32]),
                             prediction_tasks=outputs)
        model.build(dev)
        model.compile(optimizer=mm.Adagrad(0.01))
        tr = model.trainer(B)
        ys = [[y[o.target] for o in model.output_blocks()] for _, y in batches]
        tr.capture(batches[0][0], ys[0])
        runs[name] = (tr, ys)
    print(f"batch {B}, table rows {sum(c.int_domain.max + 1 for c in feats_cols if c.has_tag(Tags.CATEGORICAL))}, "
          f"launches per step: " + ", ".join(f"{n}: {tr.launches_per_step}" for n, (tr, _) in runs.items()))
    times = {n: [] for n in runs}
    for blk in range(args.blocks + 1):
        for n, (tr, ys) in runs.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for i in range(args.steps):
                tr.replay(batches[i % 4][0], ys[i % 4])
            t1.record()
            torch.cuda.synchronize()
            if blk > 0:  # block 0 warms up
                times[n].append(t0.elapsed_time(t1) / args.steps)
    for n, ts in times.items():
        med = statistics.median(ts)
        print(f"{n}: {med:.3f} ms per step (median of {len(ts)} blocks, range {min(ts):.3f}-{max(ts):.3f}), {B / med / 1e3:.1f} M samples/s")


if __name__ == "__main__":
    main()
