"""DLRM training step on multi-hot features at the Criteo shape, captured as one CUDA graph.

    python tools/train_multihot_bench.py [--batch 65536] [--steps 20] [--warmup 5] [--profile]

26 tables at the bundled Criteo cardinalities (datasets.CRITEO_MAX), D = 64, bottom [128, 64], top [128, 64, 32],
Adagrad(0.01).  Feature C{i} carries MLPerf DLRM-DCNv2's fixed bag size as a (B, L) id matrix pooled with `sum`; bag size 1
stays a one-hot (B,) column: 214 ids per sample.  Prints ms per step and samples/s (CUDA events around `--steps` graph
replays), the card's name and power limit read in the same run, and the algorithmic bytes of the bag stages.  With
--profile (a separate run: tracing slows the host) it prints each kernel's device time per step under torch.profiler.
"""
import argparse
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import models_b200 as mm  # noqa: E402
from models_b200 import datasets  # noqa: E402

BAG_SIZES = [3, 2, 1, 2, 6, 1, 1, 1, 1, 7, 3, 8, 1, 6, 9, 5, 1, 1, 1, 12, 100, 27, 10, 3, 1, 1]  # C1..C26 (MLPerf DLRM-DCNv2)


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def make_batch(B: int, seed: int, dev) -> tuple:
    g = torch.Generator(device=dev).manual_seed(seed)
    x = {}
    for i, L in enumerate(BAG_SIZES, start=1):
        rows = datasets.CRITEO_MAX[f"C{i}"] + 1
        shape = (B,) if L == 1 else (B, L)
        x[f"C{i}"] = torch.randint(0, rows, shape, generator=g, device=dev, dtype=torch.int32)
    for i in range(1, 14):
        x[f"I{i}"] = torch.rand(B, generator=g, device=dev)
    y = (torch.rand(B, generator=g, device=dev) < 0.5).float()
    return x, y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="per-kernel device time per step under torch.profiler")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_multihot_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card()}")
    B, D = args.batch, 64
    mm.set_seed(1)
    schema = datasets.criteo_schema()
    model = mm.DLRMModel(schema, embedding_dim=D, bottom_block=mm.MLPBlock([128, D]), top_block=mm.MLPBlock([128, 64, 32]),
                         embedding_options=mm.EmbeddingOptions(combiner="sum", embeddings_initializers={"hash_seed": 4321}))
    model.build(dev)
    model.compile(optimizer=mm.Adagrad(0.01))
    batches = [make_batch(B, 100 + i, dev) for i in range(4)]
    tr = model.trainer(B)
    tr.capture(*batches[0])

    def run(n):
        for i in range(n):
            tr.replay(*batches[i % len(batches)])

    run(args.warmup)
    torch.cuda.synchronize()
    ids_per_sample = sum(BAG_SIZES)
    bag_ids = sum(L for L in BAG_SIZES if L > 1)
    nnz = B * bag_ids
    if not args.profile:
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        run(args.steps)
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / args.steps
        print(f"multi-hot DLRM train step, B = {B}, {ids_per_sample} ids per sample ({bag_ids} in {sum(L > 1 for L in BAG_SIZES)} "
              f"fixed-length bags, sum), D = {D}, Adagrad, one CUDA graph ({tr.launches_per_step} launches): "
              f"{ms:.3f} ms per step, {B / (ms * 1e-3):.0f} samples/s (loss {tr.loss.item():.5f})")
    else:
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            run(args.steps)
            torch.cuda.synchronize()
        per = defaultdict(lambda: [0.0, 0])
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                per[e.name][0] += e.time_range.elapsed_us()
                per[e.name][1] += 1
        rows = sorted(((us / args.steps, n / args.steps, name) for name, (us, n) in per.items()), reverse=True)
        print(f"device time per step by kernel ({args.steps} graph replays, serial):")
        for us, n, name in rows:
            print(f"  {us:9.1f} us  {n:5.1f}x  {name[:110]}")
        print(f"  {sum(r[0] for r in rows):9.1f} us  sum of kernel times per step")
    row = D * 4
    print("algorithmic bytes of the bag stages per step (from the shapes):")
    print(f"  pooling (gather_seq) reads {bag_ids} rows x {row} B per sample = {B * bag_ids * row / 1e9:.3f} GB "
          f"(all {ids_per_sample} ids per sample: {B * ids_per_sample * row / 1e9:.3f} GB)")
    print(f"  expansion (bag_grad_rows) writes nnz x D x 4 = {nnz} x {row} B = {nnz * row / 1e9:.3f} GB")
    print(f"  the apply (sparse_rows_apply) then reads those {nnz * row / 1e9:.3f} GB of expanded rows")


if __name__ == "__main__":
    main()
