"""Wide&Deep training step on the Criteo schema, captured as one CUDA graph.

    python tools/train_wide_deep_bench.py [--multihot] [--batch 65536] [--blocks 6] [--steps 20] [--max-rows 4000000]
    python tools/train_wide_deep_bench.py [--multihot] --profile [--steps 20]

The bundled Criteo schema with tables capped at --max-rows rows.  Wide side: the 26 categorical columns (CategoryEncoding,
one_hot; multi_hot with --multihot).  Deep side: every column at inferred embedding widths, deep_block = MLPBlock([1024,
512, 256]), the deep logit MLPBlock([1]).  BinaryOutput, Adagrad(0.01), batch 65 536.  --multihot feeds the categorical
columns as fixed-length (B, L) id matrices with the MLPerf DLRM-DCNv2 bag sizes (tools/train_multihot_bench.py), to both
sides, the deep side then at embedding width 32 (the multi-hot deep update takes widths 16, 32, 64, 128).  Prints the
card's name and power limit read in the same run, launches per step, the median ms per step over --blocks blocks of --steps graph replays (CUDA events; block 0 warms up), and the bytes floors of the head kernel
(mm_wide_deep_head_fwd_bwd) and the wide update computed from the shapes.  --profile (a separate run: tracing slows the
host) prints each kernel's device time per step under torch.profiler: compare the head's and the update's lines with
their floors.
"""
import argparse
import statistics
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import models_b200 as mm  # noqa: E402
from models_b200 import datasets  # noqa: E402
from models_b200.schema import Tags  # noqa: E402

DEEP = [1024, 512, 256]
BAG_SIZES = [3, 2, 1, 2, 6, 1, 1, 1, 1, 7, 3, 8, 1, 6, 9, 5, 1, 1, 1, 12, 100, 27, 10, 3, 1, 1]  # C1..C26 (MLPerf DLRM-DCNv2)
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def floors(B: int, ids_per_sample: int, U: int) -> dict:
    """Bytes per step (computed, not measured).  Head: h (U floats) read, dh (U floats) written, 4-byte ids, one wide scalar
    per id at 32-byte sector granularity (random rows), target, logit and ds.  Wide update: the ids and ds read again, and
    per id a 32-byte sector of the kernel, the accumulator and the Adagrad slot, read and written."""
    head = {"h": 4 * U, "dh": 4 * U, "ids": 4 * ids_per_sample, "wide scalars (32-B sectors)": 32 * ids_per_sample,
            "target + logit + ds": 12}
    update = {"ids + ds": 4 * ids_per_sample + 4, "kernel, acc, slot (32-B sectors, r+w)": 2 * 3 * 32 * ids_per_sample}
    return {"head": {k: v * B for k, v in head.items()}, "update": {k: v * B for k, v in update.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--max-rows", type=int, default=4_000_000)
    ap.add_argument("--multihot", action="store_true")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_wide_deep_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card()}")
    B = args.batch
    schema = datasets.criteo_schema({k: min(v, args.max_rows - 1) for k, v in datasets.CRITEO_MAX.items()})
    cats = [c for c in schema.select_by_tag(Tags.CATEGORICAL)]
    conts = [c for c in schema.select_by_tag(Tags.CONTINUOUS)]
    wide_schema = schema.select_by_name([c.name for c in cats])
    mm.set_seed(1)
    # the multi-hot deep update (mm_bag_grad_rows) takes widths 16, 32, 64 and 128; the inferred ones include 8, 24, 48, 96
    deep_in = None
    if args.multihot:
        deep_in = mm.InputBlockV2(schema, categorical=mm.Embeddings(schema.select_by_tag(Tags.CATEGORICAL), dim=32))
    model = mm.WideAndDeepModel(schema, deep_block=mm.MLPBlock(DEEP), wide_schema=wide_schema, deep_input_block=deep_in,
                                wide_preprocess=mm.CategoryEncoding(wide_schema, output_mode="multi_hot" if args.multihot else "one_hot"),
                                prediction_tasks=mm.BinaryOutput(schema.select_by_tag(Tags.TARGET).column_names[0]))
    model.build(dev)
    model.compile(optimizer=mm.Adagrad(0.01))
    g = torch.Generator(device=dev).manual_seed(7)
    bag = {c.name: (BAG_SIZES[i] if args.multihot else 1) for i, c in enumerate(cats)}
    batches = []
    for _ in range(4):
        x = {}
        for c in cats:
            shape = (B,) if bag[c.name] == 1 else (B, bag[c.name])
            x[c.name] = torch.randint(0, c.int_domain.max + 1, shape, generator=g, device=dev, dtype=torch.int32)
        x.update({c.name: torch.rand(B, generator=g, device=dev) for c in conts})
        batches.append((x, (torch.rand(B, generator=g, device=dev) < 0.3).float()))
    tr = model.trainer(B)
    tr.capture(*batches[0])
    ids = sum(bag.values())
    U = DEEP[-1]
    print(f"{'multi-hot' if args.multihot else 'one-hot'} Wide&Deep train step, batch {B}, {ids} ids per sample, d = {tr.inp.d}, "
          f"deep {DEEP}, wide kernel {tr.wk.dense.kernel.shape[0]} rows, launches per step: {tr.launches_per_step}")
    for name, fl in floors(B, ids, U).items():
        total = sum(fl.values())
        print(f"{name} bytes per step (computed): " + ", ".join(f"{k} {v / 1e6:.1f} MB" for k, v in fl.items())
              + f"; total {total / 1e6:.1f} MB = {total / HBM_BYTES_PER_S * 1e6:.1f} us at 3.35 TB/s")
    if args.multihot:
        pairs = sum(L * (L - 1) // 2 for L in BAG_SIZES)
        print(f"deduplication: {pairs} id comparisons per sample in the head and again in mm_wide_bag_grad "
              f"({pairs * B / 1e6:.0f} M per step each)")

    if args.profile:
        for i in range(5):
            tr.replay(*batches[i % 4])
        torch.cuda.synchronize()
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            for i in range(args.steps):
                tr.replay(*batches[i % 4])
            torch.cuda.synchronize()
        per = defaultdict(lambda: [0.0, 0])
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                per[e.name][0] += e.time_range.elapsed_us()
                per[e.name][1] += 1
        out = sorted(((us / args.steps, n / args.steps, name) for name, (us, n) in per.items()), reverse=True)
        print(f"device time per step by kernel ({args.steps} graph replays)")
        for us, n, name in out:
            print(f"  {us:9.1f} us  {n:4.1f}x  {name[:110]}")
        print(f"  {sum(r[0] for r in out):9.1f} us  sum of kernel times per step")
        return

    times = []
    for blk in range(args.blocks + 1):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for i in range(args.steps):
            tr.replay(*batches[i % 4])
        t1.record()
        torch.cuda.synchronize()
        if blk > 0:
            times.append(t0.elapsed_time(t1) / args.steps)
    st = statistics.median(times)
    print(f"train step: {st:.3f} ms (median of {len(times)} blocks, range {min(times):.3f}-{max(times):.3f}), "
          f"{B / st / 1e3:.2f} M samples/s")


if __name__ == "__main__":
    main()
