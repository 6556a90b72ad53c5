"""DCN-v2 training step at bench.py's DCN shape, captured as one CUDA graph.

    python tools/train_dcn_bench.py [--batch 65536] [--blocks 6] [--steps 20] [--max-rows 4000000]
    python tools/train_dcn_bench.py --profile [--steps 20]

The bundled Criteo schema with the embedding widths InputBlockV2 infers from its full cardinalities (8 .. 120, d = 1037
with the 13 continuous columns), CrossBlock depth 3, MLPBlock([256, 128]), BinaryOutput, Adagrad(0.01), batch 65 536
(bench.py --workload dcn).  The tables keep those widths but are capped at --max-rows rows: at full size the tables and
their Adagrad slots take 42 GB, and capture's snapshot of every variable would not fit beside them on an 80 GB card.
Prints the card's name and power limit read in the same run, launches per step, and the median ms per step over
--blocks blocks of --steps graph replays (CUDA events; block 0 warms up), alternating with a block of the weight
gradient alone: mm_dense_wgrad_split on one 1037 x 1037 cross layer at the same batch, with its achieved rate from the
GEMM's FLOPs.  Also prints the GEMM FLOPs of the whole step, computed from the shapes.  --profile (a separate run: tracing
slows the host) prints each kernel's device time per step under torch.profiler.
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
from models_b200 import datasets, ops  # noqa: E402
from models_b200.inputs import infer_embedding_dim  # noqa: E402
from models_b200.schema import Tags  # noqa: E402

DEPTH, DEEP = 3, [256, 128]


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def gemm_flops(B: int, d: int) -> dict:
    """2 M N K per GEMM of one step (fp32-equivalent; the split-bf16 tensor-core path issues 3 MMAs per product)."""
    cross = DEPTH * 2 * B * d * d
    widths = [d] + DEEP
    deep = sum(2 * B * k * n for k, n in zip(widths[:-1], widths[1:]))
    return {"forward": cross + deep, "wgrad": cross + deep, "dgrad": cross + deep}  # deep dgrad of layer 0 included: dx0 feeds x_L


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--max-rows", type=int, default=4_000_000)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_dcn_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card()}")
    B = args.batch
    dims = {c.name: infer_embedding_dim(c) for c in datasets.criteo_schema().select_by_tag(Tags.CATEGORICAL)}
    schema = datasets.criteo_schema({k: min(v, args.max_rows - 1) for k, v in datasets.CRITEO_MAX.items()})
    mm.set_seed(1)
    model = mm.DCNModel(schema, depth=DEPTH, deep_block=mm.MLPBlock(DEEP), dim=dims, embeddings_initializer={"hash_seed": 99})
    model.build(dev)
    d = model.body.input_block.layout()[2]
    model.compile(optimizer=mm.Adagrad(0.01))
    g = torch.Generator(device=dev).manual_seed(7)
    cats = [c for c in schema.select_by_tag(Tags.CATEGORICAL)]
    conts = [c for c in schema.select_by_tag(Tags.CONTINUOUS)]
    batches = []
    for _ in range(4):
        x = {c.name: torch.randint(0, c.int_domain.max + 1, (B,), generator=g, device=dev, dtype=torch.int32) for c in cats}
        x.update({c.name: torch.rand(B, generator=g, device=dev) for c in conts})
        batches.append((x, (torch.rand(B, generator=g, device=dev) < 0.3).float()))
    tr = model.trainer(B)
    tr.capture(*batches[0])
    widths = sorted({tb.table.shape[1] for tb in tr.tables})
    fl = gemm_flops(B, d)
    rows = sum(tb.table.shape[0] for tb in tr.tables)
    print(f"batch {B}, d = {d}, embedding widths {widths}, {rows} table rows, launches per step: {tr.launches_per_step}")
    print("GEMM FLOP per step (2MNK, fp32-equivalent): " + ", ".join(f"{k} {v / 1e12:.3f} T" for k, v in fl.items())
          + f", total {sum(fl.values()) / 1e12:.3f} T ({3 * sum(fl.values()) / 1e12:.2f} T of bf16 MMA work with the 3-pass split)")

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
        rows = sorted(((us / args.steps, n / args.steps, name) for name, (us, n) in per.items()), reverse=True)
        print(f"device time per step by kernel ({args.steps} graph replays)")
        for us, n, name in rows:
            print(f"  {us:9.1f} us  {n:4.1f}x  {name[:110]}")
        print(f"  {sum(r[0] for r in rows):9.1f} us  sum of kernel times per step")
        return

    # the weight gradient of one cross layer alone, on the trainer's own saved operand and dz
    xs, dz = tr.xs[0], tr.dz[:, :d]
    dW = torch.zeros((d, d), dtype=torch.float32, device=dev)
    db = torch.zeros(d, dtype=torch.float32, device=dev)

    def wgrad_block():
        for _ in range(args.steps):
            ops.dense_wgrad_split(xs, d, dz, dW, db)

    def step_block():
        for i in range(args.steps):
            tr.replay(*batches[i % 4])

    times = {"step": [], "wgrad": []}
    for blk in range(args.blocks + 1):
        for name, fn in (("step", step_block), ("wgrad", wgrad_block)):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            fn()
            t1.record()
            torch.cuda.synchronize()
            if blk > 0:
                times[name].append(t0.elapsed_time(t1) / args.steps)
    st, wg = statistics.median(times["step"]), statistics.median(times["wgrad"])
    print(f"train step: {st:.3f} ms (median of {len(times['step'])} blocks, range {min(times['step']):.3f}-{max(times['step']):.3f}), "
          f"{B / st / 1e3:.2f} M samples/s, {sum(fl.values()) / st / 1e9:.1f} TFLOP/s fp32-equivalent")
    wf = 2.0 * B * d * d
    print(f"mm_dense_wgrad_split {d}x{d}, M = {B}: {wg:.3f} ms (range {min(times['wgrad']):.3f}-{max(times['wgrad']):.3f}), "
          f"{wf / wg / 1e9:.1f} TFLOP/s fp32-equivalent ({3 * wf / wg / 1e9:.1f} TFLOP/s of bf16 MMA with the 3-pass split); "
          f"{DEPTH} cross layers: {DEPTH * wg:.3f} ms of the step")


if __name__ == "__main__":
    main()
