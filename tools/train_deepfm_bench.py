"""DeepFM training step on the Criteo schema, captured as one CUDA graph.

    python tools/train_deepfm_bench.py [--batch 65536] [--blocks 6] [--steps 20] [--max-rows 4000000]
    python tools/train_deepfm_bench.py --profile [--steps 20]

The bundled Criteo schema (26 categorical, 13 continuous columns), embedding_dim = 16, deep_block = MLPBlock([400, 400,
400]) (the DeepFM paper's Criteo tower), the default deep logit MLPBlock([1]), BinaryOutput, Adagrad(0.01), batch 65 536.
The tables are capped at --max-rows rows so that capture's snapshot of every variable (tables, wide kernel, their slots)
fits beside them.  Prints the card's name and power limit read in the same run, launches per step, the median ms per step
over --blocks blocks of --steps graph replays (CUDA events; block 0 warms up), and the head kernel's bytes floor computed
from the shapes.  --profile (a separate run: tracing slows the host) prints each kernel's device time per step under
torch.profiler: compare mm_deepfm_head_fwd_bwd's line with the floor.
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

DIM, DEEP = 16, [400, 400, 400]
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def head_bytes(B: int, T: int, C: int, D: int, U: int) -> dict:
    """Bytes the head kernel must move per sample (computed, not measured): its x0 row (T D floats at the features'
    columns), h (U floats), one 4-byte id per feature, the T wide scalars at 32-byte sector granularity (random rows: one
    sector each), the C continuous values and the target, and its writes dh (U floats), ds and the logit."""
    per = {"x0 rows": 4 * T * D, "h": 4 * U, "ids": 4 * T, "wide scalars (32-B sectors)": 32 * T, "continuous + target": 4 * C + 4,
           "dh": 4 * U, "ds + logit": 8}
    return {k: v * B for k, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--max-rows", type=int, default=4_000_000)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_deepfm_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card()}")
    B = args.batch
    schema = datasets.criteo_schema({k: min(v, args.max_rows - 1) for k, v in datasets.CRITEO_MAX.items()})
    mm.set_seed(1)
    model = mm.DeepFMModel(schema, embedding_dim=DIM, deep_block=mm.MLPBlock(DEEP))
    model.build(dev)
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
    rows = sum(tb.table.shape[0] for tb in tr.tables)
    print(f"batch {B}, d = {tr.inp.d}, embedding_dim {DIM}, deep {DEEP}, {rows} table rows, wide kernel {tr.wk.dense.kernel.shape[0]} rows, "
          f"launches per step: {tr.launches_per_step}")
    T, C, U = len(tr.feats), len(tr.inp.cont), tr.U
    hb = head_bytes(B, T, C, DIM, U)
    floor_us = sum(hb.values()) / HBM_BYTES_PER_S * 1e6
    print("head kernel bytes per step (computed): " + ", ".join(f"{k} {v / 1e6:.1f} MB" for k, v in hb.items())
          + f"; total {sum(hb.values()) / 1e6:.1f} MB = {floor_us:.1f} us at 3.35 TB/s")

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

    def step_block():
        for i in range(args.steps):
            tr.replay(*batches[i % 4])

    times = {"step": []}
    for blk in range(args.blocks + 1):
        for name, fn in (("step", step_block),):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            fn()
            t1.record()
            torch.cuda.synchronize()
            if blk > 0:
                times[name].append(t0.elapsed_time(t1) / args.steps)
    st = statistics.median(times["step"])
    print(f"train step: {st:.3f} ms (median of {len(times['step'])} blocks, range {min(times['step']):.3f}-{max(times['step']):.3f}), "
          f"{B / st / 1e3:.2f} M samples/s")


if __name__ == "__main__":
    main()
