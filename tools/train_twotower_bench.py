"""Two-tower training step at bench.py's two-tower shape, captured as one CUDA graph.

    python tools/train_twotower_bench.py [--batch 16384] [--blocks 6] [--steps 20]
    python tools/train_twotower_bench.py --profile [--steps 20]

retrieval_10m_schema() (10 M x 64 item table, 1 M users), towers MLPBlock([256, 128]), in-batch negatives with false
negatives down-scored by item id, Adagrad(0.01), batch 16 384.  Prints the card's name, power limit and max SM clock read in
the same run, launches per step, and the median ms per step over --blocks blocks of --steps graph replays (CUDA events;
block 0 warms up), alternating with a block of the soft-max cross-entropy backward alone (mm_inbatch_softmax_ce_backward on
the trainer's own operands), with its achieved rate from the FLOPs computed from the shapes.  --profile (a separate run:
tracing slows the host) prints each kernel's device time per step under torch.profiler.
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
from models_b200.schema import Tags  # noqa: E402

TOWER = [256, 128]


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def ce_flops(B: int, N: int, D: int) -> dict:
    """2 B N D per product (fp32-equivalent; each is 3 split-bf16 MMAs): the forward recomputes the logits once; the
    backward recomputes them twice (dQ and dN kernels) and does the dQ and dN products."""
    p = 2 * B * N * D
    return {"forward": p, "backward": 4 * p}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16384)
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_twotower_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card()}")
    B = args.batch
    schema = datasets.retrieval_10m_schema()
    mm.set_seed(1)
    model = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock(TOWER))
    model.build(dev)
    model.compile(optimizer=mm.Adagrad(0.01))
    g = torch.Generator(device=dev).manual_seed(7)
    cats = [c for c in schema.select_by_tag(Tags.CATEGORICAL)]
    batches = []
    for _ in range(4):
        batches.append({c.name: torch.randint(0, c.int_domain.max + 1, (B,), generator=g, device=dev, dtype=torch.int32) for c in cats})
    tr = model.trainer(B)
    tr.capture(batches[0])
    D = tr.D
    fl = ce_flops(B, B, D)
    print(f"batch {B}, tower {TOWER}, output width {D}, launches per step: {tr.launches_per_step}")
    print("in-batch soft-max FLOP per step (2BND per product, fp32-equivalent): "
          + ", ".join(f"{k} {v / 1e9:.1f} G" for k, v in fl.items())
          + f" ({3 * sum(fl.values()) / 1e9:.1f} G of bf16 MMA work with the 3-pass split)")

    if args.profile:
        for i in range(5):
            tr.replay(batches[i % 4])
        torch.cuda.synchronize()
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            for i in range(args.steps):
                tr.replay(batches[i % 4])
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

    qs, its = tr.towers[0]["split"], tr.towers[1]["split"]
    q, it = (tr.towers[i]["y"] if tr.l2 else tr.towers[i]["h"][-1] for i in (0, 1))
    dq, di = torch.empty_like(q), torch.empty_like(it)
    ids = tr._static["item_id"]  # the captured graph's input buffer: the ids of the batch tr.stats and the operands hold
    c = torch.full((1,), 1.0 / B, device=dev)

    def bwd_block():
        for _ in range(args.steps):
            ops.inbatch_softmax_ce_backward(qs, its, D, tr.stats, q, it, c, dq, di, di, pos_ids=ids, neg_ids=ids,
                                            temperature=tr.temperature)

    def step_block():
        for i in range(args.steps):
            tr.replay(batches[i % 4])

    times = {"step": [], "bwd": []}
    for blk in range(args.blocks + 1):
        for name, fn in (("step", step_block), ("bwd", bwd_block)):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            fn()
            t1.record()
            torch.cuda.synchronize()
            if blk > 0:
                times[name].append(t0.elapsed_time(t1) / args.steps)
    st, bw = statistics.median(times["step"]), statistics.median(times["bwd"])
    print(f"train step: {st:.3f} ms (median of {len(times['step'])} blocks, range {min(times['step']):.3f}-{max(times['step']):.3f}), "
          f"{B / st / 1e3:.2f} M samples/s")
    bf = fl["backward"]
    print(f"mm_inbatch_softmax_ce_backward B = N = {B}, D = {D}: {bw:.3f} ms (range {min(times['bwd']):.3f}-{max(times['bwd']):.3f}), "
          f"{bf / bw / 1e9:.1f} TFLOP/s fp32-equivalent, {3 * bf / bw / 1e9:.1f} TFLOP/s of bf16 MMA work "
          f"({3 * bf / 989e12 * 1e3:.3f} ms at the data sheet's 989 TFLOP/s dense BF16)")


if __name__ == "__main__":
    main()
