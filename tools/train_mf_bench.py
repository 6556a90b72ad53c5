"""Matrix factorization training step at the two-tower benchmark's tables, captured as one CUDA graph.

    python tools/train_mf_bench.py [--batch 16384] [--blocks 6] [--steps 20]
    python tools/train_mf_bench.py --profile [--steps 20]

MatrixFactorizationModel(retrieval_10m_schema(), dim=64): a 10 M x 64 item-id table and a 1 M x 64 user-id table, in-batch
negatives with false negatives down-scored by item id, Adagrad(0.01), batch 16 384.  Two models, embeddings_l2_reg = 0 and
1e-4, each captured as one graph and timed in alternating blocks in the same run.  Prints the card's name, power limit and
max SM clock read in the same run, launches per step, and per model the median ms per step over --blocks blocks of --steps
graph replays (CUDA events; block 0 warms up), with the in-batch soft-max's bf16 MMA work per step over that time.
--profile (a separate run: tracing slows the host) prints each kernel's device time per step under torch.profiler.
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

DIM = 64
L2_REGS = (0.0, 1e-4)


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def mma_flops(B: int, D: int) -> int:
    """bf16 MMA work of one step's in-batch soft-max: 5 products of 2 B N D (N = B; the forward's logits, the backward's two
    recomputations and its dQ and dN products), each as 3 split-bf16 passes."""
    return 5 * 3 * 2 * B * B * D


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16384)
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_mf_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card()}")
    B = args.batch
    schema = datasets.retrieval_10m_schema()
    g = torch.Generator(device=dev).manual_seed(7)
    batches = [{c: torch.randint(0, schema.get(c).int_domain.max + 1, (B,), generator=g, device=dev, dtype=torch.int32)
                for c in ("user_id", "item_id")} for _ in range(4)]
    trainers = {}
    for lam in L2_REGS:
        mm.set_seed(1)
        model = mm.MatrixFactorizationModel(schema, DIM, embeddings_l2_reg=lam)
        model.build(dev)
        model.compile(optimizer=mm.Adagrad(0.01))
        tr = model.trainer(B)
        tr.capture(batches[0])
        trainers[lam] = tr
        print(f"embeddings_l2_reg {lam:g}: batch {B}, dim {DIM}, launches per step {tr.launches_per_step}")
    fl = mma_flops(B, DIM)
    print(f"in-batch soft-max bf16 MMA work per step: {fl / 1e9:.0f} GFLOP ({fl / 989e12 * 1e3:.2f} ms at the data sheet's "
          "989 TFLOP/s dense BF16)")

    if args.profile:
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        for lam, tr in trainers.items():
            for i in range(5):
                tr.replay(batches[i % 4])
            torch.cuda.synchronize()
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
            print(f"embeddings_l2_reg {lam:g}: device time per step by kernel ({args.steps} graph replays)")
            for us, n, name in rows:
                print(f"  {us:9.1f} us  {n:4.1f}x  {name[:110]}")
            print(f"  {sum(r[0] for r in rows):9.1f} us  sum of kernel times per step")
        return

    times = {lam: [] for lam in trainers}
    for blk in range(args.blocks + 1):
        for lam, tr in trainers.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for i in range(args.steps):
                tr.replay(batches[i % 4])
            t1.record()
            torch.cuda.synchronize()
            if blk > 0:
                times[lam].append(t0.elapsed_time(t1) / args.steps)
    for lam, ts in times.items():
        st = statistics.median(ts)
        loss = trainers[lam].loss
        print(f"embeddings_l2_reg {lam:g}: train step {st:.3f} ms (median of {len(ts)} blocks, range {min(ts):.3f}-{max(ts):.3f}), "
              f"{B / st / 1e3:.2f} M samples/s, {fl / st / 1e9:.0f} TFLOP/s of in-batch bf16 MMA work "
              f"({fl / 989e12 * 1e3 / st * 100:.0f} % of the data sheet's rate); last loss {float(loss[0].item()):.4f}, "
              f"regularization {float(loss[1].item()):.4g}")


if __name__ == "__main__":
    main()
