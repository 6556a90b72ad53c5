"""Training step of the multi-task Model(InputBlockV2, MMOEBlock, OutputBlock) at the Criteo shape, captured as one CUDA
graph, in two legs, and the fused gate + mixture + heads kernel (mm_mmoe_heads_fwd_bwd) timed alone against its computed
byte floor.

    python tools/train_mmoe_bench.py [--batch 65536] [--blocks 6] [--steps 20] [--max-rows 4000000]

Criteo schema with click / conversion (binary) and rating (regression) targets, tables capped at --max-rows rows, inferred
embedding widths (d = 941 at the default cap), Adagrad(0.01), MMOEBlock(4 experts of MLPBlock([64])).  Leg (a): no towers
and no gate block (the fused kernel); leg (b): the multi-task notebook's configuration, task_blocks=MLPBlock([32]) and
gate_block=MLPBlock([16]).  Prints the card's name and power limit read in the same run, launches per step, each leg's
median ms per step and samples/s over the blocks (CUDA events around --steps graph replays per block), and the fused
kernel's median time over 5 x 40 launches against the time its bytes take at 3.35 TB/s.
"""
import argparse
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import models_b200 as mm  # noqa: E402
from models_b200 import datasets, ops  # noqa: E402
from models_b200.schema import ColumnSchema, Schema, Tags  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def floor_bytes(B: int, E: int, U: int, H: int) -> int:
    """What mm_mmoe_heads_fwd_bwd must move: X read and dX written (B E U fp32 each), the gate logits read and their
    gradient written (B H E each), the targets (two int64 binary columns and one fp32 rating here) and H logits written."""
    return 4 * 2 * B * E * U + 4 * 2 * B * H * E + (8 + 8 + 4) * B + 4 * B * H


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--max-rows", type=int, default=4_000_000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_mmoe_bench.py needs a CUDA device")
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
        ys = [(torch.rand(B, generator=g, device=dev) < 0.3).long(), (torch.rand(B, generator=g, device=dev) < 0.05).long(),
              torch.rand(B, generator=g, device=dev) * 5.0]
        batches.append((x, ys))
    E, U = 4, 64

    def leg(name, towers, gate):
        mm.set_seed(1)
        out = mm.OutputBlock(schema, task_blocks=towers)
        model = mm.Model(mm.InputBlockV2(schema), mm.MMOEBlock(out, expert_block=mm.MLPBlock([U]), num_experts=E, gate_block=gate),
                         out)
        model.build(dev)
        model.compile(optimizer=mm.Adagrad(0.01))
        tr = model.trainer(B)
        tr.capture(batches[0][0], batches[0][1])
        print(f"{name}: batch {B}, d = {model.body.input_width()}, launches per step {tr.launches_per_step}")
        times = []
        for blk in range(args.blocks + 1):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for i in range(args.steps):
                tr.replay(*batches[i % 4])
            t1.record()
            torch.cuda.synchronize()
            if blk > 0:  # block 0 warms up
                times.append(t0.elapsed_time(t1) / args.steps)
        med = statistics.median(times)
        print(f"  step: {med:.3f} ms (median of {len(times)} blocks, range {min(times):.3f}-{max(times):.3f}), "
              f"{B / med / 1e3:.2f} M samples/s")
        return model, tr

    leg("leg (b) task_blocks=MLPBlock([32]), gate_block=MLPBlock([16])", mm.MLPBlock([32]), mm.MLPBlock([16]))
    torch.cuda.empty_cache()
    model, tr = leg("leg (a) fused heads, no towers, no gate block", None, None)
    # the fused kernel alone, with the training step's arguments on the trainer's own buffers (gradients into scratch)
    mo, H = model.body.mmoe, tr.H
    G = tr.G
    loss = torch.zeros(1 + H, device=dev)
    dw, db = torch.zeros_like(tr.head.kernel), torch.zeros_like(tr.head.bias)
    ys = batches[0][1]

    def call():
        ops.mmoe_heads_fwd_bwd(tr.X, E, mo.gate_logits(tr.L), mo.temperature, tr.head.kernel, tr.head.bias, tr.losses, ys,
                               tr.logits.view(H, B), loss, dx=G[:, :tr.EU], d_gate_logits=mo.gate_logits(G[:, tr.EU:]), dw=dw, db=db,
                               loss_weights=tr.loss_weights, mask_relu=True)

    for _ in range(20):
        call()
    ks = []
    for _ in range(5):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(40):
            call()
        t1.record()
        torch.cuda.synchronize()
        ks.append(t0.elapsed_time(t1) / 40 * 1e3)
    kt = statistics.median(ks)
    nbytes = floor_bytes(B, E, U, H)
    fl = nbytes / HBM_BYTES_PER_S * 1e6
    print(f"mm_mmoe_heads_fwd_bwd: {kt:.1f} us (median of 5 x 40 launches); computed floor {nbytes / 1e6:.1f} MB = "
          f"{fl:.1f} us at 3.35 TB/s; floor / measured = {fl / kt:.2f}")


if __name__ == "__main__":
    main()
