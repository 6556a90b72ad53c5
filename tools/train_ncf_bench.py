"""NCFModel training step at the two-tower benchmark's id tables, captured as one CUDA graph, and its fused head kernel.

    python tools/train_ncf_bench.py [--batch 65536] [--blocks 6] [--steps 20]

NCFModel(retrieval_10m_schema()'s user_id / item_id columns + a binary `click` target, embedding_dim=64,
MLPBlock([256, 64])): four tables (GMF and MLP branch, 1 M x 64 users and 10 M x 64 items each), Adagrad(0.01), batch
65 536.  Two models, embeddings_l2_reg = 0 and 1e-4, each captured as one graph and timed in alternating blocks in the same
run.  Prints the card's name, power limit and max SM clock read in the same run, launches per step, and per model the
median ms per step and samples/s over --blocks blocks of --steps graph replays (CUDA events; block 0 warms up).  Then
mm_ncf_head_fwd_bwd alone (the training form, on the model's own buffers) against its byte floor, computed here from the
shapes: per sample the two ids, the two GMF rows read, h read, du / di / dh written and the logit written.
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

DIM, UNITS = 64, (256, 64)
L2_REGS = (0.0, 1e-4)
HBM_BYTES_PER_S = 3.35e12  # the data sheet's H100 SXM HBM3 bandwidth


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def head_bytes(B: int, D: int, U: int, H: int, id_bytes: int) -> int:
    """Bytes mm_ncf_head_fwd_bwd must move per call: ids, u and i read, h read, du, di, dh written, logits written."""
    return B * (2 * id_bytes + 2 * D * 4 + U * 4 + 2 * D * 4 + U * 4 + H * 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_ncf_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card()}")
    B = args.batch
    base = datasets.retrieval_10m_schema()
    schema = Schema([base.get("user_id"), base.get("item_id"),
                     ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64")])
    g = torch.Generator(device=dev).manual_seed(7)
    batches = [({c: torch.randint(0, schema.get(c).int_domain.max + 1, (B,), generator=g, device=dev, dtype=torch.int32)
                 for c in ("user_id", "item_id")}, torch.randint(0, 2, (B,), generator=g, device=dev).float()) for _ in range(4)]
    trainers = {}
    for lam in L2_REGS:
        mm.set_seed(1)
        model = mm.benchmark.NCFModel(schema, DIM, mm.MLPBlock(list(UNITS)), embeddings_l2_reg=lam)
        model.build(dev)
        model.compile(optimizer=mm.Adagrad(0.01))
        tr = model.trainer(B)
        tr.capture(batches[0][0], [batches[0][1]])
        trainers[lam] = tr
        print(f"embeddings_l2_reg {lam:g}: batch {B}, dim {DIM}, mlp {list(UNITS)}, launches per step {tr.launches_per_step}")

    times = {lam: [] for lam in trainers}
    for blk in range(args.blocks + 1):
        for lam, tr in trainers.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for i in range(args.steps):
                x, y = batches[i % 4]
                tr.replay(x, [y])
            t1.record()
            torch.cuda.synchronize()
            if blk > 0:
                times[lam].append(t0.elapsed_time(t1) / args.steps)
    for lam, ts in times.items():
        st = statistics.median(ts)
        tr = trainers[lam]
        print(f"embeddings_l2_reg {lam:g}: train step {st:.3f} ms (median of {len(ts)} blocks, range {min(ts):.3f}-{max(ts):.3f}), "
              f"{B / st / 1e3:.2f} M samples/s; last loss {float(tr.loss[0].item()):.4f}, regularization "
              f"{float(tr.regularization.item()):.4g}")

    # the head kernel alone, training form, on the l2 = 1e-4 trainer's buffers
    tr = trainers[L2_REGS[-1]]
    x, y = batches[1]
    a, hi = tr.arena, len(tr.arena.layers) - 1
    h, dh = tr.h[-1][:B], tr.dh[-1][:B]
    logits = tr.logits.view(-1)[:B].view(1, B)
    loss = torch.zeros(2, dtype=torch.float32, device=dev)
    reg = torch.zeros(1, dtype=torch.float32, device=dev)

    def head():
        ops.ncf_head_fwd_bwd(tr.tables[tr.t_u].table, x["user_id"], tr.tables[tr.t_i].table, x["item_id"], h, tr.head.kernel,
                             tr.head.bias, tr.losses, [y], logits, loss=loss, reg=reg, l2=1e-4, du=tr.slices[tr.t_u][:B],
                             di=tr.slices[tr.t_i][:B], dh=dh, dw=a.view(a.grad, hi, "kernel"), db=a.view(a.grad, hi, "bias"),
                             relu_h=True, oob=tr.oob)

    for _ in range(20):
        head()
    ks = []
    for _ in range(args.blocks):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(100):
            head()
        t1.record()
        torch.cuda.synchronize()
        ks.append(t0.elapsed_time(t1) / 100 * 1e3)
    a.grad.zero_()
    us = statistics.median(ks)
    nb = head_bytes(B, DIM, UNITS[-1], 1, 4)
    floor = nb / HBM_BYTES_PER_S * 1e6
    print(f"mm_ncf_head_fwd_bwd: {us:.1f} us per call (median of {len(ks)} blocks of 100, range {min(ks):.1f}-{max(ks):.1f}); "
          f"byte floor {nb / 1e6:.1f} MB = {floor:.1f} us at the data sheet's 3.35 TB/s ({us / floor:.2f}x the floor, "
          f"{nb / us / 1e6:.2f} TB/s achieved)")


if __name__ == "__main__":
    main()
