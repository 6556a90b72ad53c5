"""Two-tower training step with each pairwise ranking loss against the soft-max cross-entropy step, at
tools/train_twotower_bench.py's shape, each captured as one CUDA graph.

    python tools/train_pairwise_bench.py [--batch 16384] [--blocks 4] [--steps 10] [--kinds bpr,bpr-max,...]

retrieval_10m_schema() (10 M x 64 item table, 1 M users), towers MLPBlock([256, 128]), in-batch negatives with false
negatives down-scored by item id, Adagrad(0.01), batch 16 384.  Prints the card's name, power limit and clocks read in the
same run; then per loss kind: launches per step and the median ms per step over --blocks blocks of --steps graph replays
(CUDA events; block 0 warms up), alternating with blocks of the cross-entropy step, and the pairwise forward
(mm_inbatch_pairwise_fwd) and backward (mm_inbatch_pairwise_bwd) alone on the trainer's own operands, with their rates
from the MMA FLOPs computed from the shapes.
"""
import argparse
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import models_b200 as mm  # noqa: E402
from models_b200 import _cabi, datasets, ops  # noqa: E402
from models_b200.schema import Tags  # noqa: E402

TOWER = [256, 128]


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def pairwise_flops(B: int, N: int, D: int, kind: str) -> dict:
    """2 B N D per product (fp32-equivalent; each is 3 split-bf16 MMAs): the forward recomputes the scores once (twice for
    the -max kinds: the log-sum-exp pass); the backward recomputes them twice (dQ and dN kernels) and does the dQ and dN
    products."""
    p = 2 * B * N * D
    return {"forward": (2 if kind in ("bpr-max", "top1-max") else 1) * p, "backward": 4 * p}


def timed(fn, steps: int) -> float:
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(steps):
        fn(i)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16384)
    ap.add_argument("--blocks", type=int, default=4)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--kinds", default=",".join(_cabi.PAIRWISE_KINDS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_pairwise_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card (name, power limit, SM clock, max SM clock): {card()}")
    B = args.batch
    schema = datasets.retrieval_10m_schema()
    mm.set_seed(1)
    model = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock(TOWER))
    model.build(dev)
    g = torch.Generator(device=dev).manual_seed(7)
    cats = [c for c in schema.select_by_tag(Tags.CATEGORICAL)]
    batches = [{c.name: torch.randint(0, c.int_domain.max + 1, (B,), generator=g, device=dev, dtype=torch.int32) for c in cats}
               for _ in range(4)]

    def trainer(loss):
        model.compile(optimizer=mm.Adagrad(0.01), loss=loss)
        tr = model.trainer(B)
        tr.capture(batches[0])
        return tr

    ce = trainer(None)
    D = ce.D
    print(f"batch {B}, tower {TOWER}, output width {D}; categorical_crossentropy: {ce.launches_per_step} launches per step")
    ce_times = []
    for kind in args.kinds.split(","):
        tr = trainer(kind)
        times = {"step": [], "ce": [], "fwd": [], "bwd": []}
        qs, its = tr.towers[0]["split"], tr.towers[1]["split"]
        q, it = (tr.towers[i]["y"] if tr.l2 else tr.towers[i]["h"][-1] for i in (0, 1))
        dq, di = torch.empty_like(q), torch.empty_like(it)
        ids = tr._static["item_id"]  # the captured graph's input buffer: the ids of the batch the operands hold
        kw = dict(pos_ids=ids, neg_ids=ids, temperature=tr.temperature)
        stats = torch.empty_like(tr.stats)
        blocks = {"step": lambda i: tr.replay(batches[i % 4]), "ce": lambda i: ce.replay(batches[i % 4]),
                  "fwd": lambda i: ops.inbatch_pairwise(qs, its, D, tr.pos_logit, stats, kind, **kw),
                  "bwd": lambda i: ops.inbatch_pairwise_backward(qs, its, D, tr.pos_logit, stats, q, it, dq, di, di, kind, **kw)}
        for blk in range(args.blocks + 1):
            for name, fn in blocks.items():
                t = timed(fn, args.steps)
                if blk > 0:
                    times[name].append(t)
        ce_times += times["ce"]
        med = {k: statistics.median(v) for k, v in times.items()}
        fl = pairwise_flops(B, B, D, kind)
        print(f"{kind}: {tr.launches_per_step} launches per step; train step {med['step']:.3f} ms "
              f"(range {min(times['step']):.3f}-{max(times['step']):.3f}) vs categorical_crossentropy {med['ce']:.3f} ms "
              f"in the alternating blocks ({med['step'] / med['ce']:.2f}x)")
        for part in ("fwd", "bwd"):
            f = fl["forward" if part == "fwd" else "backward"]
            print(f"  mm_inbatch_pairwise_{part}: {med[part]:.3f} ms (range {min(times[part]):.3f}-{max(times[part]):.3f}), "
                  f"{f / med[part] / 1e9:.1f} TFLOP/s fp32-equivalent, {3 * f / med[part] / 1e9:.1f} TFLOP/s of bf16 MMA work")
        del tr
    print(f"categorical_crossentropy step over all blocks: median {statistics.median(ce_times):.3f} ms "
          f"(range {min(ce_times):.3f}-{max(ce_times):.3f})")
    print(f"card after the run: {card()}")


if __name__ == "__main__":
    main()
