#!/usr/bin/env python
"""Time two or more builds of the DLRM top tower kernel (mm_mlp_tc) in one process, on the same inputs.

    python tools/mlp_tc_ab.py LIB [LIB ...] [--blocks 20] [--launches 200] [--batch 65536]

Each LIB is a libmm_b200.so (for example this tree's models_b200/_lib/libmm_b200.so and one built from another commit).
The inputs have the headline DLRM step's top-tower shape: (B, 415) split-bf16 rows of pitch 2 * 448 (the interaction
kernel's operand format), the [128, 64, 32] relu tower and the fused sigmoid head, seeded as in tools/step_profile.py.

The libraries take turns, one block of `launches` back-to-back launches each (replayed as one CUDA graph), `blocks`
times, with one CUDA-event pair around each block.  The head output of every library is compared with the first one's,
bit for bit, and so are the fp32 rows of the last layer (one more launch with `out`), the multi-head output
(mm_mlp_tc_heads, 3 heads) and a batch that is not a multiple of the tile height.  Prints the card name and power limit,
then one JSON line per library (median and range of the per-launch block means) and one with the ratio of the block
medians to the first library's.
"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from models_b200 import _cabi, ops  # noqa: E402
from interact_ab import card, load_lib  # noqa: E402


def tower_inputs(B, dev):
    g = torch.Generator(device="cpu").manual_seed(7)
    K, widths = 415, [128, 64, 32]
    x = torch.randn((B, K), generator=g).mul_(0.5).to(dev)
    a = ops.split_rows(x)
    ws, bs, k = [], [], K
    for w in widths:
        W = (torch.randn((k, w), generator=g) * (2.0 / (k + w)) ** 0.5).to(dev)
        ws.append(ops.split_weights(W))
        bs.append((torch.randn(w, generator=g) * 0.01).to(dev))
        k = w
    head_w = (torch.randn(32, generator=g) * 0.2).to(dev)
    heads_w = (torch.randn((32, 3), generator=g) * 0.2).to(dev)
    heads_b = (torch.randn(3, generator=g) * 0.1).to(dev)
    return K, widths, a, ws, bs, head_w, heads_w, heads_b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+")
    ap.add_argument("--blocks", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--batch", type=int, default=65536)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    print(card(), flush=True)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    libs = [load_lib(p) for p in args.libs]
    _cabi._lib = libs[0]
    B = args.batch
    K, widths, a, ws, bs, head_w, heads_w, heads_b = tower_inputs(B, dev)
    acts = ["relu"] * 3
    heads = [torch.empty((B, 1), dtype=torch.float32, device=dev) for _ in libs]

    def launch(j):
        ops.mlp_tc(a, K, ws, widths, bs, acts, head_w=head_w, head_b=0.01, head_act="sigmoid", head_out=heads[j])

    def extra_outputs():
        rows = torch.full((B, widths[-1]), 7.0, dtype=torch.float32, device=dev)
        h = torch.empty((B, 1), dtype=torch.float32, device=dev)
        ops.mlp_tc(a, K, ws, widths, bs, acts, out=rows, head_w=head_w, head_b=0.01, head_act="sigmoid", head_out=h)
        multi = torch.empty((3, B), dtype=torch.float32, device=dev)
        ops.mlp_tc_heads(a, K, ws, widths, bs, acts, heads_w, heads_b, ["sigmoid", "linear", "relu"], multi)
        odd = B - 37
        tail = torch.full((odd, widths[-1]), 7.0, dtype=torch.float32, device=dev)
        ops.mlp_tc(a[:odd].contiguous(), K, ws, widths, bs, acts, out=tail)
        return [rows, h, multi, tail]

    same, firsts = [], None
    for j, lib in enumerate(libs):
        _cabi._lib = lib
        heads[j].fill_(-1.0)
        launch(j)
        extra = extra_outputs()
        torch.cuda.synchronize()
        outs = [heads[j]] + extra
        if firsts is None:
            firsts = outs
        same.append(all(torch.equal(o.view(torch.int32), f.view(torch.int32)) for o, f in zip(outs, firsts)))

    # One CUDA graph of `launches` launches per library: called from Python, each launch costs more host time than the
    # kernel takes on the device, so eager launches would time the host.
    graphs = []
    for j, lib in enumerate(libs):
        _cabi._lib = lib
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(args.launches):
                launch(j)
        graphs.append(g)
    for g in graphs:  # warm-up
        g.replay()
    torch.cuda.synchronize()
    per = [[] for _ in libs]
    for _ in range(args.blocks):
        for j, g in enumerate(graphs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            per[j].append(e0.elapsed_time(e1) / args.launches)
    med = [float(np.median(v)) for v in per]
    for j, p in enumerate(args.libs):
        print(json.dumps({"lib": p, "kernel_us_median": 1e3 * med[j], "kernel_us_min": 1e3 * float(np.min(per[j])),
                          "kernel_us_max": 1e3 * float(np.max(per[j])), "bit_identical_to_first": same[j],
                          "blocks": args.blocks, "launches_per_block": args.launches, "batch": B}))
    ratios = [[b / a for a, b in zip(per[0], per[j])] for j in range(len(libs))]
    print(json.dumps({"median_ratio_to_first": [float(np.median(r)) for r in ratios],
                      "max_ratio_to_first": [float(np.max(r)) for r in ratios]}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
