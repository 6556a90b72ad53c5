#!/usr/bin/env python
"""Time two or more builds of the DLRM bottom tower kernel (mm_tower2_small) in one process, on the same inputs.

    python tools/tower_small_ab.py LIB [LIB ...] [--blocks 20] [--launches 200] [--batch 65536]

Each LIB is a libmm_b200.so (for example this tree's models_b200/_lib/libmm_b200.so and one built from another commit).
The inputs are those of the headline DLRM step (bench.py's `build_dlrm`): the 13 fp32 continuous columns as views into
a device copy of the packed input batch, the bottom block's split-bf16 weights and biases, and split-bf16 output rows
(the interaction kernel's operand format).

The libraries take turns, one block of `launches` back-to-back launches each (replayed as one CUDA graph), `blocks`
times, with one CUDA-event pair around each block.  The output of every library is compared with the first one's, bit for bit.  Prints the card name
and power limit, then one JSON line per library (median and range of the per-launch block means) and one with the
ratio of the block medians to the first library's.
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
import models_b200 as mm  # noqa: E402
from models_b200 import _cabi, datasets, ops  # noqa: E402
from models_b200.graph import _view  # noqa: E402
from interact_ab import card, load_lib  # noqa: E402


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
    from bench import build_dlrm, host_batches

    libs = [load_lib(p) for p in args.libs]
    _cabi._lib = libs[0]  # model set-up runs on the first library
    B = args.batch
    schema, model = build_dlrm(mm, datasets)
    model.build(dev)
    n_bufs = 4
    hosts = host_batches(datasets, schema, B, n_bufs)
    body = model.body
    pieces = []
    for h in hosts:
        hb = mm.HostBatch.like(h, model.input_columns(), id_bytes=model.id_bytes())
        pd = hb.buffer.to(dev)
        cols = body.continuous({f: _view(pd, hb.offsets[f], *hb.spec[f]) for f in hb.spec})
        pieces.append([cols[k] for k in sorted(cols)])
    assert all(t.dtype == torch.float32 for t in pieces[0]), "the headline columns are fp32"
    body.bottom_forward({f: t for f, t in zip(sorted(cols), pieces[0])}, operand_out=True)  # builds the block
    (l1, l2), tail = body.bottom_block.chain()
    assert tail is None
    w1, w2 = l1.split_kernel(), l2.split_kernel()
    outs = [torch.empty((B, 2 * l2.units), dtype=torch.bfloat16, device=dev) for _ in libs]

    def launch(j, i):
        ops.tower2_small(pieces[i % n_bufs], w1, l1.units, l1.bias, l1.activation, w2, l2.units, l2.bias, l2.activation,
                         out_split=outs[j])

    same = []
    for j, lib in enumerate(libs):
        _cabi._lib = lib
        outs[j].fill_(-1.0)
        launch(j, 0)
        torch.cuda.synchronize()
        same.append(bool(torch.equal(outs[j].view(torch.int16), outs[0].view(torch.int16))))

    # One CUDA graph of `launches` launches per library: called from Python, each launch costs more host time than the
    # kernel takes on the device, so eager launches would time the host.
    graphs = []
    for j, lib in enumerate(libs):
        _cabi._lib = lib
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(args.launches):
                launch(j, i)
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
