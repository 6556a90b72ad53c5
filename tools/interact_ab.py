#!/usr/bin/env python
"""Time two or more builds of the fused DLRM lookup + interaction kernel in one process, on the same inputs.

    python tools/interact_ab.py LIB [LIB ...] [--blocks 20] [--launches 50] [--batch 65536] [--id-set uniform|far-folded]

Each LIB is a libmm_b200.so (for example this tree's models_b200/_lib/libmm_b200.so and one built from another commit).
The inputs are those of bench.py's headline `dominant()` launch: operand-format table mirrors, packed ids at
Model.id_bytes() widths, the bottom tower's split-bf16 rows, split-bf16 output.  `--id-set far-folded` folds the ids of
every table of >= 65 536 rows to id % 4096 (their rows then come from L2), as tools/far_rows_probe.py does.

The libraries take turns, one block of `launches` back-to-back launches each, `blocks` times, with one CUDA-event pair
around each block.  The output of every library is compared with the first one's, bit for bit.  Prints the card name
and power limit, then one JSON line per library (median and range of the per-launch block means) and one with the
ratio of the block medians to the first library's.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import models_b200 as mm  # noqa: E402
from models_b200 import _cabi, datasets, ops  # noqa: E402
from models_b200.graph import _view  # noqa: E402

FAR_ROWS = 65536
FOLD = 4096


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:  # the timing below does not depend on it
        return f"nvidia-smi unavailable: {type(e).__name__}: {e}"


def load_lib(path):
    lib = C.CDLL(os.fspath(Path(path).resolve()))
    for name, (res, args) in _cabi.SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+")
    ap.add_argument("--blocks", type=int, default=20)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--id-set", choices=["uniform", "far-folded"], default="uniform")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    print(card(), flush=True)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from bench import build_dlrm, host_batches

    libs = [load_lib(p) for p in args.libs]
    _cabi._lib = libs[0]  # model set-up (tables, mirrors, bottom tower) runs on the first library
    B = args.batch
    schema, model = build_dlrm(mm, datasets)
    model.build(dev)
    n_bufs = 4
    hosts = host_batches(datasets, schema, B, n_bufs)
    widths = model.id_bytes()
    body = model.body
    slots = body.slots()
    names = body.embeddings.feature_names
    operand = body.use_operand_rows()
    tabs = [body.embeddings.feature_to_table[f] for f in names]
    tables = [t.operand_mirror() if operand else t.table for t in tabs]
    rows = [t.table.shape[0] for t in tabs]
    fold = [f for f, r in zip(names, rows) if r >= FAR_ROWS] if args.id_set == "far-folded" else []
    slot_list = [slots[f] for f in names]
    idx = []
    for h in hosts:
        h2 = dict(h)
        for f in fold:
            h2[f] = np.asarray(h[f]) % FOLD
        hb = mm.HostBatch.like(h2, model.input_columns(), id_bytes=widths)
        pd = hb.buffer.to(dev)
        idx.append((pd, [_view(pd, hb.offsets[f], *hb.spec[f]) for f in names]))
    devs = [{k: torch.from_numpy(v).to(dev) for k, v in h.items()} for h in hosts]
    bottoms = [body.bottom_forward(d, operand_out=operand) for d in devs]
    width = 2 * ops.tc_padded_k(body.output_width_before_top())
    outs = [torch.empty((B, width), dtype=torch.bfloat16, device=dev) for _ in libs]
    oob = torch.zeros(1, dtype=torch.int32, device=dev)

    def launch(j, i):
        ops.dlrm_lookup_interact(tables, idx[i % n_bufs][1], slot_list, rows, 64, bottoms[i % n_bufs], slots["bottom_block"],
                                 outs[j], oob=oob, operand_rows=operand)

    # same inputs for every library: identical output rows and out-of-range counts
    same, oobs = [], []
    for j, lib in enumerate(libs):
        _cabi._lib = lib
        oob.zero_()
        launch(j, 0)
        torch.cuda.synchronize()
        oobs.append(int(oob.item()))
        same.append(bool(torch.equal(outs[j].view(torch.int16), outs[0].view(torch.int16))))

    for j, lib in enumerate(libs):  # warm-up
        _cabi._lib = lib
        for i in range(10):
            launch(j, i)
    torch.cuda.synchronize()
    per = [[] for _ in libs]
    for _ in range(args.blocks):
        for j, lib in enumerate(libs):
            _cabi._lib = lib
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.launches):
                launch(j, i)
            e1.record()
            torch.cuda.synchronize()
            per[j].append(e0.elapsed_time(e1) / args.launches)
    med = [float(np.median(v)) for v in per]
    for j, p in enumerate(args.libs):
        print(json.dumps({"lib": p, "kernel_ms_median": med[j], "kernel_ms_min": float(np.min(per[j])),
                          "kernel_ms_max": float(np.max(per[j])), "bit_identical_to_first": same[j], "oob_count": oobs[j],
                          "blocks": args.blocks, "launches_per_block": args.launches, "id_set": args.id_set}))
    ratios = [[b / a for a, b in zip(per[0], per[j])] for j in range(len(libs))]
    print(json.dumps({"median_ratio_to_first": [float(np.median(r)) for r in ratios],
                      "max_ratio_to_first": [float(np.max(r)) for r in ratios]}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
