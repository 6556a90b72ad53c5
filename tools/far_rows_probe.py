#!/usr/bin/env python
"""Where the fused DLRM lookup + interaction kernel spends its time: HBM rows or the SM side.

    python tools/far_rows_probe.py [--launches 200] [--rounds 5] [--batch 65536]

Times `ops.dlrm_lookup_interact` with CUDA events, with the arguments of bench.py's headline `dominant()` launch
(operand-format table mirrors, packed ids at Model.id_bytes() widths, split-bf16 output), on three id sets:

  (a) uniform ids, as bench.py generates them;
  (b) (a) with the ids of every table of >= 65 536 rows folded to id % 4096, repacked at the same widths: the same
      instruction stream, but those rows now come from L2 instead of HBM;
  (c) every table folded: all rows from L2, the floor on the SM side.

The sets are timed alternately, `rounds` times `launches` launches each, one event pair per launch.  Prints the card
name and power limit, then one JSON line per id set (median over rounds of the per-round mean) and the gaps.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import models_b200 as mm  # noqa: E402
from models_b200 import datasets, ops  # noqa: E402
from models_b200.graph import _view  # noqa: E402

FAR_ROWS = 65536  # tables from this size up are read from HBM at random rows; shard_model's replication boundary
FOLD = 4096


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:  # the timing below does not depend on it
        return f"nvidia-smi unavailable: {type(e).__name__}: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=65536)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    print(card(), flush=True)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from bench import build_dlrm, host_batches

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
    far = [f for f, r in zip(names, rows) if r >= FAR_ROWS]
    slot_list = [slots[f] for f in names]
    devs = [{k: torch.from_numpy(v).to(dev) for k, v in h.items()} for h in hosts]
    bottoms = [body.bottom_forward(d, operand_out=operand) for d in devs]
    a_out = torch.empty((B, 2 * ops.tc_padded_k(body.output_width_before_top())), dtype=torch.bfloat16, device=dev)

    def id_set(fold):
        out = []
        for h in hosts:
            h2 = dict(h)
            for f in fold:
                h2[f] = np.asarray(h[f]) % FOLD
            hb = mm.HostBatch.like(h2, model.input_columns(), id_bytes=widths)
            pd = hb.buffer.to(dev)
            out.append((pd, [_view(pd, hb.offsets[f], *hb.spec[f]) for f in names]))
        return out

    sets = {"a_uniform": id_set([]), "b_far_tables_folded": id_set(far), "c_all_tables_folded": id_set(names)}

    def launch(s, i):
        ops.dlrm_lookup_interact(tables, s[i % n_bufs][1], slot_list, rows, 64, bottoms[i % n_bufs], slots["bottom_block"], a_out,
                                 operand_rows=operand)

    def time_set(s):
        ev = []
        for i in range(args.launches):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            launch(s, i)
            e1.record()
            ev.append((e0, e1))
        torch.cuda.synchronize()
        return float(np.mean([a.elapsed_time(b) for a, b in ev]))

    for s in sets.values():  # warm-up of every id set
        for i in range(10):
            launch(s, i)
    torch.cuda.synchronize()
    per = {k: [] for k in sets}
    for _ in range(args.rounds):
        for k, s in sets.items():
            per[k].append(time_set(s))
    med = {k: float(np.median(v)) for k, v in per.items()}
    for k in sets:
        print(json.dumps({"id_set": k, "kernel_ms_median": med[k], "kernel_ms_rounds": per[k], "launches_per_round": args.launches}))
    a, b, c = med["a_uniform"], med["b_far_tables_folded"], med["c_all_tables_folded"]
    print(json.dumps({"far_tables": far, "b_faster_than_a": 1.0 - b / a, "c_faster_than_a": 1.0 - c / a,
                      "table_mirror": bool(operand), "batch": B}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
