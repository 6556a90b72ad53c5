#!/usr/bin/env python
"""ONE process, TWO GPUs: the fused lookup+interaction kernel on GPU 0 with half of every Criteo-TB table on GPU 1
(peer access), timed (a) with GPU 1 idle, (b) with GPU 1 running the mirrored kernel.  Separates requester-side
from serving-side effects of the NVLink row reads.  Can run under ncu (single process).

    python tools/probe/fused_peer.py [--batch 65536] [--tables all|big]
"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))
from models_b200 import datasets, ops  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--only-idle", action="store_true")
    args = ap.parse_args()
    B, D, W = args.batch, 64, 2
    rows = datasets.CRITEO_TB_ROWS
    T = len(rows)
    devs = [torch.device("cuda", 0), torch.device("cuda", 1)]
    shards = [[], []]
    for k in range(W):
        torch.cuda.set_device(k)
        for r in rows:
            lr = max((r - k + W - 1) // W, 1)
            w = torch.empty((lr, D), dtype=torch.float32, device=devs[k])
            w.uniform_(-0.05, 0.05)
            shards[k].append(w)
    # whole copies of the small tables on both GPUs (for the placements that replicate them)
    full = [[], []]
    for k in range(W):
        torch.cuda.set_device(k)
        for r in rows:
            full[k].append(torch.empty((r, D), dtype=torch.float32, device=devs[k]).uniform_(-0.05, 0.05) if r < 65536 else None)
    # enable peer access both ways (torch does it on the first peer copy)
    a = torch.zeros(4, device=devs[0]); b = a.to(devs[1]); a.copy_(b); torch.cuda.synchronize(0); torch.cuda.synchronize(1)
    F = T + 1
    Kp = ops.tc_padded_k(D + F * (F - 1) // 2)
    rng = np.random.default_rng(3)
    state = []
    for k in range(W):
        torch.cuda.set_device(k)
        idx = [[torch.from_numpy(rng.integers(0, r, B).astype(np.int32)).to(devs[k]) for r in rows] for _ in range(3)]
        bottom = torch.randn((B, D), device=devs[k])
        out = torch.empty((B, 2 * Kp), dtype=torch.bfloat16, device=devs[k])
        peers = [[shards[0][t].data_ptr(), shards[1][t].data_ptr()] for t in range(T)]
        state.append((idx, bottom, out, peers))

    def launch(k, i, sharded_tables):
        torch.cuda.set_device(k)
        idx, bottom, out, peers = state[k]
        weights = [shards[k][t] if sharded_tables(t) else full[k][t] for t in range(T)]
        ops.dlrm_lookup_interact(weights, idx[i % 3], list(range(T)), rows, D, bottom, T, out,
                                 peers=[peers[t] if sharded_tables(t) else None for t in range(T)], rank=k, world=W)

    def timed(label, sharded_tables, both):
        for i in range(3):
            launch(0, i, sharded_tables)
            if both:
                launch(1, i, sharded_tables)
        torch.cuda.synchronize(0); torch.cuda.synchronize(1)
        torch.cuda.set_device(0)
        evs = []
        for i in range(args.iters):
            torch.cuda.set_device(0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            launch(0, i, sharded_tables)
            e1.record()
            evs.append((e0, e1))
            if both:
                launch(1, i, sharded_tables)
        torch.cuda.synchronize(0); torch.cuda.synchronize(1)
        ms = float(np.mean([x.elapsed_time(y) for x, y in evs]))
        n_sh = sum(1 for t in range(T) if sharded_tables(t))
        remote = B * n_sh * 0.5 * 256
        print(json.dumps({"case": label, "peer_busy": both, "tables_sharded": n_sh, "kernel_ms": ms,
                          "remote_GBps": remote / (ms * 1e-3) / 1e9}), flush=True)

    timed("all 26 tables sharded", lambda t: True, False)
    if not args.only_idle:
        timed("all 26 tables sharded", lambda t: True, True)
        timed("tables >= 1 000 rows sharded (18), smaller ones replicated", lambda t: rows[t] >= 1000, True)
        timed("tables >= 65 536 rows sharded (8), smaller ones replicated", lambda t: rows[t] >= 65536, False)
        timed("tables >= 65 536 rows sharded (8), smaller ones replicated", lambda t: rows[t] >= 65536, True)


if __name__ == "__main__":
    main()
