#!/usr/bin/env python
"""Run ONE kernel a few times (for `ncu --set full -k regex:...` captures; never a timing source).

    python tools/run_kernel.py dense_tc [K N]   |   gather   |   fused   |   interact   |   scores
"""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import models_b200 as mm  # noqa: E402
from models_b200 import datasets, ops  # noqa: E402

dev = torch.device("cuda", 0)
what = sys.argv[1] if len(sys.argv) > 1 else "dense_tc"
B = 65536
if what == "dense_tc":
    K = int(sys.argv[2]) if len(sys.argv) > 2 else 415
    N = int(sys.argv[3]) if len(sys.argv) > 3 else 128
    x = torch.randn((B, K), device=dev)
    W = torch.randn((K, N), device=dev) * 0.05
    b = torch.zeros(N, device=dev)
    a = ops.split_rows(x)
    w = ops.split_weights(W)
    nxt = torch.zeros((B, 2 * ops.tc_padded_k(N)), dtype=torch.bfloat16, device=dev)
    for _ in range(5):
        ops.dense_tc(a, K, w, N, b, "relu", out_split=nxt)
elif what in ("gather", "fused", "fused_operand", "interact"):
    T, D = 26, 64
    F = T + 1
    schema = datasets.criteo_schema()
    cat = schema.select_by_tag(mm.Tags.CATEGORICAL)
    emb = mm.Embeddings(cat, dim=D, embeddings_initializer={"hash_seed": 4321})
    emb.build(dev)
    names = emb.feature_names
    slots = {n: i for i, n in enumerate(sorted(names + ["bottom_block"]))}
    idxs = []
    for i in range(4):  # rotating batches: the captured launch sees rows that are not L2-resident
        b = datasets.generate_batch(cat, B, seed=100 + i, index_law="uniform")
        idxs.append([torch.from_numpy(b[n]).to(dev) for n in names])
    tables = [emb.feature_to_table[n].table for n in names]
    stack = torch.empty((B, F * D), dtype=torch.float32, device=dev)
    bottom = torch.randn((B, D), device=dev)
    out = torch.empty((B, 2 * ops.tc_padded_k(D + F * (F - 1) // 2)), dtype=torch.bfloat16, device=dev)
    xs = [torch.randn((B, F, D), device=dev) for _ in range(2)]
    for i in range(6):
        idx = idxs[i % 4]
        if what == "gather":
            ops.gather_multi(tables, idx, [slots[n] * D for n in names], stack)
        elif what == "fused":
            ops.dlrm_lookup_interact(tables, idx, [slots[n] for n in names], [t.shape[0] for t in tables], D, bottom,
                                     slots["bottom_block"], out)
        elif what == "fused_operand":
            if i == 0:
                mirrors, bottom_op = [ops.split_rows(t) for t in tables], ops.split_rows(bottom)
            ops.dlrm_lookup_interact(mirrors, idx, [slots[n] for n in names], [t.shape[0] for t in tables], D, bottom_op,
                                     slots["bottom_block"], out, operand_rows=True)
        else:
            ops.dot_interaction(xs[i % 2], out, prefix=bottom)
elif what == "bottom":
    mm.set_seed(3)
    cols = {f"I{i}": torch.rand(B, device=dev) for i in range(1, 14)}
    mlp = mm.MLPBlock([128, 64])
    for _ in range(6):
        mlp(cols, operand_out=True)
elif what == "scores":
    Bq, Dq = 16384, int(sys.argv[2]) if len(sys.argv) > 2 else 128
    q = torch.randn((Bq, Dq), device=dev)
    it = torch.randn((Bq, Dq), device=dev)
    ids = torch.randint(0, 10_000_000, (Bq,), device=dev, dtype=torch.int64)
    o = torch.empty((Bq, Bq + 4), device=dev)[:, 3:4 + Bq]  # (B, 1+B) view whose negatives start 16-byte aligned
    for _ in range(3):
        ops.inbatch_scores(q, it, it, o, pos_ids=ids, neg_ids=ids)
torch.cuda.synchronize()
print("done", what)
