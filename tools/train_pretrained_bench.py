"""Cost of a pretrained feature in a DCN training step: the Criteo schema (26 tables of width 16, 13 continuous columns) plus
one pretrained feature of Dp = 768 looked up by a categorical column, B = 65 536, Adagrad, every step one CUDA-graph replay.

Legs, timed in alternating blocks in one process with CUDA events:
  none          the Criteo DCN without the pretrained feature
  unprojected   the 768 floats per sample gathered straight into x0 (mm_pretrained_gather)
  projected64   PretrainedEmbeddings(output_dims=64): gather + projection fused (mm_pretrained_project), its backward
                (mm_pretrained_project_backward) in the step
and the fused gather + projection kernel alone (20 launches per CUDA graph) against its byte floor: the B Dp 4 bytes
gathered, the ids, W and the slot written, over 3.35 TB/s.  Prints one JSON line with the card's name and power limit.

    python tools/train_pretrained_bench.py [--batch 65536] [--dp 768] [--steps 20] [--blocks 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import models_b200 as mm  # noqa: E402
from models_b200 import datasets, ops  # noqa: E402
from models_b200.graph import graph_capture  # noqa: E402

KERNELS_PER_GRAPH = 20
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
LOOKUP = "C3"


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        out["power_limit, max_sm_clock"] = q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        out["power_limit, max_sm_clock"] = "unknown"
    return out


def timed(fn, reps: int) -> float:
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0.record()
    for _ in range(reps):
        fn()
    s1.record()
    s1.synchronize()
    return s0.elapsed_time(s1) * 1e3 / reps  # us


def build_leg(leg: str, schema, P: np.ndarray, B: int, dev, x, y):
    mm.set_seed(0)
    s, op = schema, None
    if leg != "none":  # the input block binds the operator on the capture's first step
        op = mm.EmbeddingOperator(P, lookup_key=LOOKUP, embedding_name="pretrained", device=dev)
        s = op.compute_output_schema(schema)
    pe = mm.PretrainedEmbeddings(s.select_by_tag(mm.Tags.EMBEDDING), output_dims=64 if leg == "projected64" else None)
    emb = mm.Embeddings(s.select_by_tag(mm.Tags.CATEGORICAL).excluding_by_tag(mm.Tags.TARGET), dim=16)
    ib = mm.InputBlockV2(s, categorical=emb, pretrained_embeddings=pe)
    model = mm.DCNModel(s, depth=2, input_block=ib, deep_block=mm.MLPBlock([512, 256]),
                        prediction_tasks=mm.BinaryOutput("label"))
    model.compile(optimizer=mm.Adagrad(0.01))
    model.build(dev)
    tr = model.trainer(B)
    tr.capture(x, [y])
    return tr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--dp", type=int, default=768)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_pretrained_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, Dp = args.batch, args.dp
    schema = datasets.criteo_schema({k: min(v, 1_000_000) for k, v in datasets.CRITEO_MAX.items()})
    batch = datasets.generate_batch(schema, B, seed=7, index_law="uniform")
    feats, targs = datasets.split_targets(schema, batch)
    x = {k: torch.from_numpy(np.asarray(v)).to(dev) for k, v in feats.items()}
    y = torch.from_numpy(np.asarray(targs["label"], dtype=np.float32)).to(dev)
    rows = schema[LOOKUP].int_domain.max + 1
    P = np.random.default_rng(1).standard_normal((rows, Dp)).astype(np.float32)

    legs = {leg: build_leg(leg, schema, P, B, dev, x, y) for leg in ("none", "unprojected", "projected64")}
    for tr in legs.values():  # warm every graph
        tr.replay()
    torch.cuda.synchronize()
    times = {leg: [] for leg in legs}
    for _ in range(args.blocks):
        for leg, tr in legs.items():
            times[leg].append(timed(tr.replay, args.steps))
    for tr in legs.values():
        tr.check_indices()

    # the fused gather + projection alone, 20 launches per graph
    Pd = torch.from_numpy(P).to(dev)
    ids = x[LOOKUP].reshape(-1)
    W = torch.randn((Dp, 64), device=dev) * 0.03
    bias = torch.zeros(64, device=dev)
    out = torch.empty((B, 64), device=dev)
    slot = torch.empty((B, Dp), device=dev)
    graphs = {}
    for name, fn in (("project", lambda: ops.pretrained_project(Pd, ids, W, bias, out)),
                     ("gather", lambda: ops.pretrained_gather(Pd, ids, slot))):
        fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with graph_capture(g):
            for _ in range(KERNELS_PER_GRAPH):
                fn()
        graphs[name] = g
    kern = {name: [] for name in graphs}
    for _ in range(args.blocks):
        for name, g in graphs.items():
            kern[name].append(timed(g.replay, 10) / KERNELS_PER_GRAPH)
    idb = ids.element_size()
    floor_bytes = {"project": B * Dp * 4 + B * idb + Dp * 64 * 4 + 64 * 4 + B * 64 * 4,
                   "gather": B * Dp * 4 + B * idb + B * Dp * 4}
    res = {"tool": "train_pretrained_bench", "card": card(), "batch": B, "dp": Dp, "optimizer": "adagrad",
           "step_us": {leg: {"median": float(np.median(t)), "min": float(np.min(t)), "max": float(np.max(t))}
                       for leg, t in times.items()}}
    for name, t in kern.items():
        med = float(np.median(t))
        floor_us = floor_bytes[name] / HBM_BYTES_PER_S * 1e6
        res[f"{name}_kernel_us"] = {"median": med, "min": float(np.min(t)), "byte_floor_us": floor_us,
                                    "share_of_byte_floor": floor_us / med, "floor_bytes": floor_bytes[name]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
