"""Cost of evaluating the DLRM that bench.py runs (Criteo schema, B = 65 536, README towers), in one process:

  (a) forward_replay   CompiledForward replay (the serving forward, one CUDA graph)
  (b) eval_graph       one evaluate step as RankingModel.evaluate runs a full-size batch: EvalGraph replay (logits forward +
                       mm_metrics_update in one CUDA graph, static buffers refreshed by a device-to-device copy);
      eval_eager       the same step launched eagerly from Python (the smaller last batch / ragged features)
  (c) metrics_*        mm_metrics_update, H = 1 and H = 8, uniform predictions and all predictions in one AUC bucket:
                       `_kernel` = 20 back-to-back launches captured in one CUDA graph (the device time of the two kernels),
                       `_call` = the Python call ops.metrics_update (argument checks and ctypes included)

Timed in alternating blocks with CUDA events; prints one JSON line with the card name and power limit.

    python tools/eval_bench.py [--batch 65536] [--reps 50] [--blocks 5]
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
from models_b200 import _cabi, datasets, ops  # noqa: E402
from models_b200.graph import EvalGraph, graph_capture  # noqa: E402
from models_b200.metrics import MetricsSpec, MetricsState  # noqa: E402


KERNELS_PER_GRAPH = 20


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--blocks", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    B = args.batch
    schema = datasets.criteo_schema()
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([128, 64]), top_block=mm.MLPBlock([128, 64, 32]),
                         embedding_options=mm.EmbeddingOptions(embeddings_initializers={"hash_seed": 4321}))
    model.build(dev)
    b = datasets.generate_batch(schema, B, seed=1234, index_law="uniform", index_dtype=np.int32)
    feats, targets = datasets.split_targets(schema, b)
    x = {k: torch.from_numpy(v).to(dev) for k, v in feats.items()}
    y = torch.from_numpy(np.asarray(next(iter(targets.values())) if isinstance(targets, dict) else targets)).to(dev)
    hb = mm.HostBatch.like(feats, model.input_columns(), id_bytes=model.id_bytes())
    cf = model.compile(hb)
    cf.load_device(hb.buffer.to(dev))
    model.compile(optimizer="adam")
    spec = model.metrics_spec
    st = MetricsState(spec, dev)

    def eval_step():
        z, form = model.logits(x)
        st.update(z, [y], form)

    model.defer_index_check(True)  # as evaluate does: the out-of-range counter is read once at the end
    eg = EvalGraph(model, st, x, [y], None)

    g = torch.Generator().manual_seed(0)
    cases, graphs = {}, []
    for Hh in (1, 8):
        sp = MetricsSpec([mm.BinaryOutput(f"t{h}") for h in range(Hh)], [1.0] * Hh)
        s = MetricsState(sp, dev)
        s.reserve(B)
        ys = [(torch.rand(B, generator=g) < 0.3).float().to(dev) for _ in range(Hh)]
        for law, z in (("uniform", torch.randn((Hh, B), generator=g) * 3), ("one_bucket", torch.full((Hh, B), 1.3))):
            z = z.to(dev).contiguous()
            call = (lambda s=s, z=z, ys=ys, sp=sp: ops.metrics_update(
                z, sp.losses, ys, s.state, s.workspace, sp.num_buckets, [_cabi.PRED_ACT] * len(ys), sp.thresholds))
            call()
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with graph_capture(graph):
                for _ in range(KERNELS_PER_GRAPH):
                    call()
            graphs.append(graph)
            cases[f"metrics_H{Hh}_{law}_call"] = call
            cases[f"metrics_H{Hh}_{law}_kernel"] = graph.replay
    fns = {"forward_replay": cf.replay, "eval_graph": lambda: eg.replay(x, [y], None), "eval_eager": eval_step, **cases}
    for fn in fns.values():  # warm-up of every shape
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    res = {k: [] for k in fns}
    for _ in range(args.blocks):
        for k, fn in fns.items():
            res[k].append(timed(fn, args.reps))
    st.result()
    per = {k: (KERNELS_PER_GRAPH if k.endswith("_kernel") else 1) for k in res}
    out = {"card": card(), "batch": B, "unit": "us per step / per metrics_update (median of blocks)",
           **{k: float(np.median(v)) / per[k] for k, v in res.items()},
           "spread": {k: [float(min(v)) / per[k], float(max(v)) / per[k]] for k, v in res.items()}}
    out["eval_graph_minus_forward"] = out["eval_graph"] - out["forward_replay"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
