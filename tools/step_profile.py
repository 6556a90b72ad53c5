"""Where the headline DLRM step's time goes, kernel by kernel, and the top tower timed alone next to its HBM floor.

    python tools/step_profile.py [--batch 65536] [--steps 50] [--out DIR] [--tower-only]

1. The headline step (bench.py --workload dlrm: Criteo shape, emb 64, bottom [128, 64], top [128, 64, 32] + sigmoid head)
   compiled into a CUDA graph and replayed `--steps` times under torch.profiler with CUDA activities: prints each
   kernel's device time per step (the profiler's trace goes to DIR/step_trace.json when --out is given).
2. `mm_mlp_tc` alone at the headline shape (K = 415 split-bf16 input rows of pitch 2 * 448, [128, 64, 32] + fused sigmoid
   head), CUDA events around each of `--steps` back-to-back launches, next to the time a device-to-device copy needs
   to read its input once (the measured HBM floor of a kernel that must read that many bytes).
Prints the card name and power limit of the same run.
"""
import argparse
import json
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import models_b200 as mm  # noqa: E402
from models_b200 import datasets, ops  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def event_ms(fn, n, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    evs = []
    for _ in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        evs.append((e0, e1))
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in evs]))


def step_breakdown(B, steps, out_dir):
    dev = torch.device("cuda", 0)
    schema = datasets.criteo_schema()
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([128, 64]), top_block=mm.MLPBlock([128, 64, 32]),
                         embedding_options=mm.EmbeddingOptions(embeddings_initializers={"hash_seed": 4321}))
    model.build(dev)
    hosts = []
    for i in range(4):
        b = datasets.generate_batch(schema, B, seed=1234 + i, index_law="uniform", index_dtype=np.int32)
        hosts.append(datasets.split_targets(schema, b)[0])
    hbs = [mm.HostBatch.like(h, model.input_columns(), id_bytes=model.id_bytes()) for h in hosts]
    packed = [hb.buffer.to(dev) for hb in hbs]
    cf = model.compile(hbs[0])

    def step(i):
        cf.load_device(packed[i % len(packed)])
        cf.replay()

    for i in range(10):
        step(i)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for i in range(steps):
            step(i)
        torch.cuda.synchronize()
    per = defaultdict(lambda: [0.0, 0])
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            per[e.name][0] += e.time_range.elapsed_us()
            per[e.name][1] += 1
    if out_dir:
        prof.export_chrome_trace(str(Path(out_dir) / "step_trace.json"))
    rows = sorted(((us / steps, n / steps, name) for name, (us, n) in per.items()), reverse=True)
    total = sum(r[0] for r in rows)
    print(f"headline step, B = {B}: device time per step by kernel ({steps} graph replays, serial)")
    for us, n, name in rows:
        print(f"  {us:9.1f} us  {n:4.1f}x  {name[:110]}")
    print(f"  {total:9.1f} us  sum of kernel times per step")
    del cf, model
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return {name[:80]: us for us, _, name in rows}


def top_tower_alone(B, steps):
    dev = torch.device("cuda", 0)
    g = torch.Generator(device="cpu").manual_seed(7)
    K, widths = 415, [128, 64, 32]
    x = torch.randn((B, K), generator=g).mul_(0.5).to(dev)
    a = ops.split_rows(x)  # (B, 2 * 448)
    assert a.shape[1] == 2 * 448
    ws, bs, k = [], [], K
    for w in widths:
        W = (torch.randn((k, w), generator=g) * (2.0 / (k + w)) ** 0.5).to(dev)
        ws.append(ops.split_weights(W))
        bs.append((torch.randn(w, generator=g) * 0.01).to(dev))
        k = w
    head_w = (torch.randn(32, generator=g) * 0.2).to(dev)
    head_out = torch.empty((B, 1), dtype=torch.float32, device=dev)

    def run():
        ops.mlp_tc(a, K, ws, widths, bs, ["relu"] * 3, head_w=head_w, head_b=0.01, head_act="sigmoid", head_out=head_out)

    ms = event_ms(run, steps)
    in_bytes = a.numel() * a.element_size()
    src = torch.empty(in_bytes // 2, dtype=torch.bfloat16, device=dev).normal_()
    dst = torch.empty_like(src)
    copy_ms = event_ms(lambda: dst.copy_(src), steps)
    hbm_gbs = 2 * in_bytes / (copy_ms * 1e-3) / 1e9  # the copy reads and writes `in_bytes`
    floor_ms = in_bytes / (hbm_gbs * 1e9) * 1e3
    print(f"mm_mlp_tc alone, B = {B}, K = {K}, {widths} + sigmoid head: {ms * 1e3:.1f} us (median of {steps})")
    print(f"  input {in_bytes / 1e6:.1f} MB; D2D copy rate {hbm_gbs:.0f} GB/s -> HBM floor {floor_ms * 1e3:.1f} us; "
          f"kernel / floor = {ms / floor_ms:.2f}")
    return {"mlp_tc_us": ms * 1e3, "input_mb": in_bytes / 1e6, "copy_gbs": hbm_gbs, "floor_us": floor_ms * 1e3,
            "ratio": ms / floor_ms, "head_out_checksum": float(head_out.double().sum().item())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for the profiler trace and a JSON summary")
    ap.add_argument("--tower-only", action="store_true", help="time mm_mlp_tc alone; skip the step profile")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("step_profile.py needs a CUDA device")
    name = card()
    print(f"card: {name}")
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
    tower = top_tower_alone(args.batch, args.steps)
    kernels = {} if args.tower_only else step_breakdown(args.batch, args.steps, args.out)
    if args.out:
        (Path(args.out) / "step_profile.json").write_text(json.dumps({"card": name, "tower": tower, "step_us": kernels}, indent=1))


if __name__ == "__main__":
    main()
