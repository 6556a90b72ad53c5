#!/usr/bin/env python
"""NVLink peer access patterns (torchrun, 2+ ranks): GB/s of pulling / pushing 256-byte rows from / to the next
rank's HBM, by access pattern.  Diagnostic for the row-sharded lookup; not a product path.

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29540 tools/probe/peer_probe.py
"""
import ctypes as C
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

HERE = Path(__file__).resolve().parent


def build():
    so = HERE / "_peer_probe.so"
    src = HERE / "peer_probe.cu"
    if not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
        subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
                        "-shared", "-o", str(so), str(src), "-lcudart"], check=True)
    lib = C.CDLL(str(so))
    lib.probe_run.restype = C.c_int
    lib.probe_run.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    lib = build() if rank == 0 else None
    dist.barrier(device_ids=[local])
    lib = lib or build()
    import torch.distributed._symmetric_memory as symm_mem

    gib = float(os.environ.get("PROBE_TABLE_GIB", "2"))
    table_rows = int(gib * 4 * 1024 * 1024)  # 256-byte rows per rank
    buf = symm_mem.empty((table_rows * 64,), dtype=torch.float32, device=dev)
    hdl = symm_mem.rendezvous(buf, group=dist.group.WORLD)
    buf.normal_()
    ptrs = [int(p) for p in hdl.buffer_ptrs]
    peer = ptrs[(rank + 1) % world]
    n = 4 * 1024 * 1024  # rows per launch = 1 GiB
    rng = np.random.default_rng(rank)
    span = float(os.environ.get("PROBE_SPAN_GIB", str(gib / 2)))  # rows are drawn from the first `span` GiB
    idx = torch.from_numpy(rng.integers(0, int(span * 4 * 1024 * 1024), n).astype(np.int32)).to(dev)
    sink = torch.zeros(4, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    # push target: second half of the peer's buffer (row i of the launch -> row table_rows/2 + i)
    half_off = (table_rows // 2) * 256

    def run(mode, src, dst, depth, rpg, blocks, threads):
        rc = lib.probe_run(mode, src, dst, idx.data_ptr(), n, depth, rpg, blocks, threads, sink.data_ptr(), st)
        assert rc == 0, rc

    def bench(label, mode, target, depth=1, rpg=24, blocks=132, threads=512, both=True):
        src = ptrs[rank] if target == "local" else peer
        dst = (ptrs[rank] if target == "local" else peer) + half_off
        if mode == 5:
            src = ptrs[rank]
        active = both or rank == 0
        dist.barrier(device_ids=[local])
        if active:
            for _ in range(2):
                run(mode, src, dst, depth, rpg, blocks, threads)
        torch.cuda.synchronize()
        dist.barrier(device_ids=[local])
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        if active:
            for _ in range(4):
                run(mode, src, dst, depth, rpg, blocks, threads)
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / 4
        t = torch.tensor([ms], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if rank == 0:
            used = (n // rpg) * rpg if mode in (1, 2, 6) else n
            print(json.dumps({"table_gib": gib, "span_gib": span, "pattern": label, "target": target, "both_directions": both, "depth": depth, "rows_per_group": rpg,
                              "blocks": blocks, "threads": threads, "ms": float(t.item()),
                              "GBps_per_gpu": used * 256 / (float(t.item()) * 1e-3) / 1e9}), flush=True)

    if os.environ.get("PROBE_MIXED"):
        # src = local buffer, dst = peer buffer (both read); half of the 1 GiB is remote
        def mixed(label, mode, depth, rpg, threads):
            dist.barrier(device_ids=[local])
            for _ in range(2):
                rc = lib.probe_run(mode, ptrs[rank], peer, idx.data_ptr(), n, depth, rpg, 132, threads, sink.data_ptr(), st); assert rc == 0
            torch.cuda.synchronize()
            dist.barrier(device_ids=[local])
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(4):
                lib.probe_run(mode, ptrs[rank], peer, idx.data_ptr(), n, depth, rpg, 132, threads, sink.data_ptr(), st)
            t1.record()
            torch.cuda.synchronize()
            t = torch.tensor([t0.elapsed_time(t1) / 4], device=dev, dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            if rank == 0:
                used = (n // rpg) * rpg
                print(json.dumps({"pattern": label, "depth": depth, "rows_per_group": rpg, "threads": threads, "ms": float(t.item()),
                                  "remote_GBps_per_gpu": used * 128 / (float(t.item()) * 1e-3) / 1e9,
                                  "total_GBps_per_gpu": used * 256 / (float(t.item()) * 1e-3) / 1e9}), flush=True)
        for depth, rpg, threads in ((1, 24, 512), (2, 24, 512), (4, 24, 256)):
            mixed("half local / half remote rows, MIXED inside one LDGSTS instruction", 7, depth, rpg, threads)
            mixed("half local / half remote rows, local and remote in SEPARATE instructions", 8, depth, rpg, threads)
        dist.destroy_process_group()
        return
    if os.environ.get("PROBE_SHORT"):
        for target in ("local", "peer"):
            bench("random rows, ld.global.v4 x8 in flight/lane (16 lanes/row)", 4, target, blocks=132 * 4, threads=512)
            bench("random rows, LDGSTS 8 lanes/row", 1, target, 1, 24, 132, 512)
            bench("random rows, LDGSTS 8 lanes/row", 1, target, 2, 24, 132, 512)
            bench("random rows, cp.async.bulk 256 B", 2, target, 2, 24, 132, 512)
        dist.destroy_process_group()
        return
    for target in ("local", "peer"):
        for both in ((True, False) if target == "peer" else (True,)):
            bench("sequential 16-B loads", 0, target, blocks=132 * 8, threads=512, both=both)
            bench("sequential 16-B stores", 3, target, blocks=132 * 8, threads=512, both=both)
            bench("random rows, ld.global.v4 x8 in flight/lane (16 lanes/row)", 4, target, blocks=132 * 4, threads=512, both=both)
            bench("random rows PUSH (local read -> peer store)", 5, target, blocks=132 * 4, threads=512, both=both)
            for depth, rpg, threads in ((1, 24, 512), (2, 24, 512), (4, 24, 256), (8, 12, 256)):
                bench("random rows, LDGSTS 8 lanes/row", 1, target, depth, rpg, 132, threads, both)
            bench("random rows, LDGSTS 16 lanes/row", 6, target, 2, 24, 132, 512, both)
            for depth, rpg, threads in ((1, 24, 512), (2, 24, 512), (4, 24, 256), (8, 12, 256)):
                bench("random rows, cp.async.bulk 256 B", 2, target, depth, rpg, 132, threads, both)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
