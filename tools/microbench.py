#!/usr/bin/env python
"""Per-kernel microbenchmarks (CUDA events, L2-cold inputs: tables >> L2, rotating buffers).

    python tools/microbench.py [--only gather,interact,fused,dense,scores] [--iters 20]

Prints one JSON line per kernel with achieved algorithmic GB/s (or TFLOP/s) and the fraction of
the measured peak (MEASURED_PEAKS.json).  Never under a profiler.
"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import models_b200 as mm  # noqa: E402
from models_b200 import datasets, ops  # noqa: E402


def peaks():
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        d = json.loads(p.read_text())
        return d["hbm_gbs"], d["bf16_tflops"]
    return 6650.0, 1590.0


def timeit(fn, iters, warmup=3):
    for _ in range(warmup):
        fn(0)
    torch.cuda.synchronize()
    evs = []
    for i in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn(i)
        b.record()
        evs.append((a, b))
    torch.cuda.synchronize()
    t = sorted(x.elapsed_time(y) for x, y in evs)
    return float(np.mean(t)), float(t[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="gather,interact,fused,dense,scores")
    ap.add_argument("--catalog-items", type=int, default=10_000_000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--law", default="uniform")
    args = ap.parse_args()
    only = set(args.only.split(","))
    dev = torch.device("cuda", 0)
    hbm, tf = peaks()
    B, T, D = args.batch, 26, 64
    F = T + 1
    res = []

    def report(name, ms_mean, ms_min, bytes_=None, flops=None, **extra):
        r = {"kernel": name, "ms_mean": ms_mean, "ms_min": ms_min, **extra}
        if bytes_ is not None:
            r["algorithmic_bytes"] = bytes_
            r["GBps"] = bytes_ / (ms_mean * 1e-3) / 1e9
            r["frac_hbm"] = r["GBps"] / hbm
        if flops is not None:
            r["TFLOPs"] = flops / (ms_mean * 1e-3) / 1e12  # tensor-core FLOPs actually issued (x3 for the split)
            r["frac_bf16_peak"] = r["TFLOPs"] / tf
        print(json.dumps(r), flush=True)
        res.append(r)

    if only & {"gather", "interact", "fused", "fused2"}:
        schema = datasets.criteo_schema()
        cat = schema.select_by_tag(mm.Tags.CATEGORICAL)
        emb = mm.Embeddings(cat, dim=D, embeddings_initializer={"hash_seed": 4321})
        emb.build(dev)
        names = emb.feature_names
        slots = {n: i for i, n in enumerate(sorted(names + ["bottom_block"]))}
        nb = 4
        idx = []
        for i in range(nb):
            b = datasets.generate_batch(cat, B, seed=100 + i, index_law=args.law)
            idx.append([torch.from_numpy(b[n]).to(dev) for n in names])
        tables = [emb.feature_to_table[n].table for n in names]
        stack = [torch.empty((B, F * D), dtype=torch.float32, device=dev) for _ in range(2)]
        bottom = torch.randn((B, D), device=dev)
        out = [torch.empty((B, D + F * (F - 1) // 2), dtype=torch.float32, device=dev) for _ in range(2)]
        if "gather" in only:
            m, mn = timeit(lambda i: ops.gather_multi(tables, idx[i % nb], [slots[n] * D for n in names], stack[i % 2]), args.iters)
            report("mm_gather_multi (26 tables, D=64, int32)", m, mn, bytes_=B * (2 * T * D * 4 + T * 4), law=args.law)
        if "interact" in only:
            x = torch.randn((B, F, D), device=dev)
            m, mn = timeit(lambda i: ops.dot_interaction(x, out[i % 2], prefix=bottom), args.iters)
            report("mm_dot_interaction (F=27, D=64, +prefix)", m, mn, bytes_=B * (F * D * 4 + (D + 351) * 4),
                   flops=B * 351 * 64 * 2)
        if "fused" in only:
            rows = [t.shape[0] for t in tables]
            m, mn = timeit(lambda i: ops.dlrm_lookup_interact(tables, idx[i % nb], [slots[n] for n in names], rows, D, bottom,
                                                              slots["bottom_block"], out[i % 2]), args.iters)
            report("mm_dlrm_lookup_interact (int32 ids, fp32 out)", m, mn, bytes_=B * (T * D * 4 + T * 4 + D * 4 + (D + 351) * 4),
                   law=args.law)

    if "fused2" in only:
        # the real step's launch: split-bf16 output row (B, 2*448); ids as int32 and packed (1/2/3-byte)
        Kp = ops.tc_padded_k(D + F * (F - 1) // 2)
        osplit = [torch.empty((B, 2 * Kp), dtype=torch.bfloat16, device=dev) for _ in range(2)]
        rows = [t.shape[0] for t in tables]
        sl = [slots[n] for n in names]
        m, mn = timeit(lambda i: ops.dlrm_lookup_interact(tables, idx[i % nb], sl, rows, D, bottom, slots["bottom_block"], osplit[i % 2]), args.iters)
        report("mm_dlrm_lookup_interact (int32 ids, split out)", m, mn, bytes_=B * (T * D * 4 + T * 4 + D * 4 + (D + 351) * 4), law=args.law)
        def narrow(t, r):
            h = t.cpu().numpy()
            if r <= 256:
                h = h.astype(np.uint8)
            elif r <= 65536:
                h = h.astype(np.uint16)
            elif r <= (1 << 24):
                h = h.astype("<u4").view(np.uint8).reshape(-1, 4)[:, :3].copy()
            return torch.from_numpy(h).to(dev)
        pidx = [[narrow(t, r) for t, r in zip(b_, rows)] for b_ in idx]
        idb = sum(ops.index_bytes_of(t) for t in pidx[0])
        m, mn = timeit(lambda i: ops.dlrm_lookup_interact(tables, pidx[i % nb], sl, rows, D, bottom, slots["bottom_block"], osplit[i % 2]), args.iters)
        report(f"mm_dlrm_lookup_interact (packed ids {idb} B/sample, split out)", m, mn,
               bytes_=B * (T * D * 4 + idb + D * 4 + (D + 351) * 4), law=args.law)
        mirrors = [ops.split_rows(t) for t in tables]
        bottom_op = ops.split_rows(bottom)
        m, mn = timeit(lambda i: ops.dlrm_lookup_interact(mirrors, pidx[i % nb], sl, rows, D, bottom_op, slots["bottom_block"], osplit[i % 2],
                                                          operand_rows=True), args.iters)
        report(f"mm_dlrm_lookup_interact (operand-format rows, packed ids {idb} B/sample, split out)", m, mn,
               bytes_=B * (T * D * 4 + idb + D * 4 + (D + 351) * 4), law=args.law)
        del mirrors

    if "dense" in only:
        for (K, N) in [(13, 128), (128, 64), (415, 128), (128, 64), (64, 32), (32, 1), (1037, 1037), (1024, 1024)]:
            x = torch.randn((B, K), device=dev)
            W = torch.randn((K, N), device=dev) * 0.05
            b = torch.zeros(N, device=dev)
            o = torch.empty((B, N), device=dev)
            m, mn = timeit(lambda i: ops.dense_fp32(x, W, b, "relu", o), max(5, args.iters // 2))
            report(f"mm_dense_fp32 {K}->{N}", m, mn, bytes_=B * (K + N) * 4, flops=2.0 * B * K * N)

    if "scores" in only:
        Bq, Dq = 16384, 64
        q = torch.randn((Bq, Dq), device=dev)
        it = torch.randn((Bq, Dq), device=dev)
        ids = torch.randint(0, 10_000_000, (Bq,), device=dev, dtype=torch.int64)
        o = torch.empty((Bq, Bq + 4), device=dev)[:, 3:]  # negatives 16-B aligned (as retrieval._score allocates)
        for tc in (False, True):
            m, mn = timeit(lambda i: ops.inbatch_scores(q, it, it, o, pos_ids=ids, neg_ids=ids, tensor_cores=tc), max(5, args.iters // 2))
            report(f"mm_inbatch_scores 16384x16384 D=64 ({'wgmma split-bf16 incl. operand split' if tc else 'fp32 SIMT'})", m, mn,
                   bytes_=Bq * (Bq + 1) * 4, flops=2.0 * Bq * Bq * Dq)

    if "fusedce" in only:
        Bq = 16384
        ids = torch.randint(0, 10_000_000, (Bq,), device=dev, dtype=torch.int64)
        for Dq in (64, 128):
            q = torch.randn((Bq, Dq), device=dev)
            it = torch.randn((Bq, Dq), device=dev)
            m, mn = timeit(lambda i: ops.inbatch_softmax_ce(q, it, it, pos_ids=ids, neg_ids=ids), max(5, args.iters // 2))
            report(f"mm_inbatch_softmax_ce 16384x16384 D={Dq} (fused CE stats, incl. operand split + positive scores)", m, mn,
                   flops=2.0 * Bq * Bq * Dq * 3, logical_flops=2.0 * Bq * Bq * Dq)

    if "catalog" in only:
        Bq, Dq, I = 16384, 64, args.catalog_items
        q = torch.randn((Bq, Dq), device=dev)
        E = torch.empty((I, Dq), device=dev)
        ops.init_uniform_hash(E, 77, -0.5, 0.5)
        es = ops.split_rows(E)
        tg = torch.randint(0, I, (Bq,), device=dev)
        for k, stats in ((0, True), (10, False), (10, True)):
            m, mn = timeit(lambda i: ops.catalog_score(q, es, I, targets=tg if stats else None, k=k, want_stats=stats), 3, warmup=1)
            report(f"mm_catalog_score B=16384 I={I} D=64 (lse={stats}, topk={k})", m, mn, flops=2.0 * Bq * I * Dq * 3,
                   logical_flops=2.0 * Bq * I * Dq)

    if "tc_dense" in only:
        for (K, N) in [(415, 128), (128, 64), (13, 128), (1024, 1024), (1037, 1037), (512, 256), (415, 1024)]:
            x = torch.randn((B, K), device=dev)
            W = torch.randn((K, N), device=dev) * 0.05
            b = torch.zeros(N, device=dev)
            a, w = ops.split_rows(x), ops.split_weights(W)
            nxt = torch.zeros((B, 2 * ops.tc_padded_k(N)), dtype=torch.bfloat16, device=dev)
            m, mn = timeit(lambda i: ops.dense_tc(a, K, w, N, b, "relu", out_split=nxt), max(5, args.iters // 2))
            report(f"mm_dense_tc {K}->{N} (3-pass split-bf16, split out)", m, mn, flops=2.0 * B * K * N * 3,
                   bytes_=B * (2 * ops.tc_padded_k(K) * 2 + 2 * ops.tc_padded_k(N) * 2), logical_flops=2.0 * B * K * N)

    if "mlp" in only:
        # README towers: whole-tower kernel (mm_mlp_tc) vs the per-layer wgmma chain (mm_dense_tc)
        for K, widths, head in ((415, [128, 64, 32], True), (13, [128, 64], False)):
            x = torch.randn((B, K), device=dev)
            Ws = [torch.randn((k, n), device=dev) / (k ** 0.5) for k, n in zip([K] + widths[:-1], widths)]
            bs = [torch.zeros(n, device=dev) for n in widths]
            ws = [ops.split_weights(W) for W in Ws]
            a = ops.split_rows(x)
            hw = torch.randn(widths[-1], device=dev)
            out = torch.empty((B, 1 if head else widths[-1]), device=dev)
            acts = ["relu"] * len(widths)
            io_bytes = B * (2 * ops.tc_padded_k(K) * 2 + out.shape[1] * 4)

            def fused(i):
                if head:
                    ops.mlp_tc(a, K, ws, widths, bs, acts, head_w=hw, head_b=0.1, head_act="sigmoid", head_out=out)
                else:
                    ops.mlp_tc(a, K, ws, widths, bs, acts, out=out)

            bufs = [torch.zeros((B, 2 * ops.tc_padded_k(n)), dtype=torch.bfloat16, device=dev) for n in widths[:-1]]

            def layered(i):
                cur, k = a, K
                for li, n in enumerate(widths):
                    last = li == len(widths) - 1
                    if last and head:
                        ops.dense_tc_head(cur, k, ws[li], n, bs[li], "relu", hw, 0.1, "sigmoid", out)
                    elif last:
                        ops.dense_tc(cur, k, ws[li], n, bs[li], "relu", out_f32=out)
                    else:
                        ops.dense_tc(cur, k, ws[li], n, bs[li], "relu", out_split=bufs[li])
                        cur, k = bufs[li], n

            name = f"{K}->" + "->".join(map(str, widths)) + ("->1" if head else "")
            m, mn = timeit(fused, args.iters)
            report(f"mm_mlp_tc {name} (one launch)", m, mn, bytes_=io_bytes)
            m, mn = timeit(layered, args.iters)
            report(f"mm_dense_tc chain {name} ({len(widths)} launches)", m, mn, bytes_=io_bytes)

    if "bottom" in only:
        # DLRM bottom path: 13 continuous columns -> 128 -> 64 (fp32 rows out / operand-format rows out)
        from models_b200 import blocks

        mm.set_seed(3)
        cols = {f"I{i}": torch.rand(B, device=dev) for i in range(1, 14)}
        mlp = mm.MLPBlock([128, 64])
        for small in (True, False):
            blocks._SMALL_TOWER[0] = small
            for op in (False, True):
                m, mn = timeit(lambda i: mlp(cols, operand_out=op), args.iters)
                report(f"bottom tower 13->128->64 ({'mm_tower2_small' if small else 'mm_concat_split + mm_mlp_tc'}, "
                       f"{'split-bf16 rows' if op else 'fp32 rows'} out; eager: includes launch gaps)", m, mn, bytes_=B * (13 * 4 + 64 * 4))
        blocks._SMALL_TOWER[0] = True

    if "models" in only:
        mm.set_seed(1)
        # config 5: DCN-v2, bundled Criteo, inferred dims (d = 1037), depth 3, deep [256, 128]
        schema = datasets.criteo_schema()
        dcn = mm.DCNModel(schema, depth=3, deep_block=mm.MLPBlock([256, 128]),
                          embeddings_initializer={"hash_seed": 99})
        b, _ = datasets.split_targets(schema, datasets.generate_batch(schema, B, seed=5, index_law="uniform"))
        cf = dcn.compile(b)
        m, mn = timeit(lambda i: cf.replay(), max(5, args.iters // 2))
        report("mm.DCNModel fwd (config 5: d=1037, depth 3, deep [256,128], B=65536, graph)", m, mn,
               flops=3 * (3 * 2 * 1037 * 1037 + 2 * (1037 * 256 + 256 * 128)) * B, logical_flops=7.05e6 * B,
               samples_per_s=B / (m * 1e-3))
        del dcn, cf
        torch.cuda.empty_cache()
        # wide-tower DLRM (SURVEY §8(d) config 2 variant): bottom [512,256,64], top [1024,1024,512,256]
        wide = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([512, 256, 64]),
                            top_block=mm.MLPBlock([1024, 1024, 512, 256]),
                            embedding_options=mm.EmbeddingOptions(embeddings_initializers={"hash_seed": 4321}))
        cfw = wide.compile(b)
        m, mn = timeit(lambda i: cfw.replay(), max(5, args.iters // 2))
        wf = 2.0 * (13 * 512 + 512 * 256 + 256 * 64 + 415 * 1024 + 1024 * 1024 + 1024 * 512 + 512 * 256 + 256) * B
        report("mm.DLRMModel wide towers fwd (bottom [512,256,64], top [1024,1024,512,256], B=65536, graph)", m, mn,
               flops=3 * wf, logical_flops=wf, samples_per_s=B / (m * 1e-3))
        del wide, cfw
        torch.cuda.empty_cache()
        # config 3: two-tower, 10M-item catalog, in-batch negatives, B = 16384
        rs = datasets.retrieval_10m_schema()
        tt = mm.TwoTowerModel(rs, query_tower=mm.MLPBlock([256, 128]),
                              embedding_options=mm.EmbeddingOptions(embeddings_initializers={"hash_seed": 5}))
        Bt = 16384
        tb = datasets.generate_batch(rs, Bt, seed=6, index_law="zipf")
        cft = tt.compile(tb, training=True)
        m, mn = timeit(lambda i: cft.replay(), max(5, args.iters // 2))
        report("mm.TwoTowerModel train-mode fwd (config 3: 10M items, towers [256,128], in-batch, B=16384, graph)", m, mn,
               bytes_=Bt * (Bt + 1) * 4, samples_per_s=Bt / (m * 1e-3))


if __name__ == "__main__":
    main()
