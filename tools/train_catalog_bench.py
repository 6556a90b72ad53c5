"""Training step of the weight-tied next-item classifier Model(InputBlockV2, MLPBlock, CategoricalOutput), captured as one
CUDA graph, in two legs, and its output layer's launches timed alone against the computed floors.

    python tools/train_catalog_bench.py [--blocks 5] [--steps 5] [--legs a,b] [--dropout 0.2] [--label-smoothing 0.1]

Schema: user_id (1 M rows x 64), two small user columns (100 and 1 000 rows), a fixed-length 20-id item history tied to
the output (mean-pooled), and the next_item target; MLPBlock([128, 64]), D = 64, T = 1, a bias, Adagrad(0.01).  Leg (a):
N_I = 1 M, B = 16 384; leg (b): N_I = 10 M, B = 4096.  Item ids are uniform.  Prints the card's name and power limit read
in the same run, launches per step, each leg's median ms per step and samples/s over the blocks (CUDA events around --steps
graph replays per block), and CUDA-event times of the output layer's launches on the step's own buffers: the soft-max
statistics (mm_catalog_score), the backward's dq + dn kernels (mm_catalog_softmax_ce_backward), the row merge
(mm_slices_add_dense, on the step's uniform ids and on the same ids with half of them replaced by a padding id 0) and the
tied table's update (mm_dense_apply over N_I D), next to the output layer's FLOP floor
(5 products x 3 split-bf16 passes x 2 B N_I D at 989 TFLOP/s) and the table update's byte floor (Adagrad reads E, dE and
the accumulator and writes E, the accumulator and the cleared dE: 6 x 4 N_I D bytes at 3.35 TB/s).

--dropout rate and / or --label-smoothing eps build a second, identical model with MLPBlock(dropout=rate) (a mask drawn in
each layer's epilogue) compiled with CategoricalCrossEntropy(label_smoothing=eps), and time its captured step in blocks
alternating with the plain step's, so both rows share the card's state (read by nvidia-smi in the same run); the smoothed
backward (column sums of E and x, the smoothed dq + dn kernels) is timed beside the plain one.
"""
import argparse
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import models_b200 as mm  # noqa: E402
from models_b200 import ops  # noqa: E402
from models_b200.schema import ColumnSchema, Schema, Tags  # noqa: E402

PEAK_BF16 = 989e12  # H100 SXM data sheet, dense
HBM_BYTES_PER_S = 3.35e12
D, L = 64, 20


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def schema(n_items: int) -> Schema:
    def cat(name, rows, **kw):
        return ColumnSchema(name, tags=(Tags.CATEGORICAL,), dtype="int64",
                            properties={"domain": {"min": 0, "max": rows - 1, "name": kw.pop("dom", name)}, **kw.pop("props", {})},
                            **kw)

    return Schema([cat("user_id", 1_000_000), cat("user_age", 100), cat("user_city", 1000),
                   cat("item_history", n_items, dom="item_id", is_list=True, is_ragged=False,
                       props={"value_count": {"min": L, "max": L}}),
                   ColumnSchema("next_item", tags=(Tags.TARGET,), dtype="int64")])


def batch(s: Schema, n_items: int, B: int, seed: int, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    f = {c.name: torch.randint(0, c.int_domain.max + 1, (B, L) if c.is_list else (B,), generator=g, device=dev)
         for c in s if not c.has_tag(Tags.TARGET)}
    return f, torch.randint(0, n_items, (B,), generator=g, device=dev)


def events(fn, n: int) -> float:
    """Median ms of fn over 3 blocks of n calls (CUDA events)."""
    out = []
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) / n)
    return statistics.median(out)


def step(s: Schema, n_items: int, B: int, eps: float, rate: float, dev):
    """(model, trainer) of the benchmark's model with its step captured; eps > 0: the label-smoothed loss; rate > 0:
    dropout after the MLP's layers."""
    mm.set_seed(1)
    emb = mm.Embeddings(s.select_by_tag(Tags.CATEGORICAL), dim={"user_id": 64, "user_age": 8, "user_city": 16, "item_history": D},
                        embeddings_initializer={"hash_seed": 5}, sequence_combiner="mean")
    out = mm.CategoricalOutput(emb.tables["item_id"], target_name="next_item")
    model = mm.Model(mm.InputBlockV2(s, categorical=emb), mm.MLPBlock([128, D], dropout=rate or None), out)
    model.compile(optimizer=mm.Adagrad(0.01),
                  loss=mm.losses.CategoricalCrossEntropy(from_logits=True, label_smoothing=eps) if eps else None)
    model.build(dev)
    tr = model.trainer(B)
    x, y = batch(s, n_items, B, 0, dev)
    tr.capture(x, [y])
    for i in range(3):  # warm-up replays
        tr.replay()
    torch.cuda.synchronize()
    return model, tr


def leg(name: str, n_items: int, B: int, args, dev) -> None:
    s = schema(n_items)
    eps, rate = float(args.label_smoothing), float(args.dropout)
    runs = [("plain", *step(s, n_items, B, 0.0, 0.0, dev))]
    if eps or rate:
        runs.append((f"dropout={rate}, label_smoothing={eps}", *step(s, n_items, B, eps, rate, dev)))
    per_block = {k: [] for k, _, _ in runs}
    for _ in range(args.blocks):  # the steps alternate block by block
        for k, _, tr in runs:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.steps):
                tr.replay()
            b.record()
            b.synchronize()
            per_block[k].append(a.elapsed_time(b) / args.steps)
    for k, _, tr in runs:
        pb = per_block[k]
        ms = statistics.median(pb)
        print(f"leg ({name}) {k}: N_I = {n_items:,}, B = {B:,}, D = {D}: {tr.launches_per_step} launches per step, "
              f"{ms:.2f} ms per step (median of {args.blocks} blocks x {args.steps} replays, spread "
              f"{min(pb):.2f}-{max(pb):.2f}), {B / ms * 1e3:,.0f} samples/s")
    if len(runs) > 1:
        print(f"  {runs[1][0]} / plain: {statistics.median(per_block[runs[1][0]]) / statistics.median(per_block['plain']):.4f}")
    if eps:
        _, tr_s = runs[1][1:]
        wk = tr_s.wk
        tr_s.forward_backward(tr_s._static, tr_s._static_y)
        xs = tr_s.h_split[-1][:B]
        yy = tr_s._static_y[0]
        t_sm = events(lambda: ops.catalog_softmax_ce_backward(xs, wk.e_split, D, tr_s.stats, yy, tr_s._scale(B), tr_s.dh[-1][:B],
                                                              wk.dE, db=wk.db, bias=wk.bt, workspace=tr_s.ws_bwd,
                                                              label_smoothing=eps), 3)
        print(f"  smoothed backward (column sums + dq + dn) {t_sm:.2f} ms")
        del tr_s
    del runs[1:]
    _, model, tr = runs[0]
    # the output layer's launches alone, on the step's own buffers (after a forward_backward of the captured batch)
    wk = tr.wk
    tr.forward_backward(tr._static, tr._static_y)
    xs = tr.h_split[-1][:B]
    yy = tr._static_y[0]
    t_stats = events(lambda: ops.catalog_stats_split(xs, D, wk.e_split, tr.stats, yy, tr.ws_stats, bias=wk.bt), 5)
    t_bwd = events(lambda: ops.catalog_softmax_ce_backward(xs, wk.e_split, D, tr.stats, yy, tr._scale(B), tr.dh[-1][:B], wk.dE,
                                                           db=wk.db, bias=wk.bt, workspace=tr.ws_bwd), 3)
    bag = tr._bags[tr.tt]
    t_merge = events(lambda: ops.slices_add_dense(bag["apply_ids"], bag["rows"], wk.dE, workspace=tr.ws_merge), 10)
    padded = bag["apply_ids"].clone()  # a history half made of padding id 0: one run of ~n / 2 equal ids
    padded[torch.rand(padded.shape, device=dev) < 0.5] = 0
    t_pad = events(lambda: ops.slices_add_dense(padded, bag["rows"], wk.dE, workspace=tr.ws_merge), 10)
    e_flat = wk.E.view(-1)
    t_upd = events(lambda: ops.dense_apply("adagrad", e_flat, wk.dE.view(-1), wk.s1.view(-1), None, tr.hyper), 10)
    flop_ms = 5 * 3 * 2 * B * n_items * D / PEAK_BF16 * 1e3
    upd_floor = 6 * 4 * n_items * D / HBM_BYTES_PER_S * 1e3
    print(f"  statistics {t_stats:.2f} ms + backward (dq + dn) {t_bwd:.2f} ms = {t_stats + t_bwd:.2f} ms against the output "
          f"layer's FLOP floor {flop_ms:.1f} ms ({flop_ms / (t_stats + t_bwd):.0%})")
    print(f"  row merge ({bag['rows'].shape[0]:,} rows) {t_merge:.3f} ms uniform, {t_pad:.3f} ms half padding; table update {t_upd:.2f} ms against its byte floor "
          f"{upd_floor:.2f} ms ({upd_floor / t_upd:.0%})")
    del tr, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--legs", default="a,b")
    ap.add_argument("--label-smoothing", type=float, default=0.0)
    ap.add_argument("--dropout", type=float, default=0.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_catalog_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card()}")
    legs = {"a": (1_000_000, 16_384), "b": (10_000_000, 4096)}
    for k in args.legs.split(","):
        leg(k, *legs[k], args, dev)


if __name__ == "__main__":
    np.set_printoptions(precision=4)
    main()
