#!/usr/bin/env python
"""Compare two or more builds of the in-batch loss kernels (inbatch_flash.cu) in one process, on the same inputs.

    python tools/inbatch_ab.py LIB [LIB ...] [--blocks 10] [--launches 5]

Each LIB is a libmm_b200.so (for example this tree's models_b200/_lib/libmm_b200.so and one built from another commit).
Cases, all with seeded inputs:
  * in-batch (N = B = 16 384, the negatives are the positives, dpos aliasing dneg, false negatives down-scored by ids
    with repeats off the diagonal) at D = 64 and D = 128: mm_inbatch_softmax_ce_backward (T = 1, scalar c = 1 / B) and
    mm_inbatch_pairwise_fwd + _bwd for all seven kinds;
  * ragged (B = 1000, N = 1300 separate negatives, D = 100, T = 0.05, down-scored): the soft-max backward with logQ and a
    per-row row_scale, and every pairwise kind with dpos in its own buffer.
The soft-max forward statistics come from the first library (mm_inbatch_softmax_ce is not part of the comparison).  Every
library's stats, loss, dq, dpos and dneg are compared with the first one's, bit for bit.

Timing: the libraries take turns, one block of `launches` calls each (one soft-max backward, or one pairwise forward +
backward), `blocks` times, with one CUDA-event pair around each block, for each in-batch case.  Prints the card name
and power limit, then one JSON line per case and library (median and range of the per-call block means) and one per
case with the ratios of the block medians to the first library's.  Passing one library twice measures the spread of
repeating the same code.
"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from models_b200 import _cabi, ops  # noqa: E402
from interact_ab import card, load_lib  # noqa: E402

MIN_FLOAT = -655.04


def case_inputs(B, N, D, in_batch, dev, seed):
    """Queries, positives, negatives (the positives when in_batch), ids with repeats, their split operands."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    q = (torch.randn((B, D), generator=g) * (2.0 / D ** 0.5)).to(dev)
    pos = (torch.randn((B, D), generator=g) * (2.0 / D ** 0.5)).to(dev)
    neg = pos if in_batch else (torch.randn((N, D), generator=g) * (2.0 / D ** 0.5)).to(dev)
    pos_ids = torch.randint(0, max(1, B // 2), (B,), generator=g).to(dev)
    neg_ids = pos_ids if in_batch else torch.randint(0, max(1, B // 2), (N,), generator=g).to(dev)
    return g, dict(q=q, pos=pos, pos_ids=pos_ids, neg_ids=neg_ids, qs=ops.split_rows(q), ns=ops.split_rows(neg), D=D,
                   in_batch=in_batch)


def make_cases(dev):
    """name -> (alloc, run, timed): alloc() makes the output buffers, run(out) writes every compared output into them."""
    cases = {}
    for D in (64, 128):
        _, x = case_inputs(16384, 16384, D, True, dev, 11 + D)
        cases[f"softmax_inbatch_D{D}"] = softmax_case(x, 1.0, None, None, dev)
        for kind in _cabi.PAIRWISE_KINDS:
            cases[f"{kind}_inbatch_D{D}"] = pairwise_case(x, kind, 1.0, dev)
    B, N = 1000, 1300
    g, x = case_inputs(B, N, 100, False, dev, 5)
    neg_prob = (torch.rand(N, generator=g) * 1e-2 + 1e-4).to(dev)
    row_scale = (torch.rand(B, generator=g) + 0.5).to(dev) / B
    cases["softmax_ragged"] = softmax_case(x, 0.05, neg_prob, row_scale, dev)
    for kind in _cabi.PAIRWISE_KINDS:
        cases[f"{kind}_ragged"] = pairwise_case(x, kind, 0.05, dev)
    return cases


def outputs(x, dev, stats_cols=0):
    """loss, dq, dneg and dpos (dneg's buffer in the in-batch layout), pre-filled so unwritten words show up"""
    B, N, D = x["qs"].shape[0], x["ns"].shape[0], x["D"]
    out = {"loss": torch.zeros(1, dtype=torch.float32, device=dev), "dq": torch.full((B, D), 7.0, device=dev),
           "dneg": torch.full((N, D), 7.0, device=dev)}
    out["dpos"] = out["dneg"] if x["in_batch"] else torch.full((B, D), 7.0, device=dev)
    if stats_cols:
        out["stats"] = torch.full((B, stats_cols), 7.0, device=dev)
    return out


def softmax_case(x, T, neg_prob, row_scale, dev):
    B, N, D = x["qs"].shape[0], x["ns"].shape[0], x["D"]
    kw = dict(pos_ids=x["pos_ids"], neg_ids=x["neg_ids"], downscore=True, false_neg_score=MIN_FLOAT, neg_prob=neg_prob,
              temperature=T)
    pos_logit = torch.empty(B, dtype=torch.float32, device=dev)
    ops.positive_scores(x["q"], x["pos"], pos_logit, None, T)
    stats = torch.empty((B, 3), dtype=torch.float32, device=dev)
    ws = torch.empty(max(ops.catalog_workspace_bytes(B, N), 16), dtype=torch.uint8, device=dev)
    ops.inbatch_softmax_ce_split(x["qs"], x["ns"], D, pos_logit, stats, ws, **kw)  # the forward, on the first library
    scale = row_scale if row_scale is not None else torch.full((1,), 1.0 / B, dtype=torch.float32, device=dev)

    def run(out):
        ops.inbatch_softmax_ce_backward(x["qs"], x["ns"], D, stats, x["q"], x["pos"], scale, out["dq"], out["dpos"], out["dneg"],
                                        loss=out["loss"], **kw)

    return (lambda: outputs(x, dev)), run, x["in_batch"]


def pairwise_case(x, kind, T, dev):
    B, D = x["qs"].shape[0], x["D"]
    kw = dict(pos_ids=x["pos_ids"], neg_ids=x["neg_ids"], downscore=True, false_neg_score=MIN_FLOAT, temperature=T,
              reg_lambda=1.0)
    pos_logit = torch.empty(B, dtype=torch.float32, device=dev)
    ops.positive_scores(x["q"], x["pos"], pos_logit, None, T)

    def run(out):
        ops.inbatch_pairwise(x["qs"], x["ns"], D, pos_logit, out["stats"], kind, loss=out["loss"], **kw)
        ops.inbatch_pairwise_backward(x["qs"], x["ns"], D, pos_logit, out["stats"], x["q"], x["pos"], out["dq"], out["dpos"],
                                      out["dneg"], kind, **kw)

    return (lambda: outputs(x, dev, 4)), run, x["in_batch"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+")
    ap.add_argument("--blocks", type=int, default=10)
    ap.add_argument("--launches", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    print(card(), flush=True)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    libs = [load_lib(p) for p in args.libs]
    _cabi._lib = libs[0]  # inputs, split operands and the soft-max forward statistics come from the first library
    cases = make_cases(dev)
    torch.cuda.synchronize()

    # bit-identity: every output of every case against the first library's
    all_same = True
    for name, (alloc, run, _) in cases.items():
        firsts, diffs = None, []
        for lib in libs:
            _cabi._lib = lib
            out = alloc()
            run(out)
            torch.cuda.synchronize()
            if firsts is None:
                firsts = out
            diffs.append({k: int((out[k].view(torch.int32) != firsts[k].view(torch.int32)).sum()) for k in sorted(out)})
        same = [not any(d.values()) for d in diffs]
        all_same &= all(same)
        print(json.dumps({"case": name, "bit_identical_to_first": same, "differing_words": diffs}), flush=True)

    # timing: alternating blocks per library, in-batch cases only
    for name, (alloc, run, timed) in cases.items():
        if not timed:
            continue
        outs = [alloc() for _ in libs]
        for j, lib in enumerate(libs):  # warm-up, and the output buffers each block reuses
            _cabi._lib = lib
            for _ in range(2):
                run(outs[j])
        torch.cuda.synchronize()
        per = [[] for _ in libs]
        for _ in range(args.blocks):
            for j, lib in enumerate(libs):
                _cabi._lib = lib
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.launches):
                    run(outs[j])
                e1.record()
                torch.cuda.synchronize()
                per[j].append(e0.elapsed_time(e1) / args.launches)
        for j, p in enumerate(args.libs):
            print(json.dumps({"case": name, "lib": p, "ms_median": float(np.median(per[j])), "ms_min": float(np.min(per[j])),
                              "ms_max": float(np.max(per[j])), "blocks": args.blocks, "calls_per_block": args.launches}))
        ratios = [[b / a for a, b in zip(per[0], per[j])] for j in range(len(libs))]
        print(json.dumps({"case": name, "median_ratio_to_first": [float(np.median(r)) for r in ratios],
                          "ratio_of_medians": [float(np.median(per[j]) / np.median(per[0])) for j in range(len(libs))]}),
              flush=True)
    print(json.dumps({"all_bit_identical": bool(all_same)}))
    return 0 if all_same else 2


if __name__ == "__main__":
    sys.exit(main())
