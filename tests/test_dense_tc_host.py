"""dense_tc_launch's plan, restated in tests/test_gpu_dense_tc_kernels.py, against the library's padding rules, and the
coverage of that file's case tables: every (schedule, tile width, ring depth) the launcher can choose, every epilogue
and every store path.  Needs the built library, not a GPU."""
from models_b200 import ops
from tests.test_gpu_dense_tc_kernels import (ACTS, CROSS, DENSE, HEAD, SCORER, fp32_paths, layout_of, padded_k, padded_n,
                                             plan, scorer_out, split_gap)

BNS = tuple(range(16, 129, 16))


def test_padding_matches_the_library():
    """mm_tc_padded_n / mm_tc_padded_k, which every caller sizes its operands by, for every N and K in 1..2048."""
    for n in range(1, 2049):
        assert ops.tc_padded_n(n) == padded_n(n), n
        assert ops.tc_padded_k(n) == padded_k(n), n


def reachable():
    """Every (schedule, BN, stages) the launcher can produce: interleaved at every BN and K, resident-A (scorer,
    Kp <= 128, >= 8 n-tiles of 128) at both of its Kp."""
    out = {("interleaved", min(padded_n(n), 128), plan(128, k, n)["stages"]) for n in BNS + (129,) for k in range(1, 2049, 7)}
    out |= {("resident", 128, plan(128, k, 1024, score=True)["stages"]) for k in (64, 128)}
    return out


def case_plans():
    """(schedule, BN, stages, case label) of every GEMM in the case tables."""
    rows = [(c.M, c.K, c.N, False, f"N{c.N} K{c.K}") for c in DENSE]
    rows += [(c.M, c.d, c.d, False, f"x{c.d}") for c in CROSS]
    rows += [(c.M, c.K, c.N, False, f"h{c.N} K{c.K}") for c in HEAD]
    rows += [(c.B, c.D, c.N, True, f"s{c.N} D{c.D}") for c in SCORER]
    out = []
    for M, K, N, score, label in rows:
        p = plan(M, K, N, score=score)
        out.append(("resident" if p["resident"] else "interleaved", p["BN"], p["stages"], label))
    return out


def test_plan_formula():
    """Spot values of the ring depth: BN 16 / 32 hold 5 stages, 48 four, 64..96 three, 112 and 128 two; one k-block
    caps the ring at 2 and two at 4; the resident schedule holds 3 (Kp = 64) or 2 (Kp = 128)."""
    assert [plan(128, 1037, n)["stages"] for n in (1, 17, 33, 50, 65, 83, 100, 113, 129)] == [5, 5, 4, 3, 3, 3, 2, 2, 2]
    assert [plan(128, k, 1)["stages"] for k in (1, 64, 65, 128, 129)] == [2, 2, 4, 4, 5]
    assert [plan(128, k, 897, score=True)["resident"] for k in (64, 128, 129)] == [True, True, False]
    assert not plan(128, 64, 896, score=True)["resident"] and not plan(128, 64, 897)["resident"]
    assert [plan(128, k, 897, score=True)["stages"] for k in (64, 128)] == [3, 2]
    assert plan(300 * 128 - 37, 64, 100)["tiles"] == 300 and plan(1, 64, 1037)["n_tiles_n"] == 9
    assert fp32_paths(128, 100, 100, 0) == {"interior", "edge"} and fp32_paths(128, 96, 96, 0) == {"interior"}
    assert fp32_paths(31, 100, 104, 4) == {"edge"} and fp32_paths(128, 96, 97, 0) == fp32_paths(128, 96, 100, 1) == {"scalar"}
    assert split_gap(1) and split_gap(100) and not split_gap(64) and not split_gap(128) and not split_gap(129)


def test_cases_reach_every_variant():
    """Prints the BN x ring-depth table of the cases that reach each pair (N/K: act(xW + b); x: cross; h: head;
    s: scorer; "-": the launcher cannot produce the pair) and checks that no reachable pair, schedule, activation,
    epilogue or store path is missing."""
    want = reachable()
    cells = {}
    for sched, bn, st, label in case_plans():
        cells.setdefault((sched, bn, st), []).append(label)
    depths = sorted({st for _, _, st in want})
    rows = [f"{'':12}" + "".join(f"{d:>26}" for d in depths)]
    for sched in ("interleaved", "resident"):
        for bn in BNS:
            if not any((sched, bn, d) in want for d in depths):
                continue
            line = f"{sched[:5]} BN{bn:<4}"
            for d in depths:
                got = cells.get((sched, bn, d), [])
                line += f"{(', '.join(got[:2]) if got else ('' if (sched, bn, d) in want else '-')):>26}"
            rows.append(line)
    print("\n".join(rows))
    assert want <= set(cells), f"(schedule, BN, stages) without a case: {sorted(want - set(cells))}"
    assert set(cells) <= want, "a case's plan is not among the reachable ones"
    wraps = {plan(c.M, c.K, c.N)["BN"] for c in DENSE if plan(c.M, c.K, c.N)["KB"] > plan(c.M, c.K, c.N)["stages"]}
    assert wraps == set(BNS), f"tile widths whose ring never wraps inside one tile: {sorted(set(BNS) - wraps)}"

    # epilogues
    assert {(c.act, c.bias) for c in DENSE} == {(a, b) for a in ACTS for b in (False, True)}
    assert {c.passes for c in DENSE} == {1, 3}
    assert {c.out for c in DENSE} == {"f32", "split", "both"}
    vec_x = {layout_of(c.layout, c.d)[1] % 4 == 0 and layout_of(c.layout, c.d)[0] % 4 == 0 for c in CROSS}
    assert vec_x == {True, False}, "cross needs vector and scalar x0 / x loads"
    assert {(c.head_act, plan(c.M, c.K, c.N)["BN"]) for c in HEAD} == {(a, bn) for a in ACTS for bn in (16, 32)}
    assert {c.bias for c in HEAD} == {False, True}
    assert {c.ids for c in SCORER} >= {None, "i32", "narrow", "wide"}
    assert {c.T for c in SCORER} == {1.0, 0.05} and {c.logq for c in SCORER} == {False, True}
    assert {(c.N, c.D, plan(c.B, c.D, c.N, score=True)["resident"]) for c in SCORER} >= {
        (896, 64, False), (897, 64, True), (896, 128, False), (897, 128, True), (896, 192, False), (897, 192, False)}
    # stores
    paths = set()
    for c in DENSE:
        if c.out != "split":
            col, stride = layout_of(c.layout, c.N)
            paths |= fp32_paths(c.M, c.N, stride, col)
    assert paths == {"interior", "edge", "scalar"}
    spaths = set()
    for c in SCORER:
        col, stride = scorer_out(c.B, c.N, c.layout)
        spaths |= fp32_paths(c.B, c.N, stride, col + 1)
    assert "scalar" in spaths and spaths & {"interior", "edge"}
    gaps = {split_gap(c.N) for c in DENSE if c.out != "f32"} | {split_gap(c.d) for c in CROSS if c.out != "f32"}
    assert gaps == {True, False}, "split outputs with and without a padding gap"
    # rows: 1, the 128-row tile edges, a ragged size, and one interleaved lap case of >= 3 ragged laps per n-tile count
    assert {1, 127, 128, 129, 1001} <= {c.M for c in DENSE}
    laps = [plan(c.M, c.K, c.N) for c in DENSE if c.M > 1001]
    assert any(p["tiles_per_cta"] >= 3 and p["tiles"] % p["grid"] and p["n_tiles_n"] == 1 for p in laps)
    assert any(p["tiles_per_cta"] >= 3 and p["tiles"] % p["grid"] and p["n_tiles_n"] > 1 for p in laps)
    big = [plan(c.B, c.D, c.N, score=True) for c in SCORER if c.B > 1001]
    assert any(p["resident"] and p["tiles_per_cta"] >= 3 and p["tiles"] % p["tiles_per_cta"] for p in big)
