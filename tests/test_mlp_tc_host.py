"""plan_tower, restated in tests/test_gpu_mlp_tc_kernels.py as `plan`, against the library's mm_mlp_tc_supported, and
the coverage of that file's case tables: every (N1P, HEADS) kernel, every (Np, KS) chain layer, the ring depths, every
activation at layer 1 and at a chain layer, every output and the DLRM table counts of the pairs hand-off.  Needs the
built library, not a GPU."""
import ctypes
import itertools

from models_b200 import _cabi, ops
from tests.test_gpu_mlp_tc_kernels import (ACTS, HEAD, HEADS, LAPS_M, OPERAND, PAIRS, PAIRS_K, ROWS, heads_acts, plan,
                                           supported, tiles_per_cta, wraps)
from tests.test_gpu_dense_tc_kernels import layout_of

N1PS = tuple(range(16, 129, 16))
WIDTHS = (1, 9, 16, 17, 32, 33, 48, 64, 65, 80, 96, 100, 112, 113, 128)
KS = sorted(set(range(1, 601, 17)) | {64, 65, 128, 129, 415, 560, 600})


def _library_supported(K, widths, with_head):
    wd = (ctypes.c_int * len(widths))(*widths)
    return bool(_cabi.load().mm_mlp_tc_supported(K, len(widths), wd, with_head))


def test_plan_matches_the_library():
    """mm_mlp_tc_supported for with_head 0 (fp32 rows), 1 (one fused head) and 2 (mm_mlp_tc_heads) over every 2- and
    3-layer tower of WIDTHS and the 4-layer towers of its multiples of 16 and their neighbours, each at several K in
    1..600; the grid holds towers on both sides of the shared-memory limit."""
    towers = [t for n in (2, 3) for t in itertools.product(WIDTHS, repeat=n)]
    towers += list(itertools.product((16, 33, 64, 65, 112, 128), repeat=4))
    fits = set()
    for i, t in enumerate(towers):
        for K in KS[i % 7::7]:
            for h in (0, 1, 2):
                want = supported(K, t, h)
                assert _library_supported(K, t, h) == want, (K, t, h)
                fits.add(want)
    assert fits == {True, False}
    assert not any(_library_supported(K, (128, 64), 0) for K in (0, -1))


def test_plan_formula():
    """Spot values: the README top tower holds 7 slots (2 KB = 14 slots per tile), one k-block caps the ring at 4, a
    16-wide layer 1 reaches the cap of 12; [112, 128, 128] fits, [128, 128, 128] does not (two 64 KB chain layers), and
    the heads' staging takes 4 KB more."""
    p = plan(415, (128, 64, 32))
    assert (p["K1p"], p["N1p"], p["KB"], p["stages"]) == (448, 128, 7, 7) and p["w_bytes"] == 32768 + 8192
    assert [(c["Np"], c["Kp"], c["KS"]) for c in p["chain"]] == [(64, 128, 8), (32, 64, 4)]
    assert plan(13, (128, 64))["stages"] == 4 and plan(415, (16, 128, 80))["stages"] == 12
    assert plan(100, (112, 128, 128))["fits"] and not plan(100, (128, 128, 128))["fits"]
    assert plan(415, (128, 64, 32), heads=True)["stages"] == 7 and plan(415, (16, 32), heads=True)["stages"] == 12
    assert ops.tc_padded_n(80) == 80 and ops.tc_padded_k(80) == 128


def _calls():
    """(label, K, widths, acts, outputs, multi-head kernel) of every launch the case tables make."""
    out = []
    for c in ROWS:
        col, stride = layout_of(c.layout, c.widths[-1])
        out.append(("rows", c.K, c.widths, c.acts, {"f32 stride N" if stride == c.widths[-1] else "f32 stride > N"} |
                    ({"f32 odd N"} if c.widths[-1] % 2 else set()), False))
    for c in HEAD:
        out.append(("head", c.K, c.widths, c.acts, {"head", "head + f32"}, False))
    for c in HEADS:
        out.append(("heads", c.K, c.widths, c.acts, {f"heads H{c.H}"}, True))
    for c in OPERAND:
        out.append(("operand", c.K, c.widths, c.acts, {"operand", "operand + f32"}, False))
    for c in PAIRS:
        out.append(("pairs", c.K, c.widths, c.acts, {"pairs f32", "pairs head"}, False))
        out.append(("pairs", c.K, c.widths, c.acts, {"pairs heads"}, True))
    return out


def test_cases_reach_every_variant():
    """Prints the kernels and chain variants with the cases that reach them, and names any variant, ring depth,
    activation or output that no case reaches."""
    calls = _calls()
    kernels, chains, stages, wrap, act1, actc, outs = {}, {}, set(), [], set(), set(), set()
    for label, K, widths, acts, o, heads in calls:
        p = plan(K, widths, heads)
        assert p["fits"] and supported(K, widths, 2 if heads else int(label == "head")), f"{label} {widths}: does not fit"
        kernels.setdefault((p["N1p"], heads), []).append(f"{label} {K}/{'x'.join(map(str, widths))}")
        for c in p["chain"]:
            chains.setdefault((c["Np"], c["KS"]), []).append(f"{label} {K}/{'x'.join(map(str, widths))}")
        stages.add(p["stages"])
        if wraps(p):
            wrap.append((label, K, widths))
        act1.add(acts[0])
        actc |= set(acts[1:])
        outs |= o
    print("\n".join(f"N1P {n:3} {'heads ' if h else 'single'}: {', '.join(v[:3])}" for (n, h), v in sorted(kernels.items())))
    print("\n".join(f"chain Np {n:3} KS {k}: {', '.join(v[:3])}" for (n, k), v in sorted(chains.items())))
    missing = sorted({(n, h) for n in N1PS for h in (False, True)} - set(kernels))
    assert not missing, f"(N1P, HEADS) kernels without a case: {missing}"
    missing = sorted({(n, k) for n in N1PS for k in (4, 8)} - set(chains))
    assert not missing, f"(Np, KS) chain variants without a case: {missing}"
    assert 4 in stages, "no case runs the smallest ring (4 slots)"
    assert 12 in stages, "no case runs the largest ring (12 slots)"
    assert any(s % 2 for s in stages), f"no case runs an odd ring depth: {sorted(stages)}"
    assert wrap, "no case wraps a tile's slots around the ring mid-tile"
    assert act1 == set(ACTS), f"layer-1 activations without a case: {sorted(set(ACTS) - act1)}"
    assert actc == set(ACTS), f"chain-layer activations without a case: {sorted(set(ACTS) - actc)}"
    want = {"f32 stride N", "f32 stride > N", "f32 odd N", "head", "head + f32", "heads H1", "heads H3", "heads H8",
            "operand", "operand + f32", "pairs f32", "pairs head", "pairs heads"}
    assert want <= outs, f"outputs without a case: {sorted(want - outs)}"
    assert {c.K for c in PAIRS} >= set(PAIRS_K), f"pairs K without a case: {sorted(set(PAIRS_K) - {c.K for c in PAIRS})}"
    assert {ops.pairs_cols(k - 64) for k in PAIRS_K} == {8, 40, 352, 496}
    assert {n for c in HEADS for n in [c.H]} == {1, 3, 8}
    assert set(ACTS) <= {a for i, c in enumerate(HEADS) for a in heads_acts(i, c.H)}
    # rows: a single row, both sides of a 64-row tile, two tiles and one, and several laps with odd and even tile counts
    assert {1, 63, 64, 65, 129} <= {c.M for c in ROWS}
    counts = tiles_per_cta(LAPS_M)
    assert LAPS_M in {c.M for c in ROWS} and max(counts) >= 3 and {n % 2 for n in counts} == {0, 1}, sorted(counts)
    assert any(not c.bias for c in ROWS) and any(c.bias for c in ROWS)
