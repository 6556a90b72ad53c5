"""The launch plans of mm_dense_wgrad[_split] and mm_dense_dgrad, restated in tests/test_gpu_dense_bwd_kernels.py, the
coverage of that file's case tables (every wgrad tile for fp32 and split X, every dgrad (KSTEPS, dZ load, store,
mask) combination) and the teeth of its bounds: on the CPU, in float64, on the same seeded data, each of a handful of
plausible kernel bugs moves some element outside the bound while the 3-pass split product itself stays inside.  Needs
no GPU."""
import pytest
import torch

from tests.test_gpu_dense_bwd_kernels import (DGRAD, TRAINER_MS, TRAINER_PAIRS, WG_TILES, WGRAD, case_dgrad_plan,
                                              case_wgrad_plan, dgrad_bound, dgrad_data, dgrad_plan, dgrad_ref, layout_of,
                                              wgrad_bounds, wgrad_data, wgrad_plan, wgrad_ref, wgrad_tile)
from tests.test_gpu_train_scale import GUARD, _dgrad_laps, _wgrad_launch

STORES = ("vec4", "vec2", "scalar")


def test_plan_formula():
    """Tiles at every K and N boundary, rows_per_cta / gx / ragged for a few (M, K, N) on 132 SMs, and the dgrad grid."""
    assert [wgrad_tile(k, 1)[0] for k in (1, 16, 17, 64, 65, 128, 129, 1165)] == [16, 16, 64, 64, 128, 128, 128, 128]
    assert [wgrad_tile(1, n)[1] for n in (1, 32, 33, 64, 65, 128, 129, 300)] == [32, 32, 64, 64, 128, 128, 128, 128]
    assert set(WG_TILES) == {wgrad_tile(k, n) for k in (1, 17, 65) for n in (1, 33, 65)}
    assert all(16 * wm * mt == ks and 8 * wn * nt == ns for (ks, ns), (wm, mt, wn, nt) in WG_TILES.items())
    p = wgrad_plan(65536, 415, 128, "f32", 416, 0, 128, 0)  # the DLRM top tower's first layer: ky 4, 66 CTAs
    assert (p["ky"], p["nz"], p["rows_per_cta"], p["gx"], p["ragged"]) == (4, 1, 1024, 64, False)
    p = wgrad_plan(257, 16, 32, "split", 0, 0, 32, 0)  # 264 CTAs' worth, the 256-row floor: one row left over
    assert (p["rows_per_cta"], p["gx"], p["last_rows"], p["ragged"], p["x_vec"]) == (256, 2, 1, True, None)
    p = wgrad_plan(9000, 1165, 1, "split", 0, 0, 1, 0)  # the wide head: 26 CTAs of 11 chunks
    assert (p["tile"], p["ky"], p["rows_per_cta"], p["gx"], p["last_rows"], p["z_vec"]) == ((128, 32), 10, 352, 26, 200, 0)
    p = wgrad_plan(4099, 13, 300, "f32", 13, 1, 300, 0)
    assert (p["tile"], p["nz"], p["rows_per_cta"], p["gx"], p["x_vec"], p["z_vec"]) == ((16, 128), 3, 256, 17, 0, 1)
    assert [dgrad_plan(1, 1, n, n, 0, 1, 0)["ksteps"] for n in (1, 32, 33, 64, 65, 128)] == [2, 2, 4, 4, 8, 8]
    q = dgrad_plan(40000, 128, 128, 132, 4, 136, 4, 144, 4)
    assert (q["ky"], q["gx"], q["laps"], q["store"], q["z_vec2"]) == (1, 264, 2, "vec4", 1)
    q = dgrad_plan(4099, 1165, 65, 1102, 1037, 1165, 0)
    assert (q["ky"], q["gx"], q["laps"], q["store"], q["z_vec2"], q["last_slab"]) == (10, 26, 2, "scalar", 0, 13)
    assert dgrad_plan(16, 64, 8, 8, 0, 136, 4, 70, 2)["store"] == "vec2"  # the mask alone rules out float4
    assert dgrad_plan(16, 64, 8, 8, 0, 68, 4, 69, 2)["store"] == "scalar"


def test_plans_agree_with_the_scale_tests():
    """The grid formulas test_gpu_train_scale's at-scale tests assert their premises with."""
    for M in (1, 255, 256, 257, 4099, 65536, 65573):
        for K in (1, 16, 17, 64, 65, 415, 1165):
            for N in (1, 32, 33, 64, 65, 128, 300):
                p = wgrad_plan(M, K, N, "f32", K, 0, N, 0, 132)
                assert (p["rows_per_cta"], p["gx"]) == _wgrad_launch(M, K, N, 132), (M, K, N)
            assert dgrad_plan(M, K, 8, 8, 0, K, 0, sms=132)["laps"] == _dgrad_laps(M, K, 132), (M, K)


def test_layouts():
    """The layouts' alignment classes, which the tables rely on to reach each load and store path."""
    def cls(layout, C):
        c, s = layout_of(layout, C)
        return 4 if c % 4 == 0 and s % 4 == 0 else 2 if c % 2 == 0 and s % 2 == 0 else 1

    for C in (1, 3, 13, 64, 65, 128, 1165):
        assert (cls("vec", C), cls("wide", C), cls("even", C), cls("odd", C), cls("off1", C)) == (4, 4, 2, 1, 1)
        assert layout_of("vec", C)[1] != layout_of("wide", C)[1] and layout_of("pad", C)[1] % 4 == 0
    assert layout_of("cat", 128) == (1037, 1165) and cls("cat", 128) == 1  # the parallel DCN body's dh[-1]


def test_wgrad_cases_reach_every_variant():
    """Prints the tile x X form table of the WGRAD cases (M/K/N of the first two per cell) and checks that every
    instantiation, both load paths of X and dZ, db given and None, ky, nz and gx >= 2, ragged and single-chunk last
    CTAs and the listed K, N and M occur."""
    plans = [(c, case_wgrad_plan(c)) for c in WGRAD]
    cells = {}
    for c, p in plans:
        cells.setdefault((p["tile"], p["xsplit"]), []).append(f"{c.M}/{c.K}/{c.N}")
    rows = [f"{'tile':>12}{'fp32 X':>34}{'split X':>34}"]
    for t in WG_TILES:
        rows.append(f"{str(t):>12}" + "".join(f"{', '.join(cells.get((t, s), [])[:2]):>34}" for s in (False, True)))
    print("\n".join(rows))
    assert set(cells) == {(t, s) for t in WG_TILES for s in (False, True)}, "a (tile, XSPLIT) instantiation without a case"
    assert {p["x_vec"] for _, p in plans if not p["xsplit"]} == {0, 1}
    assert {p["z_vec"] for _, p in plans} == {0, 1}
    assert any(p["z_vec"] == 0 and p["xsplit"] and c.N == 1 and not c.db for c, p in plans), "the wide head's call"
    assert {c.db for c in WGRAD} == {False, True}
    assert max(p["ky"] for _, p in plans) >= 3 and max(p["nz"] for _, p in plans) >= 3
    assert any(p["gx"] >= 2 and p["ragged"] for _, p in plans)
    assert any(p["gx"] >= 2 and p["last_rows"] == 32 for _, p in plans), "a last CTA of a single 32-row chunk"
    assert any(p["rows_per_cta"] > 256 for _, p in plans), "CTAs of more than 8 chunks"
    assert {1, 16, 17, 64, 65, 128, 129} <= {c.K for c in WGRAD} and max(c.K for c in WGRAD) > 256
    assert {1, 8, 32, 33, 64, 65, 128, 129} <= {c.N for c in WGRAD} and max(c.N for c in WGRAD) > 256
    assert {1, 31, 32, 33, 256, 257} <= {c.M for c in WGRAD}
    assert {"vec", "odd", "off1"} <= {c.x for c in WGRAD} and {"vec", "odd", "off1", "cat"} <= {c.dz for c in WGRAD}


def test_dgrad_cases_reach_every_variant():
    """Prints the (KSTEPS, dZ load) x (store, mask) table of the DGRAD cases and checks that every combination, ky >= 2,
    multi-lap grids, partial float4 groups on the float4 path, last slabs of <= 64 columns, masks at a stride other
    than dX's and the listed N, K and M occur."""
    plans = [(c, case_dgrad_plan(c)) for c in DGRAD]
    cells = {}
    for c, p in plans:
        cells.setdefault((p["ksteps"], p["z_vec2"], p["store"], p["mask"]), []).append(f"{c.M}/{c.K}/{c.N}")
    cols = [(s, m) for s in STORES for m in (False, True)]
    rows = [f"{'':14}" + "".join(f"{s + (' mask' if m else ''):>18}" for s, m in cols)]
    for ks in (2, 4, 8):
        for zv in (1, 0):
            rows.append(f"K{ks} {'z float2' if zv else 'z scalar':<10}" +
                        "".join(f"{', '.join(cells.get((ks, zv, s, m), [])[:1]):>18}" for s, m in cols))
    print("\n".join(rows))
    want = {(ks, zv, s, m) for ks in (2, 4, 8) for zv in (0, 1) for s in STORES for m in (False, True)}
    assert set(cells) == want, f"combinations without a case: {sorted(want - set(cells))}"
    assert any(p["ky"] >= 2 and p["laps"] >= 2 for _, p in plans) and any(p["ky"] == 1 and p["laps"] >= 2 for _, p in plans)
    assert any(p["store"] == "vec4" and c.K % 4 for c, p in plans), "a partial float4 group on the float4 path"
    assert any(p["ky"] >= 2 and p["last_slab"] <= 64 for _, p in plans), "a last slab whose second chunk is skipped"
    assert any(p["ky"] == 1 and p["last_slab"] <= 64 for _, p in plans)
    other = [(c, p) for c, p in plans if c.mask and layout_of(c.mask, c.K)[1] != layout_of(c.dx, c.K)[1]]
    assert {p["store"] for _, p in other} == set(STORES), "a mask at its own stride on every store path"
    assert {1, 8, 17, 32, 33, 64, 65, 127, 128} <= {c.N for c in DGRAD}
    assert {1, 3, 13, 64, 65, 128, 129, 415, 1165} <= {c.K for c in DGRAD}
    assert {1, 15, 16, 17} <= {c.M for c in DGRAD}


def test_trainer_cases_are_in_the_tables():
    """Every (M, K, N) the first wgrad / dgrad test ran, with fp32 X at the trainer's padded stride and split X, and
    dX without and with the mask at that stride."""
    for K, N in TRAINER_PAIRS:
        for M in TRAINER_MS:
            assert {c.x for c in WGRAD if (c.M, c.K, c.N) == (M, K, N) and c.db} >= {"pad", "split"}, (M, K, N)
            assert {c.mask for c in DGRAD if (c.M, c.K, c.N, c.dx) == (M, K, N, "pad")} >= {None, "pad"}, (M, K, N)


# ---------------------------------------------------------------------------------------------------------------
# teeth: plausible bugs break the bounds on the tables' own data
# ---------------------------------------------------------------------------------------------------------------
def _bf16(t):
    return t.to(torch.bfloat16).double()


def _split(t):
    """(hi, lo) of the split-bf16 operand, in float64."""
    hi = _bf16(t)
    return hi, _bf16((t.double() - hi).float())


def _wgrad_teeth_cases():
    return [c for c in WGRAD if 64 <= c.M <= 1000 and c.N >= 16 and c.K <= 415][:5]


def _dgrad_teeth_cases():
    return [c for c in DGRAD if c.mask and c.M >= 15 and c.M <= 1001 and c.K <= 415
            and layout_of(c.mask, c.K)[1] != layout_of(c.dx, c.K)[1]][:5]


def _breaks(got, ref, bound):
    return bool(((got - ref).abs() > bound).any())


@pytest.mark.parametrize("bug", ["three_pass_is_inside", "chunk_dropped", "ntile_misplaced", "hi_hi_only"])
def test_wgrad_bound_has_teeth(bug):
    cases = _wgrad_teeth_cases()
    assert len(cases) >= 3
    for c in cases:
        X, dZ, dw0, db0 = wgrad_data(c.M, c.K, c.N, WGRAD.index(c))
        p = case_wgrad_plan(c)
        ref, _ = wgrad_ref(X, dZ, dw0, db0)
        bw, _ = wgrad_bounds(X, dZ, dw0, db0, p["rows_per_cta"], p["gx"])
        xh, xl = _split(X)
        zh, zl = _split(dZ)
        prod = xh.t() @ zh + xh.t() @ zl + xl.t() @ zh
        if bug == "three_pass_is_inside":
            assert not _breaks(dw0.double() + prod, ref, bw), f"{c}: the 3-pass product alone breaks the bound"
            continue
        if bug == "chunk_dropped":  # rows 32..63 never reach the accumulator
            keep = torch.ones(c.M, dtype=torch.bool)
            keep[32:64] = False
            got = dw0.double() + X.double()[keep].t() @ dZ.double()[keep]
        elif bug == "ntile_misplaced":  # the accumulators of n-tiles 0 and 1 (8 columns each) land in each other's columns
            part = X.double().t() @ dZ.double()
            got = dw0.double() + torch.cat([part[:, 8:16], part[:, :8], part[:, 16:]], 1)
        else:  # one bf16 pass instead of three
            got = dw0.double() + xh.t() @ zh
        assert _breaks(got, ref, bw), f"{c}: {bug} stays within the dW bound"


@pytest.mark.parametrize("bug", ["three_pass_is_inside", "kstep_dropped", "mask_at_dx_stride", "hi_hi_only"])
def test_dgrad_bound_has_teeth(bug):
    cases = _dgrad_teeth_cases()
    assert len(cases) >= 3
    for c in cases:
        dZ, W, mask = dgrad_data(c.M, c.K, c.N, 5000 + DGRAD.index(c))
        ref, bound = dgrad_ref(dZ, W, mask), dgrad_bound(dZ, W, mask)
        zh, zl = _split(dZ)
        wh, wl = _split(W)
        on = mask > 0
        if bug == "three_pass_is_inside":
            assert not _breaks((zh @ wh.t() + zh @ wl.t() + zl @ wh.t()) * on, ref, bound), f"{c}: the 3-pass product breaks the bound"
            continue
        if bug == "kstep_dropped":  # the last 16-wide k-step's columns of dZ never reach the MMAs
            j = (c.N - 1) // 16
            d = dZ.double().clone()
            d[:, 16 * j:16 * j + 16] = 0.0
            got = (d @ W.double().t()) * on
        elif bug == "mask_at_dx_stride":  # mask element (r, k) read at r * dX's stride + k of the mask's NaN buffer
            mc, ms = layout_of(c.mask, c.K)
            buf = torch.full(((c.M + GUARD) * ms,), float("nan"), dtype=torch.float64)
            buf.view(c.M + GUARD, ms)[:c.M, mc:mc + c.K] = mask.double()
            idx = mc + torch.arange(c.M).view(-1, 1) * layout_of(c.dx, c.K)[1] + torch.arange(c.K).view(1, -1)
            wrong = buf[idx.clamp_max(buf.numel() - 1)]
            got = (dZ.double() @ W.double().t()) * (wrong > 0)
        else:  # one bf16 pass instead of three
            got = (zh @ wh.t()) * on
        assert _breaks(got, ref, bound), f"{c}: {bug} stays within the dX bound"
