"""The pretrained-embedding kernels (include/mm_b200.h K24) per element against float64: mm_pretrained_gather,
mm_pretrained_project (each instantiation: int32 / int64 ids and the dense-input path) and mm_pretrained_project_backward,
at widths Dp 1..1024 and d' 1..256, batches that take one, several and a ragged last lap of the grid, with NaN guard
columns around the slot, out-of-range ids counted and the backward bit-identical over two runs."""
import numpy as np
import pytest
import torch

from models_b200 import _cabi, ops

pytestmark = pytest.mark.gpu
DPS = [1, 12, 16, 300, 768, 1024]
OUTS = [1, 16, 64, 200, 256]
BATCHES = [1, 37, 1001, 65536, 65573]
GUARD = 3  # NaN columns left and right of the slot


def close(got, ref, tol, what, mag=None):
    """max |got - ref| relative to max |ref|, or to max |mag| (the size of the summed terms) where the sum cancels."""
    got = got.detach().double().cpu()
    ref = ref.detach().double().cpu()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    scale = max(float((ref if mag is None else mag).abs().max()) if ref.numel() else 0.0, 1e-30)
    err = float((got - ref).abs().max()) / scale if ref.numel() else 0.0
    assert err < tol, f"{what}: max |diff| / max |ref| = {err:.3e} (tol {tol})"


def _source(kind, B, Dp, rows, g, device):
    """(P, ids, P rows as read per sample in float64): kind "i32" / "i64" (ids into P) or "dense" (P is the (B, Dp) input)."""
    if kind == "dense":
        P = torch.randn((B, Dp), generator=g).to(device)
        return P, None, P.double()
    P = torch.randn((rows, Dp), generator=g).to(device)
    ids = torch.randint(0, rows, (B,), generator=g).to(device=device, dtype=torch.int32 if kind == "i32" else torch.int64)
    return P, ids, P.double()[ids.long()]


def _guarded(B, w, device):
    buf = torch.full((B, w + 2 * GUARD + 1), float("nan"), device=device)
    return buf, buf[:, GUARD:GUARD + w]


def _laps(B, N):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = -(-B // 64) * -(-N // 64)
    grid = min(tiles, sms * _cabi.PRETRAINED_CTAS_PER_SM)
    return tiles, grid


@pytest.mark.parametrize("kind", ["i32", "i64", "dense"])
@pytest.mark.parametrize("Dp", DPS)
def test_gather_matches_and_leaves_guards(device, kind, Dp):
    g = torch.Generator().manual_seed(Dp)
    for B in (1, 37, 1001):
        P, ids, rows = _source(kind, B, Dp, 97, g, device)
        buf, slot = _guarded(B, Dp, device)
        ops.pretrained_gather(P, ids, slot)
        assert torch.equal(slot.double().cpu(), rows.cpu()), (kind, Dp, B)
        assert torch.isnan(buf[:, :GUARD]).all() and torch.isnan(buf[:, GUARD + Dp:]).all()


@pytest.mark.parametrize("kind", ["i32", "i64", "dense"])
@pytest.mark.parametrize("Dp,N", [(Dp, N) for Dp in DPS for N in OUTS])
def test_project_matches_float64(device, kind, Dp, N):
    g = torch.Generator().manual_seed(Dp * 7 + N)
    B = 1001
    P, ids, rows = _source(kind, B, Dp, 211, g, device)
    W = (torch.randn((Dp, N), generator=g) / Dp ** 0.5).to(device)
    b = torch.randn(N, generator=g).to(device)
    buf, slot = _guarded(B, N, device)
    ops.pretrained_project(P, ids, W, b, slot)
    close(slot, rows @ W.double() + b.double(), 1e-5, f"project {kind} Dp={Dp} N={N}")
    assert torch.isnan(buf[:, :GUARD]).all() and torch.isnan(buf[:, GUARD + N:]).all()


@pytest.mark.parametrize("B", BATCHES)
def test_project_grid_laps(device, B):
    """One lap (B = 1, 37, 1001), several (65 536) and a ragged last lap (65 573) of the launch formula's grid."""
    Dp, N = 768, 256
    tiles, grid = _laps(B, N)
    if B >= 65536:
        assert tiles > grid, "the large batches must take more than one lap"
        if B == 65573:
            assert tiles % grid != 0, "65 573 samples must leave a ragged last lap"
    else:
        assert tiles <= grid
    g = torch.Generator().manual_seed(B)
    P, ids, rows = _source("i32", B, Dp, 4096, g, device)
    W = (torch.randn((Dp, N), generator=g) / Dp ** 0.5).to(device)
    buf, slot = _guarded(B, N, device)
    ops.pretrained_project(P, ids, W, None, slot)
    close(slot, rows @ W.double(), 1e-5, f"B={B}")
    assert torch.isnan(buf[:, :GUARD]).all() and torch.isnan(buf[:, GUARD + N:]).all()
    gbuf, gslot = _guarded(B, Dp, device)
    ops.pretrained_gather(P, ids, gslot)
    assert torch.equal(gslot.double().cpu(), rows.cpu())


def test_out_of_range_ids_are_counted_and_read_zero(device):
    P = torch.randn((10, 16), device=device)
    ids = torch.tensor([0, 10, -1, 3, 99], dtype=torch.int64, device=device)
    oob = torch.zeros(1, dtype=torch.int32, device=device)
    out = torch.full((5, 16), 7.0, device=device)
    ops.pretrained_gather(P, ids, out, oob)
    assert int(oob.item()) == 3
    assert torch.equal(out[[1, 2, 4]], torch.zeros((3, 16), device=device))
    W, b = torch.randn((16, 70), device=device), torch.randn(70, device=device)
    y = torch.zeros((5, 70), device=device)
    ops.pretrained_project(P, ids, W, b, y, oob)
    assert int(oob.item()) == 6, "the projection counts each sample once, whatever its number of column tiles"
    close(y[[1, 2, 4]], b.expand(3, 70), 1e-6, "out-of-range rows project to the bias")


@pytest.mark.parametrize("kind", ["i32", "i64", "dense"])
@pytest.mark.parametrize("l2", [False, True])
@pytest.mark.parametrize("Dp,N,B", [(1, 1, 37), (12, 16, 1001), (300, 200, 1001), (768, 64, 65536), (1024, 256, 65573),
                                    (16, 256, 1)])
def test_project_backward_matches_float64_and_repeats(device, kind, l2, Dp, N, B):
    g = torch.Generator().manual_seed(Dp + N + B + l2)
    P, ids, rows = _source(kind, B, Dp, 509, g, device)
    adds = [torch.randn((B, N + 5), generator=g).to(device)[:, 2:2 + N] for _ in range(3)]
    ypre = torch.randn((B, N), generator=g).to(device) if l2 else None
    dW, db = torch.full((Dp, N), float("nan"), device=device), torch.full((N,), float("nan"), device=device)
    ops.pretrained_project_backward(P, ids, adds, dW, db, ypre=ypre)
    gsum = sum(a.double() for a in adds)
    gmag = sum(a.double().abs() for a in adds)
    if l2:
        y = ypre.double().clone().requires_grad_(True)
        (y / torch.sqrt(torch.clamp((y * y).sum(1, keepdim=True), min=1e-12)) * gsum).sum().backward()
        gsum = y.grad
        # (g - u (u . g)) / |y| cancels exactly at N = 1; its terms are bounded by 2 |g| / |y|
        gmag = 2 * gmag.sum(1, keepdim=True) / ypre.double().norm(dim=1, keepdim=True)
        gmag = gmag.expand(-1, N)
    close(dW, rows.t() @ gsum, 1e-5, "dW", mag=rows.abs().t() @ gmag)
    close(db, gsum.sum(0), 1e-5, "db", mag=gmag.sum(0))
    dW2, db2 = torch.zeros_like(dW), torch.zeros_like(db)
    ops.pretrained_project_backward(P, ids, adds, dW2, db2, ypre=ypre)
    assert torch.equal(dW, dW2) and torch.equal(db, db2), "two runs of the backward differ"


def test_argument_checks(device):
    P = torch.zeros((4, 1025), device=device)
    with pytest.raises(NotImplementedError, match="1024"):
        ops.pretrained_gather(P, torch.zeros(2, dtype=torch.int32, device=device), torch.zeros((2, 1025), device=device))
    P = torch.zeros((4, 8), device=device)
    with pytest.raises(NotImplementedError, match="256"):
        ops.pretrained_project(P, None, torch.zeros((8, 257), device=device), None, torch.zeros((4, 257), device=device))
    with pytest.raises(ValueError, match="rows"):
        ops.pretrained_gather(P, None, torch.zeros((5, 8), device=device))
