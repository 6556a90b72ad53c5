"""The Dense layers' backward GEMMs of every training step (models_b200/csrc/train_dense.cu) at every variant their
launchers dispatch:

  * mm_dense_wgrad / mm_dense_wgrad_split (dW += X^T dZ, db += column sums of dZ): wgrad_dispatch picks one of nine
    (KS, NS) tiles of wgrad_kernel<WM, MT, WN, NT, XSPLIT> from K (<= 16 / <= 64 / > 64) and N (<= 32 / <= 64 / > 64),
    each compiled for fp32 X and for split-bf16 X: 18 kernels.  launch_wgrad spreads the batch over gx CTAs of
    rows_per_cta rows (a multiple of 32, at least 256) per (k-tile, n-tile); fp32 X and dZ rows are read as float4 when
    row stride and base allow (x_vec, z_vec), as scalars otherwise.
  * mm_dense_dgrad (dX = dZ W^T, zeroed where mask <= 0): dgrad_kernel<KSTEPS> for N <= 32 / <= 64 / <= 128, with 8-byte
    or scalar dZ loads (z_vec2) and three stores: through a shared-memory stage as float4 (x_vec4), as float2 (x_vec2) or
    as scalars; the mask's stride and alignment gate x_vec2 and x_vec4 along with dX's.

`wgrad_plan` and `dgrad_plan` restate both launchers; tests/test_dense_bwd_host.py checks, without a GPU, that the case
tables reach every variant and that the bounds below catch plausible kernel bugs.

Each case makes one call and compares EVERY output element with float64 computed on the device.  Bounds, with E = 2^-24
and UNIT = 3 * 2^-16 (one 3-pass split-bf16 product a b = ah bh + ah bl + al bh: a = ah + al leaves at most
2^-8 * 2^-8 of |a| since bf16 rounds within 2^-8, as does b, and al bl is dropped; see test_gpu_dense_tc_kernels):
  * dW: a CTA sums its rows_per_cta batch rows in 32-row chunks, three MMA accumulations per 16 rows: a chain of
    3 rows / 16 fp32 additions onto its accumulator, each within E of the sum of the absolute terms; the gx CTAs along
    the batch then meet in fp32 atomics onto the starting value dw0, gx more additions, each within E (|dw0| + the
    absolute terms).  So |dW - dw0 - X^T dZ| <= (UNIT + (3 rows / 16 + gx) E) (|X|^T |dZ|) + gx E |dw0| to first order,
    asserted at twice the first term: 2 (UNIT + (3 rows / 16 + gx) E) (|X|^T |dZ|) + gx E |dw0| (every one of the gx
    atomics rounds onto a sum that holds dw0, so the starting value's share grows with gx, not just E |dw0|).
  * db: a thread sums the dZ values it stages (at most rows_per_cta of them), the CTA folds its threads through
    shared-memory atomics (at most 256 more additions), gx atomics onto db0: 2 (rows + 256 + gx) E sum |dZ| + gx E |db0|.
  * dX: N split products (UNIT each) summed in fp32 by the MMAs (N E): 2 (UNIT + N E) (|dZ| |W|^T), and exactly 0 where
    the mask is <= 0.
A lost 32-row chunk, a dropped 16-wide k-step, an n-tile of dW written to the wrong columns, a mask read at dX's stride
or a one-pass (hi * hi) product moves elements by far more (tests/test_dense_bwd_host.py shows each on these data).

The data gives the bounds teeth: exact-zero rows in X and dZ, a relu-like non-negative X (exact zeros, and the mask of
dgrad), both signs in dZ and W, and one 32-row block scaled by 40, so that a bound taken relative to the largest
element would hide errors in the small ones.  Every fp32 operand is a view of a NaN buffer with guard rows past M and,
in most layouts, guard columns beside the view (a read outside the operand poisons the result); every output is a view
of a NaN buffer whose elements outside the output must stay NaN.  dW and db start non-zero (the kernels accumulate)
and are contiguous views at the head of NaN buffers whose tails must stay NaN.  wgrad's CTAs meet in float atomics, so
its runs are not compared bit for bit; dgrad has none: a repeat and a 16-row-aligned window launched alone must
reproduce its rows bit for bit."""
from collections import namedtuple

import pytest
import torch

from models_b200 import ops
from tests.test_gpu_train_scale import E, GUARD, U, _nan, _sms, _within

pytestmark = pytest.mark.gpu
UNIT = 3 * U  # relative error of one 3-pass split-bf16 product
SMS = 132  # SMs of an H100 SXM: the tables are sized for it (the GPU tests plan with the device's own count)
D_CAT = 1037  # d of the DCN-v2 body whose [cross | deep] head input the wide head reads (d + 128 = 1165 columns)
TAIL = 64  # NaN floats past dW and db

# wgrad_dispatch's tiles: (KS, NS) -> (WM, MT, WN, NT); KS = 16 WM MT, NS = 8 WN NT, 32 WM WN threads
WG_TILES = {
    (16, 32): (1, 1, 4, 1), (16, 64): (1, 1, 8, 1), (16, 128): (1, 1, 8, 2),
    (64, 32): (4, 1, 2, 2), (64, 64): (2, 2, 4, 2), (64, 128): (2, 2, 4, 4),
    (128, 32): (4, 2, 2, 2), (128, 64): (4, 2, 2, 4), (128, 128): (4, 2, 4, 4),
}


def _c4(n):
    return (n + 3) // 4 * 4


def layout_of(layout, C):
    """(first column of the view in its row, row stride) of an (M, C) operand; buffers start 16-byte aligned.
    dense: contiguous; pad: columns 0..C of rows of _c4(C) floats (the trainer's padded stride); vec: columns 4..4+C of
    rows of 4k floats; wide: as vec at another stride; even: columns 2..2+C of rows of 4k + 2 floats (8-byte aligned
    only); odd: columns 2..2+C of rows of 4k + 1 floats; off1: columns 1..1+C of rows of 4k floats (4-byte aligned);
    cat: columns d..d+C of a (M, d + C) buffer, d = 1037, as the parallel DCN body cuts its deep output's gradient out
    of the head's input gradient."""
    return {"dense": (0, C), "pad": (0, _c4(C)), "vec": (4, _c4(C) + 8), "wide": (4, _c4(C) + 16),
            "even": (2, _c4(C) + 6), "odd": (2, _c4(C) + 5), "off1": (1, _c4(C) + 8), "cat": (D_CAT, D_CAT + C)}[layout]


# ---------------------------------------------------------------------------------------------------------------
# the launchers, restated
# ---------------------------------------------------------------------------------------------------------------
def wgrad_tile(K, N):
    """wgrad_dispatch's (KS, NS)."""
    return (128 if K > 64 else 64 if K > 16 else 16), (128 if N > 64 else 64 if N > 32 else 32)


def wgrad_plan(M, K, N, x_form, x_stride, x_offset, dz_stride, dz_offset, sms=SMS):
    """What mm_dense_wgrad (x_form "f32") or mm_dense_wgrad_split ("split") launches; offsets in floats from a 16-byte
    aligned address.  launch_wgrad: ky x nz tiles of dW, 2 SMs' worth of CTAs shared among them, rows_per_cta = the
    batch over those CTAs rounded up to 32 and at least 256, gx = the CTAs along the batch; the last CTA holds
    last_rows rows (ragged: not a multiple of the 32-row chunk)."""
    KS, NS = wgrad_tile(K, N)
    ky, nz = -(-K // KS), -(-N // NS)
    ctas = max(1, 2 * sms // (ky * nz))
    rows = max(256, -(-(-(-M // ctas)) // 32) * 32)
    gx = -(-M // rows)
    last = M - (gx - 1) * rows
    split = x_form == "split"
    return dict(tile=(KS, NS), xsplit=split, ky=ky, nz=nz, rows_per_cta=rows, gx=gx, last_rows=last, ragged=last % 32 != 0,
                x_vec=None if split else int(x_stride % 4 == 0 and x_offset % 4 == 0),
                z_vec=int(dz_stride % 4 == 0 and dz_offset % 4 == 0))


def dgrad_plan(M, K, N, dz_stride, dz_offset, dx_stride, dx_offset, mask_stride=None, mask_offset=None, sms=SMS):
    """What mm_dense_dgrad launches: KSTEPS 16-wide k-steps, ky 128-column slabs of dX, gx CTAs of 8 warps (a warp per
    16 rows) capped at 2 SMs / ky, laps of the grid-stride loop, the load / store flags and the store path they select;
    last_slab = dX columns of the last slab (<= 64: its second 64-column chunk is skipped)."""
    ksteps = 2 if N <= 32 else 4 if N <= 64 else 8
    ky = -(-K // 128)
    tiles = -(-M // 16)
    gx = min(-(-tiles // 8), max(1, 2 * sms // ky))
    laps = -(-tiles // (gx * 8))
    masked = mask_stride is not None

    def aligned(s, o, q):
        return s % q == 0 and o % q == 0

    x_vec2 = aligned(dx_stride, dx_offset, 2) and (not masked or aligned(mask_stride, mask_offset, 2))
    x_vec4 = aligned(dx_stride, dx_offset, 4) and (not masked or aligned(mask_stride, mask_offset, 4))
    return dict(ksteps=ksteps, ky=ky, gx=gx, laps=laps, z_vec2=int(aligned(dz_stride, dz_offset, 2)), x_vec2=int(x_vec2),
                x_vec4=int(x_vec4), store="vec4" if x_vec4 else "vec2" if x_vec2 else "scalar", mask=masked,
                last_slab=K - (ky - 1) * 128)


# ---------------------------------------------------------------------------------------------------------------
# case tables (importable without CUDA)
# ---------------------------------------------------------------------------------------------------------------
# x: "split" (the forward layer's split-bf16 operand) or the fp32 layout of X; dz: the layout of dZ
Wgrad = namedtuple("Wgrad", "M K N x dz db")
# dz, dx: layouts; mask: None or the mask's layout
Dgrad = namedtuple("Dgrad", "M K N dz dx mask")

# the (K, N) pairs and batch sizes the trainer's first kernel tests ran: the interaction output (415), the bottom
# tower's 13 columns, the top and bottom towers' layers
TRAINER_PAIRS = ((13, 128), (128, 64), (415, 128), (64, 32), (31, 24), (24, 8), (200, 100), (16, 16))
TRAINER_MS = (1, 37, 1000, 4099)

WGRAD = [
    # (16, 32): K = N = M = 1; gx = 2 with a ragged last CTA of one row
    Wgrad(1, 1, 1, "vec", "dense", True), Wgrad(257, 16, 32, "split", "off1", False),
    # (16, 64): a 13-column bottom tower's 64-unit layer; a last CTA of exactly one 32-row chunk (288 = 256 + 32)
    Wgrad(31, 13, 64, "odd", "vec", True), Wgrad(288, 16, 33, "split", "odd", True),
    # (16, 128): nz = 3 (N > 256), 17 CTAs with a ragged last one
    Wgrad(33, 16, 65, "off1", "dense", False), Wgrad(4099, 13, 300, "split", "vec", True),
    # (64, 32): dZ cut from a (M, d + u) buffer at column d (odd stride, 4-byte aligned base)
    Wgrad(32, 17, 8, "dense", "cat", True), Wgrad(256, 64, 32, "split", "dense", False),
    Wgrad(256, 64, 64, "vec", "off1", True), Wgrad(33, 17, 33, "split", "cat", True),
    Wgrad(257, 33, 129, "off1", "vec", False), Wgrad(1, 64, 128, "split", "odd", True),
    # (128, 32): the DCN wide head (split X, db None, H = 1: scalar dZ loads at row stride 1), ky = 10, 26 CTAs of 352
    # rows (11 chunks) with a ragged last one
    Wgrad(9000, 1165, 1, "split", "dense", False), Wgrad(31, 65, 32, "vec", "cat", True),
    Wgrad(33, 128, 33, "odd", "off1", True), Wgrad(257, 129, 64, "split", "vec", False),
    # (128, 128): ky = 4 and nz = 3; the parallel DCN body's last deep layer (u = 128 cut from the head's input
    # gradient) over 79 CTAs, the last one a single chunk
    Wgrad(32, 415, 300, "vec", "odd", True), Wgrad(20000, 129, 128, "split", "cat", True),
]
WGRAD += [Wgrad(M, K, N, x, "dense", True) for K, N in TRAINER_PAIRS for M in TRAINER_MS for x in ("pad", "split")]


def _dgrad_core():
    """One case per (KSTEPS, z_vec2, store path, mask), spread over N, K and M."""
    ns = {2: (1, 8, 17, 32), 4: (33, 64), 8: (65, 127, 128)}
    ks = (1, 3, 13, 64, 65, 128, 129, 415, 1165)
    ms = (1, 15, 16, 17, 100, 1001)
    # dX (and mask) layouts per store path: the mask's stride differs from dX's in every masked case, and the mask
    # alone gates the path in some
    stores = {("vec4", False): (("vec", None), ("dense4", None)), ("vec4", True): (("vec", "wide"), ("wide", "vec")),
              ("vec2", False): (("even", None), ("even", None)), ("vec2", True): (("even", "vec"), ("vec", "even")),
              ("scalar", False): (("odd", None), ("off1", None)), ("scalar", True): (("vec", "odd"), ("off1", "wide"))}
    out, i = [], 0
    for kst in (2, 4, 8):
        for zv in (True, False):
            for store in ("vec4", "vec2", "scalar"):
                for masked in (False, True):
                    N = ns[kst][i % len(ns[kst])]
                    K = ks[i % len(ks)]
                    dz = (("vec", "even") if zv else ("odd", "off1", "cat"))[i % (2 if zv else 3)]
                    dx, mask = stores[(store, masked)][i % 2]
                    if dx == "dense4":
                        dx = "dense" if K % 4 == 0 else "vec"
                    out.append(Dgrad(ms[i % len(ms)], K, N, dz, dx, mask))
                    i += 1
    return out


# two or more grid-stride laps: 2 500 tiles over 264 CTAs (ky = 1); 257 tiles over 26 CTAs (ky = 10) with the wide
# head's layout (dZ cut from the head's input gradient, dX at the odd stride d + u)
DGRAD_LAPS = [Dgrad(40000, 128, 128, "vec", "vec", "wide"), Dgrad(4099, 1165, 65, "cat", "dense", None)]
DGRAD = _dgrad_core() + DGRAD_LAPS
DGRAD += [Dgrad(M, K, N, "dense", "pad", mask) for K, N in TRAINER_PAIRS for M in TRAINER_MS for mask in (None, "pad")]

# the DCN wide head: H heads on the (M, d + 128) [cross | deep] input, masked (the stacked body's relu output) or not
WIDE_HEAD = [(1, True), (3, False), (8, True)]
WIDE_M = 4099


def _offset(layout, C):
    return layout_of(layout, C)[0]


def case_wgrad_plan(c, sms=SMS):
    xc, xs = layout_of(c.x, c.K) if c.x != "split" else (0, 0)
    zc, zs = layout_of(c.dz, c.N)
    return wgrad_plan(c.M, c.K, c.N, "split" if c.x == "split" else "f32", xs, xc, zs, zc, sms)


def case_dgrad_plan(c, sms=SMS):
    zc, zs = layout_of(c.dz, c.N)
    xc, xs = layout_of(c.dx, c.K)
    mc, ms = layout_of(c.mask, c.K) if c.mask else (None, None)
    return dgrad_plan(c.M, c.K, c.N, zs, zc, xs, xc, ms, mc, sms)


def wgrad_id(c):
    return f"M{c.M}-K{c.K}-N{c.N}-x_{c.x}-dz_{c.dz}-{'db' if c.db else 'nodb'}"


def dgrad_id(c):
    return f"M{c.M}-K{c.K}-N{c.N}-dz_{c.dz}-dx_{c.dx}-{'mask_' + c.mask if c.mask else 'nomask'}"


# ---------------------------------------------------------------------------------------------------------------
# data and bounds (CPU or device, float64)
# ---------------------------------------------------------------------------------------------------------------
def _block(M):
    """The 32-row block scaled by 40."""
    a = (M // 2) // 32 * 32
    return slice(a, a + 32)


def wgrad_data(M, K, N, seed):
    """fp32 X (M, K) relu-like (exact zeros, every 7th row zero, one block x40), dZ (M, N) of both signs (every 11th
    row zero), and non-zero starting values dw0 (K, N), db0 (N,): CPU tensors from a seeded generator."""
    g = torch.Generator().manual_seed(seed)
    X = torch.randn((M, K), generator=g).clamp_min(0.0)
    dZ = torch.randn((M, N), generator=g)
    r = torch.arange(M)
    X[r % 7 == 3] = 0.0
    dZ[r % 11 == 5] = 0.0
    X[_block(M)] *= 40.0
    dw0 = torch.randn((K, N), generator=g) * 0.5
    db0 = torch.randn(N, generator=g) * 0.5
    return X, dZ, dw0, db0


def dgrad_data(M, K, N, seed):
    """dZ (M, N) of both signs (every 11th row zero, one block x40), the Keras kernel W (K, N) / sqrt(N) and the relu-like
    mask (M, K) (exact zeros, every 7th row zero): CPU tensors from a seeded generator."""
    g = torch.Generator().manual_seed(seed)
    dZ = torch.randn((M, N), generator=g)
    W = torch.randn((K, N), generator=g) / N ** 0.5
    mask = torch.randn((M, K), generator=g).clamp_min(0.0)
    r = torch.arange(M)
    dZ[r % 11 == 5] = 0.0
    dZ[_block(M)] *= 40.0
    mask[r % 7 == 3] = 0.0
    return dZ, W, mask


def wgrad_ref(X, dZ, dw0, db0):
    Xd, Zd = X.double(), dZ.double()
    return dw0.double() + Xd.t() @ Zd, db0.double() + Zd.sum(0)


def wgrad_bounds(X, dZ, dw0, db0, rows, gx):
    """The dW and db bounds of the module docstring."""
    xa, za = X.double().abs(), dZ.double().abs()
    bw = 2 * (UNIT + (3 * rows / 16 + gx) * E) * (xa.t() @ za) + gx * E * dw0.double().abs()
    bb = 2 * (rows + 256 + gx) * E * za.sum(0) + gx * E * db0.double().abs()
    return bw, bb


def dgrad_ref(dZ, W, mask):
    ref = dZ.double() @ W.double().t()
    return ref if mask is None else ref * (mask > 0)


def dgrad_bound(dZ, W, mask):
    N = dZ.shape[1]
    b = 2 * (UNIT + N * E) * (dZ.double().abs() @ W.double().abs().t())
    return b if mask is None else b * (mask > 0)


# ---------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------
def _buffer(M, C, layout, device):
    """(NaN buffer with GUARD rows past M, (M, C) view in the layout, first column)."""
    c, stride = layout_of(layout, C)
    buf = _nan((M + GUARD, stride), device)
    return buf, buf[:M, c:c + C], c


def _operand(t, layout, device):
    buf, view, _ = _buffer(t.shape[0], t.shape[1], layout, device)
    view.copy_(t.to(device))
    return view


def _offset_of(t):
    """t's first element in floats past a 16-byte boundary."""
    return (t.data_ptr() // 4) % 4


def _untouched(buf, M, c, C, what):
    """Nothing of the NaN buffer outside its (M, C) view at column c was written."""
    assert bool(torch.isnan(buf[M:]).all()), f"{what}: a guard row past M was written"
    assert bool(torch.isnan(buf[:, :c]).all()) and bool(torch.isnan(buf[:, c + C:]).all()), f"{what}: a guard column was written"


def _accumulator(t0, device):
    """(buffer, view): t0's values at the head of a NaN buffer with TAIL more floats."""
    buf = _nan((t0.numel() + TAIL,), device)
    view = buf[:t0.numel()].view(t0.shape)
    view.copy_(t0.to(device))
    return buf, view


# ---------------------------------------------------------------------------------------------------------------
# 1. wgrad: every (tile, XSPLIT) instantiation, both load paths of X and dZ, db given and None
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", WGRAD, ids=wgrad_id)
def test_wgrad_matches_float64(device, c):
    X, dZ, dw0, db0 = wgrad_data(c.M, c.K, c.N, WGRAD.index(c))
    sms = _sms(device)
    dz = _operand(dZ, c.dz, device)
    if c.x == "split":
        x = ops.split_rows(X.to(device))
        p = wgrad_plan(c.M, c.K, c.N, "split", 0, 0, dz.stride(0), _offset_of(dz), sms)
    else:
        x = _operand(X, c.x, device)
        p = wgrad_plan(c.M, c.K, c.N, "f32", x.stride(0), _offset_of(x), dz.stride(0), _offset_of(dz), sms)
    assert p == case_wgrad_plan(c, sms), f"premise: the operands' layout gives {p}"
    wbuf, dw = _accumulator(dw0, device)
    bbuf, db = _accumulator(db0, device) if c.db else (None, None)
    if c.x == "split":
        ops.dense_wgrad_split(x, c.K, dz, dw, db)
    else:
        ops.dense_wgrad(x, dz, dw, db)
    Xd, Zd = X.to(device), dZ.to(device)
    rw, rb = wgrad_ref(Xd, Zd, dw0.to(device), db0.to(device))
    bw, bb = wgrad_bounds(Xd, Zd, dw0.to(device), db0.to(device), p["rows_per_cta"], p["gx"])
    _within(dw, rw, bw, f"dW ({p['tile']}, split {p['xsplit']})")
    assert bool(torch.isnan(wbuf[dw.numel():]).all()), "dW: a float past the (K, N) matrix was written"
    if c.db:
        _within(db, rb, bb, "db")
        assert bool(torch.isnan(bbuf[c.N:]).all()), "db: a float past N was written"


# ---------------------------------------------------------------------------------------------------------------
# 2. dgrad: every (KSTEPS, dZ load, store, mask) combination
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", DGRAD, ids=dgrad_id)
def test_dgrad_matches_float64(device, c):
    dZ, W, Mk = dgrad_data(c.M, c.K, c.N, 5000 + DGRAD.index(c))
    sms = _sms(device)
    dz = _operand(dZ, c.dz, device)
    Wd = W.to(device)
    mask = _operand(Mk, c.mask, device) if c.mask else None
    buf, dx, col = _buffer(c.M, c.K, c.dx, device)
    p = dgrad_plan(c.M, c.K, c.N, dz.stride(0), _offset_of(dz), dx.stride(0), _offset_of(dx),
                   None if mask is None else mask.stride(0), None if mask is None else _offset_of(mask), sms)
    assert p == case_dgrad_plan(c, sms), f"premise: the operands' layout gives {p}"
    if c in DGRAD_LAPS:
        assert p["laps"] >= 2, f"premise: M = {c.M}, K = {c.K} gives {p['laps']} lap(s)"
    ops.dense_dgrad(dz, Wd, dx, mask=mask)
    Zd, Md = dZ.to(device), None if mask is None else Mk.to(device)
    _within(dx, dgrad_ref(Zd, Wd, Md), dgrad_bound(Zd, Wd, Md), f"dX ({p['ksteps']} k-steps, {p['store']} stores)")
    _untouched(buf, c.M, col, c.K, "dX")
    # no atomics: a repeat gives the same bits, and so does a 16-row-aligned window launched alone
    buf2, dx2, _ = _buffer(c.M, c.K, c.dx, device)
    ops.dense_dgrad(dz, Wd, dx2, mask=mask)
    assert torch.equal(dx2, dx), "dX: a repeat differs"
    if c.M >= 32:
        lo = (c.M // 2) // 16 * 16
        wbuf, wdx, wcol = _buffer(c.M - lo, c.K, c.dx, device)
        ops.dense_dgrad(dz[lo:], Wd, wdx, mask=None if mask is None else mask[lo:])
        assert torch.equal(wdx, dx[lo:]), f"dX: rows [{lo}, {c.M}) launched alone differ"
        _untouched(wbuf, c.M - lo, wcol, c.K, "dX (window)")


# ---------------------------------------------------------------------------------------------------------------
# 3. the DCN wide head as the trainer composes it
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,masked", WIDE_HEAD, ids=lambda v: str(v))
def test_wide_head_composition_matches_float64(device, H, masked):
    """The output heads on a (M, d + 128) head input, d = 1037, as the DCN trainer runs them when that input is wider
    than mm_heads_fwd_bwd's 256: logits x W from dense_tc, the loss kernel on them with an identity kernel (dz out, db
    accumulated), dW from dense_wgrad_split on x's split operand (db None) and dX from dense_dgrad on dz, into a
    NaN-guarded (M, d + 128) buffer at its odd row stride; dX masked by x > 0 (a stacked body's relu output) or not.
    Against float64 autograd of the same heads.  Bounds: z within ez = (UNIT + K E) (|x| |W|) + E |z| (dense_tc, then
    the bias added in fp32; the identity kernel's products and sums are exact); dz = lambda l'(z) / M moves by
    1/4 (BCE) or 2 (MSE) of that, plus 8 E (|l'| + 1) lambda / M of its own rounding (test_gpu_heads_kernels); dW, dX
    add that error through |x| and |W| to their own bounds above; db is a sum of M such dz in some order,
    within sum edz + M E sum |dz|."""
    M, K = WIDE_M, D_CAT + 128
    g = torch.Generator().manual_seed(H)
    xh = torch.randn((M, K), generator=g).clamp_min(0.0)
    xh[_block(M)] *= 40.0
    xh[torch.arange(M) % 7 == 3] = 0.0
    Wh = torch.randn((K, H), generator=g) / K ** 0.5
    losses = ["binary_crossentropy" if h % 3 != 1 else "mse" for h in range(H)]
    ys = [(torch.rand(M, generator=g) < 0.4).float() if l == "binary_crossentropy" else torch.randn(M, generator=g)
          for l in losses]
    lws = [1.0 + 0.25 * h for h in range(H)]
    x, W = xh.to(device), Wh.to(device)
    b = torch.tensor([0.3 * (h + 1) * (-1) ** h for h in range(H)], device=device)
    ys = [y.to(device) for y in ys]

    xs = ops.split_rows(x)
    z = torch.empty((M, H), device=device)
    ops.dense_tc(xs, K, ops.split_weights(W), H, None, "linear", out_f32=z)
    logits = torch.empty((H, M), device=device)
    loss = torch.zeros(1 + H, device=device)
    dz = torch.empty((M, H), device=device)
    db = torch.zeros(H, device=device)
    ops.heads_fwd_bwd(z, torch.eye(H, device=device), b, losses, ys, logits, loss, dz, None, db, loss_weights=lws,
                      mask_relu=False)
    wbuf, dW = _accumulator(torch.zeros((K, H)), device)
    sms = _sms(device)
    p = wgrad_plan(M, K, H, "split", 0, 0, H, 0, sms)
    assert p["tile"] == (128, 32) and p["xsplit"] and p["z_vec"] == int(H % 4 == 0)
    ops.dense_wgrad_split(xs, K, dz, dW, None)
    buf, dx, _ = _buffer(M, K, "dense", device)
    q = dgrad_plan(M, K, H, H, 0, K, 0, K if masked else None, 0 if masked else None, sms)
    assert q["store"] == "scalar" and q["z_vec2"] == int(H % 2 == 0)
    ops.dense_dgrad(dz, W, dx, mask=x if masked else None)

    xd = x.double().requires_grad_(True)
    Wd = W.double().requires_grad_(True)
    bd = b.double().requires_grad_(True)
    zr = xd @ Wd + bd
    total = 0.0
    for h, l in enumerate(losses):
        y = ys[h].double()
        lh = (torch.nn.functional.binary_cross_entropy_with_logits(zr[:, h], y) if l == "binary_crossentropy"
              else ((zr[:, h] - y) ** 2).mean())
        total = total + lws[h] * lh
    total.backward()
    zr = zr.detach()
    ax, aw = x.double().abs(), W.double().abs()
    ez = (UNIT + K * E) * (ax @ aw) + E * zr.abs()
    edz, adz = [], []
    for h, l in enumerate(losses):
        y = ys[h].double()
        gt, cz = (torch.sigmoid(zr[:, h]) - y, 0.25) if l == "binary_crossentropy" else (2 * (zr[:, h] - y), 2.0)
        edz.append(lws[h] / M * (cz * ez[:, h] + 8 * E * (gt.abs() + 1)))
        adz.append((lws[h] / M * gt).abs())
    edz, adz = torch.stack(edz, 1), torch.stack(adz, 1)  # (M, H)
    bw = ax.t() @ edz + 2 * (UNIT + (3 * p["rows_per_cta"] / 16 + p["gx"]) * E) * (ax.t() @ adz)
    _within(dW, Wd.grad, bw, f"dW ({H} heads)")
    assert bool(torch.isnan(wbuf[K * H:]).all()), "dW: a float past the (K, H) matrix was written"
    want = xd.grad * (x > 0) if masked else xd.grad
    bx = edz @ aw.t() + 2 * (UNIT + H * E) * (adz @ aw.t())
    _within(dx, want, bx * (x > 0) if masked else bx, f"dX ({H} heads, mask {masked})")
    _untouched(buf, M, 0, K, "dX")
    _within(db, bd.grad, edz.sum(0) + M * E * adz.sum(0), f"db ({H} heads)")
