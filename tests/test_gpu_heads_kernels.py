"""The output heads at every instantiation they dispatch: mm_heads_fwd_bwd (the loss, dx, dW and db of every DLRM and DCN
step, and the forward of multi-output models whose last layer is wider than 32) and mm_mlp_tc_heads (the whole top tower
with its heads fused into the epilogue) at every head count.

mm_heads_fwd_bwd is compiled for H = 1..8 heads x {the scalar head_kernel (one warp per row), head_kernel_v4 with a lane
group of G = 2, 4, 8, 16 or 32 (32 / G rows per warp)} x {training, forward only}: 96 kernels.  heads_variant restates the
run-time choice; CASES reaches every (H, variant, training) triple (tests/test_multitask_host.py checks that and prints
the table).  Each case fixes K (partly live lane groups: K = 4, 12, 20, 36, 68, 100) and the layouts:
    x   "dense" (M, K) | "slice" columns 4..4+K of a wider row (ldx > K, aligned) | "off1" columns 1..1+K (misaligned:
        the scalar kernel);
    dx  "dense" | "strided" columns 4..4+K with guard columns | "off1" columns 1..1+K (misaligned: scalar training);
    w   "dense" | "off1" one float past an aligned address (the scalar kernel for H = 1, no effect for H > 1).
Every buffer carries NaN outside the operand (columns beside a slice, 32 rows past M); output guards must stay NaN.
M runs over 1, rows per warp +- 1, 1 001 and a value with three grid-stride laps whose last lap is ragged (asserted from
run_heads' grid formula and the device's SM count).  x holds exact zeros (the relu mask is strict x > 0); about one row
in eight is scaled so that its logits reach +-20..60 (saturated BCE); BCE targets are hard (int) or soft (float), MSE
targets sit around 40 (residuals far from 0); every target dtype, shared and per-head sample weights with zeros, unequal
loss weights, and non-zero starting values in loss, dW and db, which the kernel accumulates into.

Bounds are per element, in float64, from the fp32 arithmetic (EPS = 2^-24):
  * z = x . w_h + b_h is a sum of K + 1 fp32 terms in some order: |err| <= C_DOT (K + 2) EPS sum |x w| + EPS |b|, C_DOT = 1;
  * dz = lambda sw l'(z) / M moves by at most 1/4 (BCE) or 2 (MSE) of z's error, plus the target's rounding to fp32 and
    8 EPS (|l'| + 1) for expf, the sigmoid and the products;
  * dx = sum_h dz_h w_h is within sum_h (err dz_h + (H + 1) EPS |dz_h|) |w_h|, and exactly 0 where the mask is 0;
  * dW, db and the losses are sums over the batch: one lane's laps, the warp's row groups, the CTA's 8 warps and one
    atomic per CTA onto the starting value, a chain of `chain` additions: err <= propagated + chain EPS (sum |terms| +
    |start|)."""
import ctypes as C

import pytest
import torch

from models_b200 import _cabi, ops
from tests.multitask_oracle import BCE, MSE, heads_ref
from tests.test_gpu_forward_scale import _chain
from tests.test_gpu_train_scale import GUARD, RAGGED, _nan, _sms, _within

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -24
C_DOT = 1.0  # the constant of the dot-product bound
WARPS = 8  # warps per CTA (256 threads)
ROW_GUARD = 32  # NaN rows past M in x and dx
VARIANTS = ("scalar", "G2", "G4", "G8", "G16", "G32")
LAYOUT = {"dense": 0, "slice": 4, "strided": 4, "off1": 1}  # first column of the operand in its row (floats)


def heads_variant(H, K, ldx, x_addr, w_addr, lddx=None, dx_addr=None):
    """The kernel mm_heads_fwd_bwd launches: "scalar" (head_kernel) or "G<g>" (head_kernel_v4<g, H, TRAIN>).  Restates
    run_heads (models_b200/csrc/train_dense.cu:314-323: the float4 path needs K % 4 == 0, K <= 128, 16-byte aligned
    rows of x and dx, and for one head an aligned kernel) and launch_heads<H, TRAIN> (train_dense.cu:285-297: G from
    K / 4).  dx_addr None: forward only, where the kernel gets no dx."""
    vec = (K % 4 == 0 and K <= 128 and ldx % 4 == 0 and x_addr % 16 == 0 and (H > 1 or w_addr % 16 == 0)
           and (dx_addr is None or (lddx % 4 == 0 and dx_addr % 16 == 0)))
    if not vec:
        return "scalar"
    g = K // 4
    return "G2" if g <= 2 else "G4" if g <= 4 else "G8" if g <= 8 else "G16" if g <= 16 else "G32"


def _ld(K, layout):
    """Row stride of an operand of K columns in the given layout."""
    return K if layout == "dense" else ((K + 3) // 4) * 4 + 8


def case_variants(case):
    """(training variant, forward variant) of a case, from its layouts (allocations are 16-byte aligned)."""
    H, K, xl, dxl, wl = case
    x, w = 4 * LAYOUT[xl], 4 * LAYOUT[wl]
    return (heads_variant(H, K, _ld(K, xl), x, w, _ld(K, dxl), 4 * LAYOUT[dxl]), heads_variant(H, K, _ld(K, xl), x, w))


# (H, K, x layout, dx layout, w layout): one row per (H, variant), then two cases whose misaligned dx alone sends the
# training step to the scalar kernel (their forward runs G8 / G32)
CASES = [
    (1, 64, "dense", "dense", "off1"), (2, 1, "slice", "strided", "dense"), (3, 7, "dense", "strided", "off1"),
    (4, 130, "slice", "dense", "dense"), (5, 256, "dense", "strided", "dense"), (6, 32, "off1", "strided", "dense"),
    (7, 12, "off1", "dense", "off1"), (8, 256, "slice", "strided", "off1"),
    (1, 4, "slice", "strided", "dense"), (2, 8, "dense", "dense", "off1"), (3, 4, "dense", "strided", "dense"),
    (4, 8, "slice", "dense", "dense"), (5, 4, "slice", "strided", "off1"), (6, 8, "dense", "strided", "dense"),
    (7, 4, "dense", "dense", "dense"), (8, 8, "slice", "strided", "off1"),
    (1, 16, "dense", "strided", "dense"), (2, 12, "slice", "dense", "dense"), (3, 16, "slice", "strided", "off1"),
    (4, 12, "dense", "strided", "off1"), (5, 16, "dense", "dense", "dense"), (6, 12, "slice", "strided", "dense"),
    (7, 16, "slice", "dense", "off1"), (8, 12, "dense", "strided", "dense"),
    (1, 32, "slice", "dense", "dense"), (2, 20, "dense", "strided", "dense"), (3, 20, "slice", "dense", "off1"),
    (4, 32, "dense", "strided", "dense"), (5, 20, "slice", "strided", "dense"), (6, 32, "slice", "dense", "off1"),
    (7, 20, "dense", "strided", "dense"), (8, 32, "dense", "dense", "dense"),
    (1, 64, "slice", "strided", "dense"), (2, 36, "dense", "dense", "dense"), (3, 64, "slice", "strided", "dense"),
    (4, 36, "slice", "dense", "off1"), (5, 64, "dense", "strided", "off1"), (6, 36, "dense", "strided", "dense"),
    (7, 64, "slice", "dense", "dense"), (8, 36, "slice", "strided", "dense"),
    (1, 100, "dense", "strided", "dense"), (2, 128, "slice", "dense", "dense"), (3, 68, "dense", "strided", "dense"),
    (4, 100, "slice", "strided", "off1"), (5, 128, "dense", "dense", "dense"), (6, 68, "slice", "strided", "dense"),
    (7, 100, "dense", "strided", "off1"), (8, 128, "slice", "strided", "dense"),
    (3, 32, "dense", "off1", "dense"), (8, 100, "slice", "off1", "dense"),
]


def _rpw(variant):
    """Rows a warp takes per iteration."""
    return 1 if variant == "scalar" else 32 // int(variant[1:])


def _rows(variant):
    """1, rows per warp +- 1, a ragged size and one of three laps (9 002 row groups over the 4 224 warps of 132 SMs; the
    last group holds one row)."""
    r = _rpw(variant)
    return sorted({1, r - 1, r + 1, 1001, 9001 * r + 1} - {0})


PARAMS = [pytest.param(c, M, id="H{}-K{}-x{}-dx{}-w{}".format(*c) + f"-M{M}") for c in CASES for M in _rows(case_variants(c)[0])]


def _grid(M, variant, sms, multi):
    """(CTAs, laps) of run_heads' grid: blocks = min(ceil(M / 8), 4 SMs), 8 warps each, grid-stride over row groups."""
    ctas = min(-(-M // 8), 4 * sms)
    warps = WARPS * ctas
    groups = -(-M // _rpw(variant))
    laps = -(-groups // warps)
    if multi:
        assert laps >= 2 and groups % warps, f"premise: M = {M} gives {laps} lap(s) of {warps} warps, not ragged"
    return ctas, laps


def _operand(M, K, layout, device):
    """(buffer, view): a NaN-filled (M + ROW_GUARD, ld) buffer and its (M, K) operand in the given layout."""
    buf = _nan((M + ROW_GUARD, _ld(K, layout)), device)
    c = LAYOUT[layout]
    return buf, buf[:M, c:c + K]


def _inputs(case, M, device, seed):
    H, K, xl, _, wl = case
    i = CASES.index(case)
    g = torch.Generator(device=device).manual_seed(seed)
    X, x = _operand(M, K, xl, device)
    v = torch.randn((M, K), generator=g, device=device)
    v[torch.rand((M, K), generator=g, device=device) < 0.25] = 0.0  # exact zeros at the strict relu mask
    Wb = torch.empty(K * H + 4, device=device)
    W = Wb[LAYOUT[wl]:LAYOUT[wl] + K * H].view(K, H)
    W.copy_(torch.randn((K, H), generator=g, device=device) / K ** 0.5)
    b = torch.tensor([0.3 * (h + 1) * (-1) ** h for h in range(H)], device=device)
    # about one row in eight scaled so that its largest |x . w_h| is 20..60: saturated sigmoids
    big = torch.rand(M, generator=g, device=device) < 0.125
    zmax = (v.double() @ W.double()).abs().amax(1)
    f = (20 + 40 * torch.rand(M, generator=g, device=device).double()) / (zmax + 1e-3)
    v = torch.where(big[:, None], v * f.clamp(1.0, 1e3)[:, None].float(), v)
    x.copy_(v)
    losses = [BCE if (h + i) % 3 != 1 else MSE for h in range(H)]
    dts = (torch.int32, torch.int64, torch.float32, torch.float64)
    ys = []
    for h, l in enumerate(losses):
        dt = dts[(h + i) % 4]
        if l == BCE:
            y = (torch.rand(M, generator=g, device=device) < 0.4).double() if not dt.is_floating_point else \
                torch.rand(M, generator=g, device=device).double()  # soft targets
        else:
            y = 40 + 10 * torch.randn(M, generator=g, device=device).double()
            y = y.round() if not dt.is_floating_point else y
        ys.append(y.to(dt))

    def weights():
        s = torch.rand(M, generator=g, device=device) * 2
        return torch.where(torch.rand(M, generator=g, device=device) < 0.2, torch.zeros_like(s), s)

    form = (i + M) % 3
    sw = None if form == 0 else weights() if form == 1 else [None if h % 3 == 1 else weights() for h in range(H)]
    lws = [0.5 + 0.375 * h for h in range(H)]
    return X, x, W, b, losses, ys, sw, lws


@pytest.mark.parametrize("case,M", PARAMS)
def test_heads_every_instantiation_matches_float64(device, case, M):
    """Training (logits, [total, loss_h], dx, dW, db accumulated onto non-zero starting values) and then the forward
    alone (the activated predictions; gradient buffers handed to the C entry keep their bits), per element against
    float64 within the bounds of the module docstring."""
    H, K, xl, dxl, wl = case
    train_v, fwd_v = case_variants(case)
    ctas, laps = _grid(M, train_v, _sms(device), M > 1001)
    chain = laps + 5 + WARPS + ctas + 2
    X, x, W, b, losses, ys, sw, lws = _inputs(case, M, device, 11 * CASES.index(case) + M)
    mask = CASES.index(case) % 3 != 2
    sws = sw if isinstance(sw, list) else [sw] * H
    D, dx = _operand(M, K, dxl, device)
    assert heads_variant(H, K, x.stride(0), x.data_ptr(), W.data_ptr(), dx.stride(0), dx.data_ptr()) == train_v
    assert heads_variant(H, K, x.stride(0), x.data_ptr(), W.data_ptr()) == fwd_v
    g = torch.Generator(device=device).manual_seed(M)
    loss0 = torch.randn(1 + H, generator=g, device=device)
    dW0 = torch.randn((K, H), generator=g, device=device) * 0.1
    db0 = torch.randn(H, generator=g, device=device) * 0.1
    loss, dW, db = loss0.clone(), dW0.clone(), db0.clone()
    Z = _nan((H * M + GUARD,), device)
    z = Z[:H * M].view(H, M)
    ops.heads_fwd_bwd(x, W, b, losses, ys, z, loss, dx, dW, db, loss_weights=lws, mask_relu=mask, sample_weight=sw)
    torch.cuda.synchronize()
    tot, per, zr, rdx, rdW, rdb = heads_ref(x, W, b, losses, ys, sws, lws, mask)

    ax, aw = x.double().abs(), W.double().abs()
    ez = (C_DOT * (K + 2) * EPS * (ax @ aw) + EPS * b.double().abs()).t()  # (H, M)
    _within(z, zr, ez, "logits")
    assert bool(torch.isnan(Z[H * M:]).all()), "a logit past H M was written"
    edz, adz, lb = [], [], []
    for h, l in enumerate(losses):
        zh, y = zr[h], ys[h].double()
        s = sws[h].double() if sws[h] is not None else torch.ones_like(zh)
        if l == BCE:
            lt, gt, cz = zh.clamp_min(0) - zh * y + torch.log1p(torch.exp(-zh.abs())), torch.sigmoid(zh) - y, 0.25
        else:
            lt, gt, cz = (zh - y) ** 2, 2 * (zh - y), 2.0
        edz.append(s * lws[h] / M * (cz * ez[h] + 2 * EPS * y.abs() + 8 * EPS * (gt.abs() + 1)))
        adz.append((gt * s * lws[h] / M).abs())
        sl = float((s * lt.abs()).sum()) / M
        lb.append(float((s / M * (gt.abs() * (ez[h] + EPS * y.abs()) + 4 * EPS * (lt.abs() + zh.abs() + 1))).sum())
                  + chain * EPS * (sl + abs(float(loss0[1 + h]))))
    edz, adz = torch.stack(edz), torch.stack(adz)  # (H, M)
    t64 = dict(dtype=torch.float64, device=device)
    _within(loss[1:], per + loss0[1:].double(), torch.tensor(lb, **t64), "per-head losses")
    tb = sum(lw * e for lw, e in zip(lws, lb)) + H * chain * EPS * (sum(lw * float(p.abs()) for lw, p in zip(lws, per))
                                                                      + abs(float(loss0[0])))
    _within(loss[:1], tot.reshape(1) + loss0[:1].double(), torch.tensor([tb], **t64), "total loss")
    bdx = (edz + (H + 1) * EPS * adz).t() @ aw.t()  # (M, K)
    if mask:
        bdx = bdx * (x > 0)  # exactly 0 where the mask is
    _within(dx, rdx, bdx, "dx")
    assert bool(torch.isnan(D[M:]).all()), "dx: a guard row past M was written"
    c = LAYOUT[dxl]
    assert bool(torch.isnan(D[:, :c]).all()) and bool(torch.isnan(D[:, c + K:]).all()), "dx: a guard column was written"
    _within(dW, rdW + dW0.double(), ax.t() @ edz.t() + chain * EPS * (ax.t() @ adz.t() + dW0.double().abs()), "dW")
    _within(db, rdb + db0.double(), edz.sum(1) + chain * EPS * (adz.sum(1) + db0.double().abs()), "db")

    # forward only, through the C entry with the gradient buffers given: they must keep their bits
    kept = [t.clone() for t in (loss, D, dW, db)]
    P = _nan((H * M + GUARD,), device)
    pred = P[:H * M].view(H, M)
    kinds = (C.c_int * H)(*[_cabi.LOSS_KINDS[l] for l in losses])
    _cabi.check(_cabi.load().mm_heads_fwd_bwd(x.data_ptr(), M, K, x.stride(0), H, W.data_ptr(), b.data_ptr(), kinds, None, None,
                                              None, None, pred.data_ptr(), loss.data_ptr(), dx.data_ptr(), dx.stride(0), 1,
                                              dW.data_ptr(), db.data_ptr(), torch.cuda.current_stream().cuda_stream),
                "mm_heads_fwd_bwd")
    torch.cuda.synchronize()
    for t, k, what in zip((loss, D, dW, db), kept, ("loss", "dx", "dW", "db")):
        assert torch.equal(t.view(torch.int32), k.view(torch.int32)), f"forward only wrote {what}"
    assert bool(torch.isnan(P[H * M:]).all()), "a prediction past H M was written"
    for h, l in enumerate(losses):
        if l == BCE:
            sig = torch.sigmoid(zr[h])
            _within(pred[h], sig, ez[h] / 4 + 8 * EPS * sig, f"prediction {h} (sigmoid)")
        else:
            _within(pred[h], zr[h], ez[h], f"prediction {h} (linear)")


# ---------------------------------------------------------------------------------------------------------------
# mm_mlp_tc_heads
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("width", [8, 16, 24, 32])
@pytest.mark.parametrize("H", range(1, 9))
def test_mlp_tc_heads_every_head_count(device, H, width):
    """The tower [64, width] relu on K = 100 inputs with H fused heads, sigmoid and linear mixed, each with its own
    non-zero bias, at M = 1, 63, 65 and 65 573 (several 128-row tiles per CTA, the last one ragged).  Per element within
    test_gpu_forward_scale's _chain bound (split-bf16 layers, then the head as one more layer); the (H, M) output is the
    head of a NaN buffer whose guard past H M must stay NaN."""
    K, widths = 100, [64, width]
    g = torch.Generator(device=device).manual_seed(100 * H + width)
    Ws = [torch.randn((k, n), generator=g, device=device) / k ** 0.5 for k, n in zip([K] + widths[:-1], widths)]
    bs = [torch.randn(n, generator=g, device=device) * 0.1 for n in widths]
    Hw = torch.randn((width, H), generator=g, device=device) / width ** 0.5
    Hb = torch.tensor([0.3 * (h + 1) * (-1) ** h for h in range(H)], device=device)
    acts = ["sigmoid" if (h + width // 8) % 2 == 0 else "linear" for h in range(H)]
    ws = [ops.split_weights(w) for w in Ws]
    tower = list(zip(Ws, bs, ["relu", "relu"]))
    for M in (1, 63, 65, RAGGED):
        x = torch.randn((M, K), generator=g, device=device)
        Ob = _nan((H * M + GUARD,), device)
        out = Ob[:H * M].view(H, M)
        ops.mlp_tc_heads(ops.split_rows(x), K, ws, widths, bs, ["relu", "relu"], Hw, Hb, acts, out)
        torch.cuda.synchronize()
        assert bool(torch.isnan(Ob[H * M:]).all()), f"M = {M}: an output past H M was written"
        h, eh = _chain(x.double(), tower)
        for j, act in enumerate(acts):
            y, ey = _chain(h, [(Hw[:, j:j + 1].contiguous(), Hb[j:j + 1], act)], eh)
            _within(out[j], y[:, 0], ey[:, 0], f"M = {M}: head {j} ({act})")
