"""The DCN-v2 and two-tower training steps, and the pipelined forwards, at the sizes the benchmark runs: B = 65 536 for
DCN-v2 (Criteo, d = 1037, cross depth 3, deep [256, 128]), B = 16 384 for the two-tower model (10 M-row item table,
towers [256, 128]).  At the batches of the per-kernel tests every grid-stride loop here finishes in one lap; each
large-batch test below asserts from the launcher's own grid formula and the device's SM count that the kernel makes at
least two, and also runs a ragged size (B + 37).

References are float64 on the device, in chunks where they would be large.  Bounds are per element and derived from
the arithmetic (conventions of test_gpu_train_scale): a 3-pass split-bf16 product is within U = 2^-16 of |a b|, an fp32
operation rounds by at most E = 2^-24 of its result, an fp32 sum of n terms is within n E of the sum of the absolute
terms.  A lost, repeated or stale lap moves an element by O(1) of its scale, far above those bounds.  Output buffers
carry NaN guard rows past the batch and NaN padding columns; they must stay NaN."""
import gc

import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets, ops
from models_b200._cabi import HYPER_BETA1, HYPER_BETA2
from models_b200.core import Prediction
from models_b200.graph import HostBatch, _view
from models_b200.train import DENSE_PATH_MAX_ROWS
from tests import twotower_train_oracle as O
from tests.test_gpu_forward_scale import _chunks, _dense_tc_laps, _nan_bf16, _split_padding_zero
from tests.test_gpu_train_scale import (BIG, CAP, E, GUARD, RAGGED, U, _ce_ref_chunked, _check_sparse_update, _dgrad_laps, _nan,
                                        _rule, _sms, _untouched, _wgrad_launch, _within)

pytestmark = pytest.mark.gpu
D_DCN = 1037  # the DCN input width of the Criteo schema: 26 tables of inferred widths 8..120 + 13 continuous columns
LD = 1040  # DCNTrainer's row stride for (B, d) buffers
TT = 16384  # the two-tower benchmark batch
COUNTING_SORT_MAX_ROWS = 1024  # tables up to this size take the counting-sort path of the sparse update


def _free():
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _release_memory():
    """The full-size models of one test hold tens of GB: return them to the device before the next test."""
    yield
    _free()


def _filled(B, ld, d, gen, device, scale=1.0):
    """A NaN-filled (B + GUARD, ld) buffer whose (B, d) view holds N(0, scale^2) values; returns (buffer, view)."""
    buf = _nan((B + GUARD, ld), device)
    v = buf[:B, :d]
    v.copy_(torch.randn((B, d), generator=gen, device=device) * scale)
    return buf, v


# ---------------------------------------------------------------------------------------------------------------
# A1. mm_cross_backward at d = 1037
# ---------------------------------------------------------------------------------------------------------------
def _cross_bwd_laps(B, sms):
    """Laps of cross_backward_kernel (mm_cross_backward: 8 rows per CTA, ceil(B / 8) CTAs capped at 16 SMs)."""
    ctas = min(-(-B // 8), 16 * sms)
    return -(-B // (8 * ctas))


@pytest.mark.parametrize("top", [True, False])
@pytest.mark.parametrize("B", [BIG, RAGGED])
def test_cross_backward_at_scale(device, B, top):
    """One cross layer of DCNTrainer's backward at the benchmark's d = 1037, row stride 1040, Kp = tc_padded_k(1037):
    the top layer (p None: g is read only and must stay bit-identical; acc = g z) and a lower layer (g += p in place,
    acc += g z).  Against float64 of the device inputs: g = g0 + p within E |g0 + p| (one rounding); dz = g x0 within
    2 E (|g0| + |p|) |x0| (the rounded g, then the product); acc within 3 E ((|g0| + |p|) |z| + |acc0|) (the rounded g,
    the product and the sum, which the compiler may contract into one FMA).  dz_split equals split_rows(dz) bit for
    bit, and its padding columns [1037, Kp) are zero in both halves.  The NaN padding columns 1037..1039 of the inputs
    are never read and those of the outputs never written."""
    d = D_DCN
    laps = _cross_bwd_laps(B, _sms(device))
    assert laps >= 2, f"premise: B = {B} gives {laps} lap(s)"
    Kp = ops.tc_padded_k(d)
    gen = torch.Generator(device=device).manual_seed(B + top)
    (x0b, x0), (zb, z), (gb, g), (pb, p), (accb, acc) = (_filled(B, LD, d, gen, device) for _ in range(5))
    dzb = _nan((B + GUARD, LD), device)
    dzs = _nan_bf16((B + GUARD, 2 * Kp), device)
    g0, acc0 = g.clone(), acc.clone()
    ops.cross_backward(x0, z, g, None if top else p, acc, top, dzb[:B, :d], dzs[:B])
    if top:
        assert torch.equal(g, g0), "top layer: g changed although no p was given"
    for what, buf in (("g", gb), ("acc", accb), ("dz", dzb)):
        _untouched(buf, B, d, what)
    assert torch.equal(dzs[:B], ops.split_rows(dzb[:B, :d])), "dz_split is not split_rows(dz)"
    _split_padding_zero(dzs, B, d, "dz_split")
    for s, e in _chunks(B):
        gd, pd = g0[s:e].double(), (0.0 if top else p[s:e].double())
        gs, ga = gd + pd, gd.abs() + (0.0 if top else p[s:e].double().abs())
        x0d, zd, a0 = x0[s:e].double(), z[s:e].double(), acc0[s:e].double()
        if not top:
            _within(g[s:e], gs, E * gs.abs(), f"g rows [{s}, {e})")
        _within(dzb[s:e, :d], gs * x0d, 2 * E * ga * x0d.abs(), f"dz rows [{s}, {e})")
        want = gs * zd + (0.0 if top else a0)
        _within(acc[s:e], want, 3 * E * (ga * zd.abs() + (0.0 if top else a0.abs())), f"acc rows [{s}, {e})")


# ---------------------------------------------------------------------------------------------------------------
# A2. mm_cross_combine at (65 536, 1037)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [BIG, RAGGED])
def test_cross_combine_at_scale(device, B):
    """out = x0 z + x (fma3_kernel) over B x 1037 elements, about 126 laps of its 16 SMs x 256 threads: once with every
    operand at DCNTrainer's row stride 1040, once with four different strides (1040, 1044, 1048, 1052) so that an
    operand addressed with another operand's stride is caught.  One fused multiply-add per element: within
    E |x0 z + x| of float64.  NaN padding columns of the inputs are never read, those of the output never written."""
    d = D_DCN
    sms = _sms(device)
    ctas = min(-(-B * d // 256), 16 * sms)
    laps = -(-B * d // (ctas * 256))
    assert laps >= 2, f"premise: B = {B} gives {laps} lap(s)"
    gen = torch.Generator(device=device).manual_seed(B + d)
    x0 = torch.randn((B, d), generator=gen, device=device)
    z = torch.randn((B, d), generator=gen, device=device)
    x = torch.randn((B, d), generator=gen, device=device)
    for strides in ((LD, LD, LD, LD), (LD, LD + 4, LD + 8, LD + 12)):
        bufs = [_nan((B + GUARD, ld), device) for ld in strides]
        for buf, src in zip(bufs[:3], (x0, z, x)):
            buf[:B, :d].copy_(src)
        ops.cross_combine(bufs[0][:B, :d], bufs[1][:B, :d], bufs[2][:B, :d], bufs[3][:B, :d])
        _untouched(bufs[3], B, d, f"out (strides {strides})")
        for s, e in _chunks(B):
            want = x0[s:e].double() * z[s:e].double() + x[s:e].double()
            _within(bufs[3][s:e, :d], want, E * want.abs(), f"out (strides {strides}) rows [{s}, {e})")
        del bufs
        _free()


# ---------------------------------------------------------------------------------------------------------------
# A3. mm_concat_backward with the DCN input layout
# ---------------------------------------------------------------------------------------------------------------
def _dcn_widths():
    """(column offsets, widths, d) of the input block DCNModel infers for the uncapped Criteo schema."""
    model = mm.DCNModel(datasets.criteo_schema(), depth=3, deep_block=mm.MLPBlock([256, 128]))
    return model.body.input_block.layout()


@pytest.mark.parametrize("n_add", [3, 4])
@pytest.mark.parametrize("B", [BIG, RAGGED])
def test_concat_backward_dcn_layout_at_scale(device, B, n_add):
    """The real DCN layout: 26 tables at columns 0..1023 (widths 8..120), 13 continuous columns at 1024..1036, with the
    stacked body's 3 addends (g, p, acc) and the parallel body's 4 (+ the deep branch's input gradient), all at row
    stride 1040.  The kernel starts from 0 and adds the addends in order, so every slice equals torch's fp32
    a0 + a1 + a2 (+ a3) bit for bit.  Every addend holds NaN in the continuous columns: a slice that reads them fails.
    The grid is shared by the slices (sized by the widest): on a 132-SM H100 the width-8 slices take one lap even at
    B = 65 573 (4 SMs x 256 elements per lap) and every width from 16 up takes 2 to 15; the lap count of each width is
    asserted.  Each slice buffer has NaN guard rows and 4 NaN padding columns that must stay NaN."""
    cols, widths, d = _dcn_widths()
    assert d == D_DCN
    tabs = sorted((cols[f], widths[f], f) for f in datasets.CRITEO_MAX)
    conts = sorted(cols[f] for f in widths if f not in datasets.CRITEO_MAX)
    assert [c for c, _, _ in tabs][0] == 0 and tabs[-1][0] + tabs[-1][1] == 1024 and conts == list(range(1024, 1037))
    sms = _sms(device)
    qmax = max(w for _, w, _ in tabs) // 4
    grid = min(-(-B * qmax // 256), 4 * sms)
    laps = {w: -(-B * (w // 4) // (grid * 256)) for _, w, _ in tabs}
    assert max(laps.values()) >= 2, f"premise: laps per slice width {laps}"
    if sms == 132:
        assert laps[8] == 1 and all(n >= 2 for w, n in laps.items() if w >= 16), f"laps per slice width {laps}"
    gen = torch.Generator(device=device).manual_seed(B + n_add)
    adds = []
    for _ in range(n_add):
        _, a = _filled(B, LD, d, gen, device)
        a[:, 1024:] = float("nan")
        adds.append(a)
    dsts = [_nan((B + GUARD, w + 4), device) for _, w, _ in tabs]
    ops.concat_backward(adds, [(dst[:B, :w], c) for dst, (c, w, _) in zip(dsts, tabs)])
    for dst, (c, w, f) in zip(dsts, tabs):
        want = adds[0][:, c:c + w] + adds[1][:, c:c + w]
        for a in adds[2:]:
            want = want + a[:, c:c + w]
        assert torch.equal(dst[:B, :w], want), f"slice of {f} (width {w} at column {c}, {laps[w]} lap(s)) is not a0 + .. + a{n_add - 1}"
        _untouched(dst, B, w, f"slice of {f}")


# ---------------------------------------------------------------------------------------------------------------
# A4. mm_dense_wgrad[_split] and the transposed-kernel dgrad at the DCN and two-tower step shapes
# ---------------------------------------------------------------------------------------------------------------
WGRAD_CASES = [(M, K, N) for K, N in ((D_DCN, D_DCN), (D_DCN, 256), (256, 128)) for M in (BIG, RAGGED)] + \
              [(TT + 37, 192, 256), (TT + 37, 256, 128)]


@pytest.mark.parametrize("M,K,N", WGRAD_CASES)
def test_wgrad_and_dgrad_at_step_shapes(device, M, K, N):
    """The dense layers of the DCN step (cross 1037 -> 1037, deep 1037 -> 256 and 256 -> 128) and of the two-tower step
    (192 -> 256, 256 -> 128), as DCNTrainer / TwoTowerTrainer call them.
    wgrad: dW = X^T dZ and db from the split operand (mm_dense_wgrad_split) and from fp32 X at a row stride that is a
    multiple of 4; bound of test_dense_wgrad_at_scale, 2 (U + (3 rows / 16 + CTAs) E) (|X|^T |dZ|) for dW and
    2 (rows + 256 + CTAs) E sum |dZ| for db.  dW sits in a buffer with a NaN tail that must stay NaN.
    dgrad (what _dgrad runs): N > 128 on the tensor cores, mm_dense_tc(split_rows(dZ), N, split_weights(W^T), K, None,
    None, out_f32=dX), within (U + N E) (|dZ| |W|^T); N <= 128 mm_dense_dgrad, within 4 U (|dZ| |W|^T) (at
    M = 16 421, K = 256 that kernel makes a single lap; test_dense_dgrad_at_scale covers its laps).  dX at row stride
    1040 for K = 1037 (the trainer's), K + 4 otherwise, with NaN guard rows and padding."""
    sms = _sms(device)
    rows, gx = _wgrad_launch(M, K, N, sms)
    assert rows // 32 >= 2, f"premise: {rows} rows per CTA is a single chunk"
    wide = N > 128
    if wide:
        assert _dense_tc_laps(M, K, sms) >= 2, "premise: the transposed dgrad makes a single lap"
    elif M >= BIG:
        assert _dgrad_laps(M, K, sms) >= 2, "premise: dense_dgrad makes a single lap"
    gen = torch.Generator(device=device).manual_seed(M + 3 * K + N)
    ld = LD if K == D_DCN else K + 4
    xb, x = _filled(M, ld, K, gen, device)
    if K == 256:
        x.clamp_(min=0.0)  # a relu layer's output
    dz = torch.randn((M, N), generator=gen, device=device)
    W = torch.randn((K, N), generator=gen, device=device) / K ** 0.5
    xd, zd = x.double(), dz.double()
    ref_w, ref_b = xd.t() @ zd, zd.sum(0)
    bw = 2 * (U + (3 * rows / 16 + gx) * E) * (xd.abs().t() @ zd.abs())
    bb = 2 * (rows + 256 + gx) * E * zd.abs().sum(0)
    del xd
    for split in (True, False):
        wbuf = _nan((K * N + 64,), device)
        wbuf[:K * N].zero_()
        dw = wbuf[:K * N].view(K, N)
        db = torch.zeros(N, device=device)
        if split:
            ops.dense_wgrad_split(ops.split_rows(x), K, dz, dw, db)
        else:
            ops.dense_wgrad(x, dz, dw, db)
        _within(dw, ref_w, bw, f"dW (split operand {split})")
        _within(db, ref_b, bb, f"db (split operand {split})")
        assert bool(torch.isnan(wbuf[K * N:]).all()), "dW: written past its end"
    del ref_w, bw, wbuf
    _free()
    dxb = _nan((M + GUARD, ld), device)
    dx = dxb[:M, :K]
    if wide:
        ops.dense_tc(ops.split_rows(dz), N, ops.split_weights(W.t().contiguous()), K, None, None, out_f32=dx)
    else:
        ops.dense_dgrad(dz, W, dx)
    _untouched(dxb, M, K, "dX")
    Wd = W.double()
    for s, e in _chunks(M):
        z = dz[s:e].double()
        bound = ((U + N * E) if wide else 4 * U) * (z.abs() @ Wd.abs().t())
        _within(dx[s:e], z @ Wd.t(), bound, f"dX rows [{s}, {e})")


# ---------------------------------------------------------------------------------------------------------------
# A5. mm_l2_normalize / mm_l2_normalize_backward past one lap
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [64, 128])
def test_l2_normalize_and_backward_at_scale(device, D):
    """y = x / sqrt(max(|x|^2, 1e-12)) and its backward at B = 65 573 (one warp per row, 32 SMs x 8 warps per lap: two
    laps), rows at strides D + 4 (x), D + 8 (y), D + 12 (dy), every 97th row zero and every 97th (offset 5) of norm
    ~1e-7 < 1e-6, so that both branches of the backward run.  The backward runs in place (dx aliasing dy), as
    TwoTowerTrainer calls it.  Bounds: the fp32 sum of D squares is within D E of |x|^2, so n = sqrt(.) within
    (D / 2 + 1) E and y within (D + 3) E |y|; dx = (dy - y (y . dy)) / n within (2 D + 8) E of
    (|dy| + |y| sum |x| |dy| / n) / n.  Below the threshold n is the constant 1e-6 and dx = dy / 1e-6."""
    B = RAGGED
    blocks = min(-(-B * 32 // 256), 32 * _sms(device))
    laps = -(-B // (blocks * 8))
    assert laps >= 2, f"premise: B = {B} gives {laps} lap(s)"
    gen = torch.Generator(device=device).manual_seed(D)
    xb, x = _filled(B, D + 4, D, gen, device)
    x[::97] = 0.0
    x[5::97] *= 1e-8
    x[B - 1] = 0.0
    yb = _nan((B + GUARD, D + 8), device)
    ops.l2_normalize(x, out=yb[:B, :D])
    _untouched(yb, B, D, "y")
    gb, dy = _filled(B, D + 12, D, gen, device)
    dy0 = dy.clone()
    ops.l2_normalize_backward(x, dy, dy)
    _untouched(gb, B, D, "dx (in place)")
    xd, gd = x.double(), dy0.double()
    ss = (xd * xd).sum(1, keepdim=True)
    on = ss >= float(np.float32(1e-12))
    assert int((~on).sum()) >= 2 * (B // 97) and bool(on.any()), "premise: rows on both sides of the threshold"
    n = torch.where(on, ss.sqrt(), torch.full_like(ss, float(np.float32(1e-6))))
    y = xd / n
    _within(yb[:B, :D], y, (D + 3) * E * y.abs(), "y")
    yg = torch.where(on, (xd * gd).sum(1, keepdim=True) / n, torch.zeros_like(ss))
    want = (gd - y * yg) / n
    scale = (gd.abs() + y.abs() * (xd.abs() * gd.abs()).sum(1, keepdim=True) / n) / n
    _within(dy, want, (2 * D + 8) * E * scale, "dx (in place)")


# ---------------------------------------------------------------------------------------------------------------
# A6. mm_dense_apply over a DCN-sized arena
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
def test_dense_apply_over_many_laps(device, opt):
    """SGD, Adagrad and Adam over n = 3 500 003 floats (the DCN arena holds about 3.5 M; 8 SMs x 256 threads per lap:
    13 laps) with grad_scale = 0.3.  The weights against _rule at g = fl(0.3f g) (one rounding, E |g s|, which moves the
    update by at most lip E |g s|): bound 2 (lip E |g s| + E |w| + 8 E terms).  The optimizer states within 6 E of their
    terms (the scaled g rounded, then two products and a sum).  The gradient is exactly zero afterwards; 64 NaN floats
    past the end of every buffer stay NaN."""
    n = 3_500_003
    blocks = min(-(-n // 256), 8 * _sms(device))
    laps = -(-n // (blocks * 256))
    assert laps >= 2, f"premise: n = {n} gives {laps} lap(s)"
    eps = 1e-6 if opt == "adam" else 1e-7
    o = {"sgd": mm.SGD(0.05), "adagrad": mm.Adagrad(0.05), "adam": mm.Adam(0.01, epsilon=eps)}[opt]
    hyper = torch.from_numpy(o.hyper()).to(device)
    gen = torch.Generator(device=device).manual_seed(len(opt))

    def buf(values):
        b = _nan((n + 64,), device)
        b[:n].copy_(values)
        return b

    wb = buf(torch.randn(n, generator=gen, device=device) * 0.1)
    gb = buf(torch.randn(n, generator=gen, device=device))
    s1b = s2b = None
    if opt == "adagrad":
        s1b = buf(0.1 + torch.rand(n, generator=gen, device=device))
    elif opt == "adam":
        s1b = buf(torch.randn(n, generator=gen, device=device) * 0.01)
        s2b = buf(torch.rand(n, generator=gen, device=device) * 1e-4)
    w0, g0 = wb[:n].double(), gb[:n].double()
    s10 = None if s1b is None else s1b[:n].double()
    s20 = None if s2b is None else s2b[:n].double()
    ops.opt_tick(hyper)
    ops.opt_tick(hyper)  # step 2: Adam's lr_t differs from lr
    scale = 0.3
    ops.dense_apply(opt, wb[:n], gb[:n], None if s1b is None else s1b[:n], None if s2b is None else s2b[:n], hyper, grad_scale=scale)
    hy = hyper.cpu().numpy()
    gs = g0 * float(np.float32(scale))
    st1 = s10 if opt == "adagrad" else None
    st2 = (s10, s20) if opt == "adam" else None
    want, lip, terms = _rule(opt, w0, st1, st2, gs, hy)
    dg = E * gs.abs()
    if opt == "adam":  # Adam's derivative grows as |g| shrinks: also take it at the smallest |g| within dg
        lip = torch.maximum(lip, _rule(opt, w0, st1, st2, gs.sign() * (gs.abs() - dg).clamp_min(0.0), hy)[1])
    _within(wb[:n], want, 2 * (lip * dg + E * want.abs() + 8 * E * terms), f"{opt}: weights")
    assert torch.equal(gb[:n], torch.zeros(n, device=device)), f"{opt}: the gradient was not cleared everywhere"
    if opt == "adagrad":
        _within(s1b[:n], s10 + gs * gs, 6 * E * (s10 + gs * gs), "adagrad: accumulator")
    elif opt == "adam":
        b1, b2 = float(hy[HYPER_BETA1]), float(hy[HYPER_BETA2])
        _within(s1b[:n], b1 * s10 + (1 - b1) * gs, 6 * E * (b1 * s10.abs() + (1 - b1) * gs.abs()), "adam: m")
        _within(s2b[:n], b2 * s20 + (1 - b2) * gs * gs, 6 * E * (b2 * s20 + (1 - b2) * gs * gs), "adam: v")
    for what, b in (("weights", wb), ("gradient", gb), ("state1", s1b), ("state2", s2b)):
        if b is not None:
            assert bool(torch.isnan(b[n:]).all()), f"{opt}: {what} written past the arena"


# ---------------------------------------------------------------------------------------------------------------
# Shared by B and C: float64 references of a training step and the checks that follow them
# ---------------------------------------------------------------------------------------------------------------
class _Ref:
    """float64 autograd bookkeeping of a chain of Dense layers: the parameters, the terms |X|^T |dZ| and sum |dZ| of each
    dense gradient (the scale of the fp32 sums that make it), and per sample whether a relu unit is on in one
    implementation and off in the other."""

    def __init__(self, layers):
        self.layers = layers
        self.P = [(l.kernel.double().requires_grad_(True), None if l.bias is None else l.bias.double().requires_grad_(True))
                  for l in layers]
        self.terms = {}
        self.pre = []

    def dense(self, h, li, saved=None, flips=None):
        (Wk, bk), l = self.P[li], self.layers[li]
        z = h @ Wk + (bk if bk is not None else 0.0)
        z.retain_grad()
        self.pre.append((li, h.detach(), z))
        if l.activation != "relu":  # linear, or a head whose loss takes the logits
            return z
        with torch.no_grad():  # on/off differently: only ever a unit within rounding of zero
            flip = (saved > 0) != (z > 0)
            band = (h.abs() @ Wk.abs() + (bk.abs() if bk is not None else 0.0)) * 2.0 ** -10
            assert bool((z.abs()[flip] <= band[flip]).all()), f"layer {l.name}: a unit far from zero is on/off differently"
        flips.append(flip.any(1))
        return torch.relu(z)

    def collect(self):
        """Adds the terms of the layers run since the last call (after backward)."""
        for li, hin, z in self.pre:
            name = self.layers[li].name
            self.terms[f"{name}/kernel"] = self.terms.get(f"{name}/kernel", 0.0) + hin.abs().t() @ z.grad.abs()
            self.terms[f"{name}/bias"] = self.terms.get(f"{name}/bias", 0.0) + z.grad.abs().sum(0)
        self.pre = []

    def grads(self, prefix=lambda l: ""):
        out = {}
        for l, (Wk, bk) in zip(self.layers, self.P):
            out[f"{prefix(l)}{l.name}/kernel"] = Wk.grad
            if bk is not None:
                out[f"{prefix(l)}{l.name}/bias"] = bk.grad
        return out, {f"{prefix(l)}{k}": v for l in self.layers for k, v in self.terms.items() if k.startswith(f"{l.name}/")}


def _check_gradients(tr, want_loss, want, terms, slices, flipped, B, slice_terms=None):
    """(b) of the step tests: the loss at rtol 1e-5; each dense gradient's Frobenius error under 1e-4 of the Frobenius
    norm of its terms; the slices per element within 1e-3 |ref| + 3e-4 max |ref slices of that sample| or, given their
    terms, 1e-3 |ref| + 1e-4 terms, leaving out the samples with a relu unit on/off differently (fewer than 1 % of the
    batch)."""
    np.testing.assert_allclose(float(tr.loss[0].item()), want_loss, rtol=1e-5)
    got = tr.gradients()
    assert sorted(got) == sorted(want)
    for k in want:
        fro = float((got[k].double() - want[k]).norm() / terms[k].norm())
        assert fro < 1e-4, f"{k}: Frobenius error {fro:.3e} of the terms' scale"
    n_flip = int(flipped.sum())
    assert n_flip < B // 100, f"{n_flip} samples have a relu unit on/off differently"
    keep = ~flipped
    scale = torch.stack([s.abs().amax(1) for s in slices]).amax(0)[keep].unsqueeze(1)
    for t, f in enumerate(tr.feats):
        r = slices[t][keep]
        bound = 1e-3 * r.abs() + (3e-4 * scale if slice_terms is None else 1e-4 * slice_terms[t][keep])
        _within(tr._slices[t][keep], r, bound, f"slices of {f}")


def _same_bits(got, want, what):
    if not torch.equal(got.view(torch.int16), want.view(torch.int16)):
        bad = (got.view(torch.int16) != want.view(torch.int16)).nonzero()
        raise AssertionError(f"{what}: {bad.shape[0]} of {got.numel()} elements differ (first at {bad[0].tolist()}: got "
                             f"{float(got[tuple(bad[0])])}, want {float(want[tuple(bad[0])])}; NaN got/want "
                             f"{int(torch.isnan(got).sum())}/{int(torch.isnan(want).sum())})")


def _check_operands(tr, transposed):
    """Every layer's split kernel is the split of its current kernel bit for bit; `transposed` (after a backward, which
    refreshes them before use): so is the transposed split kernel of every wide layer."""
    for li, (l, ws) in enumerate(zip(tr._tc_layers, tr._wsplit)):
        assert l._w_split is ws
        _same_bits(ws, ops.split_weights(l.kernel), f"layer {li} ({l.name}): _w_split")
    for li, w in tr._wide.items() if transposed else ():
        l = tr._tc_layers[li]
        _same_bits(w["wT_split"], ops.split_weights(l.kernel.t().contiguous()), f"layer {li} ({l.name}): wT_split")


def _step_variables(tr):
    out = [t.table for t in tr.tables]
    a = tr.arena
    for i in range(len(a.layers)):
        out += [v for v in (a.view(a.w, i, "kernel"), a.view(a.w, i, "bias")) if v is not None]
    return out


def _graph_vs_eager(ta, tb, packed, static, inputs, y, hosts, columns, label=None):
    """(a) of the step tests: two graph replays of `ta` on packed ids against two eager steps of its twin `tb` on int64
    ids; the losses at rtol 1e-6 and every variable within 1e-5 of its scale (same kernels; only the order of the fp32
    atomics differs)."""
    dev = static.device
    ta.capture(inputs, y, clone=False)
    for i in (0, 1):
        static.copy_(packed[i])
        la = float(ta.replay()[0].item())
        x = {k: torch.from_numpy(np.asarray(hosts[i][k]).astype(np.int64) if np.asarray(hosts[i][k]).dtype.kind in "iu"
                                 else np.asarray(hosts[i][k])).to(dev) for k in columns}
        yb = None if label is None else torch.from_numpy(np.asarray(hosts[i][label])).to(dev)
        lb = float(tb.step(x, yb)[0].item())
        np.testing.assert_allclose(la, lb, rtol=1e-6)
    for i, (va, vb) in enumerate(zip(_step_variables(ta), _step_variables(tb))):
        err = float((va - vb).abs().max()) / max(float(vb.abs().max()), 1e-30)
        assert err < 1e-5, f"variable {i}: graph replay on packed ids vs eager on int64 ids differ by {err:.3e} of the scale"


def _check_update(tr, opt, before, slices, ids, what):
    """(c) of the step tests: the sparse update of every table (_check_sparse_update); returns the largest fold count
    of each table."""
    hy = tr.hyper.cpu().numpy()
    hottest = {}
    for t, f in enumerate(tr.feats):
        cnt = _check_sparse_update(opt, f"{what}, table of {f}", before[t], (tr.tables[t].table, tr.tstate1[t], tr.tstate2[t]),
                                   ids[t], slices[t], hy)
        hottest[f] = int(cnt.max())
    return hottest


# ---------------------------------------------------------------------------------------------------------------
# B. the DCN-v2 step as the benchmark's model would train it
# ---------------------------------------------------------------------------------------------------------------
def _dcn_bench_model(device, seed, stacked=True):
    """DCNModel(Criteo schema capped at 400 000 rows, depth 3, deep [256, 128]) with every table at the width the
    uncapped schema infers (so d stays 1037), Adagrad(0.01)."""
    _, widths, _ = _dcn_widths()
    dims = {f: widths[f] for f in datasets.CRITEO_MAX}
    schema = datasets.criteo_schema({k: min(v, CAP - 1) for k, v in datasets.CRITEO_MAX.items()})
    mm.set_seed(seed)
    model = mm.DCNModel(schema, depth=3, deep_block=mm.MLPBlock([256, 128]), stacked=stacked, dim=dims)
    model.build(device)
    model.compile(optimizer=mm.Adagrad(0.01))
    assert model.body.input_block.layout()[2] == D_DCN
    return schema, model


def _dcn_packed(schema, model, B, seeds, device):
    label = schema.select_by_tag(mm.Tags.TARGET).column_names[0]
    hosts = [datasets.generate_batch(schema, B, seed=s, index_law="uniform", index_dtype=np.int32) for s in seeds]
    names = model.input_columns() + [label]
    hbs = [HostBatch.like(h, names, id_bytes=model.id_bytes()) for h in hosts]
    packed = [hb.buffer.to(device) for hb in hbs]
    static = packed[0].clone()
    views = {k: _view(static, hbs[0].offsets[k], shp, dt) for k, (shp, dt) in hbs[0].spec.items()}
    return label, hosts, packed, static, {k: v for k, v in views.items() if k != label}, views[label]


def _dcn_reference(tr, inputs, y, B, chunk=4096):
    """float64 autograd on the device of DCNTrainer's step (x0 from the tables and the continuous columns, 3 cross layers
    x_{l+1} = x0 (x_l W_l + b_l) + x_l, the relu deep tower on x_L (stacked) or x0 (parallel), the head on the deep output
    or on [cross | deep], mean BCE), in sample chunks.  Returns the loss, the dense gradients and their terms by variable
    name, the slices per table and the per-sample relu flips."""
    L, nd = len(tr.cross), len(tr.deep)
    ref = _Ref(tr.cross + tr.deep + [tr.head])
    ids = [ops.widen_index(i).long() for i in tr._idx]
    saved = [h[:B] for h in tr.h]
    if not tr.stacked:
        saved[-1] = tr.cat[:B, tr.doff:tr.doff + tr.deep[-1].units]
    yd = y.reshape(-1).double()
    loss, slices, flips = 0.0, [[] for _ in ids], []
    for s, e in _chunks(B, chunk):
        x0 = torch.zeros((e - s, tr.inp.d), dtype=torch.float64, device=yd.device)
        for t, f in enumerate(tr.feats):
            c, w = tr.inp.cols[f], tr.tables[t].table.shape[1]
            x0[:, c:c + w] = tr.tables[t].table[ids[t][s:e]].double()
        for n in tr.inp.cont:
            x0[:, tr.inp.cols[n]] = inputs[n].reshape(-1)[s:e].double()
        x0.requires_grad_(True)
        flip = []
        x = x0
        for l in range(L):
            x = x0 * ref.dense(x, l) + x
        h = x if tr.stacked else x0
        for i in range(nd):
            h = ref.dense(h, L + i, saved[i][s:e], flip)
        head_in = h if tr.stacked else torch.cat([x, h] if tr.order == ("cross", "deep") else [h, x], dim=1)
        logit = ref.dense(head_in, L + nd).reshape(-1)
        yy = yd[s:e]
        part = (torch.clamp(logit, min=0) - logit * yy + torch.log1p(torch.exp(-logit.abs()))).sum() / B
        part.backward()
        loss += float(part.detach())
        for t, f in enumerate(tr.feats):
            c, w = tr.inp.cols[f], tr.tables[t].table.shape[1]
            slices[t].append(x0.grad[:, c:c + w])
        flips.append(torch.stack(flip).any(0))
        ref.collect()
    grads, terms = ref.grads()
    return loss, grads, terms, [torch.cat(s) for s in slices], torch.cat(flips)


def test_dcn_train_step_at_benchmark_size(device):
    """DCNModel(Criteo schema capped at 400 000 rows, depth 3, deep [256, 128]) with the uncapped schema's widths
    (d = 1037), Adagrad, B = 65 536, packed 1/2/3-byte ids through HostBatch into one CUDA graph.  The tables cover every
    sparse path: counting sort (<= 1024 rows), the dense accumulator (<= DENSE_PATH_MAX_ROWS) and the election at widths
    48, 64, 96 and 120.
    (a) two graph replays against two eager steps of a twin model on int64 ids (_graph_vs_eager);
    (b) forward_backward on a third batch, after two updates, so that the refreshed split kernels and transposed split
        kernels are the ones in use (asserted bit for bit: at lr 0.01 most updates are a few ulps, so a stale transposed
        kernel would stay inside every tolerance), against float64 autograd (_check_gradients; observed on an H100: the
        slices within 4.1e-2 of their bound, 30 samples with a relu unit on/off differently);
    (c) the Adagrad update of every table against the float64 rule on the summed slices (_check_sparse_update); then
        every layer's split kernel equals split_weights(kernel) bit for bit.  (The transposed split kernels stay one
        update behind until the next backward refreshes them before use.)"""
    B = BIG
    schema, ma = _dcn_bench_model(device, 41)
    _, mb = _dcn_bench_model(device, 41)
    label, hosts, packed, static, inputs, y = _dcn_packed(schema, ma, B, (5150, 5151, 5152), device)
    ta, tb = ma.trainer(B), mb.trainer(B)
    assert ta.inp.d == D_DCN and ta.stacked and sorted(ta._wide) == [0, 1, 2, 3]  # the cross layers and the 256-unit layer
    rows = {f: t.table.shape[0] for f, t in zip(ta.feats, ta.tables)}
    widths = {f: t.table.shape[1] for f, t in zip(ta.feats, ta.tables)}
    assert min(rows.values()) <= COUNTING_SORT_MAX_ROWS and any(COUNTING_SORT_MAX_ROWS < r <= DENSE_PATH_MAX_ROWS for r in rows.values())
    assert {widths[f] for f, r in rows.items() if r > DENSE_PATH_MAX_ROWS} == {48, 64, 96, 120}
    assert set(ma.id_bytes().values()) == {1, 2, 3}
    _graph_vs_eager(ta, tb, packed, static, inputs, y, hosts, ma.input_columns(), label)
    del tb, mb
    _free()

    # (b)
    static.copy_(packed[2])
    ta.forward_backward(inputs, y)
    _check_operands(ta, transposed=True)
    want_loss, want, terms, ref_slices, flipped = _dcn_reference(ta, inputs, y, B)
    _check_gradients(ta, want_loss, want, terms, ref_slices, flipped, B)
    del want, terms, ref_slices
    _free()

    # (c)
    before = [(t.table.clone(), a.clone(), None) for t, a in zip(ta.tables, ta.tstate1)]
    slices = [s.clone() for s in ta._slices]  # the update folds duplicates into the slices in place
    ids = [ops.widen_index(i).long() for i in ta._idx]
    ta.apply_gradients()
    _check_update(ta, "adagrad", before, slices, ids, "Adagrad step")
    _check_operands(ta, transposed=False)


def test_dcn_parallel_step_gradients_at_scale(device):
    """The parallel body at B = 65 573: the deep tower on x0, the head on [cross | deep] of 1037 + 128 = 1165 inputs,
    beyond the fused loss kernel's 256 (the wide-head composition: tensor-core logits, mm_heads_fwd_bwd with an
    identity kernel, mm_dense_wgrad_split and mm_dense_dgrad of the head).  forward_backward on packed ids against
    float64 autograd, with the checks of (b) above (observed on an H100: dense gradients within 1.9e-5 of their terms,
    slices within 2.7e-2 of their bound, 52 samples with a relu unit on/off differently)."""
    B = RAGGED
    schema, model = _dcn_bench_model(device, 43, stacked=False)
    _, _, _, _, inputs, y = _dcn_packed(schema, model, B, (6160,), device)
    tr = model.trainer(B)
    assert not tr.stacked and tr.wide_head and tr.head.input_dim == D_DCN + 128
    tr.forward_backward(inputs, y)
    want_loss, want, terms, ref_slices, flipped = _dcn_reference(tr, inputs, y, B)
    _check_gradients(tr, want_loss, want, terms, ref_slices, flipped, B)


# ---------------------------------------------------------------------------------------------------------------
# C. the two-tower step as the benchmark's model would train it
# ---------------------------------------------------------------------------------------------------------------
def _tt_bench_model(device, seed):
    mm.set_seed(seed)
    model = mm.TwoTowerModel(datasets.retrieval_10m_schema(), query_tower=mm.MLPBlock([256, 128]))
    model.build(device)
    model.compile(optimizer=mm.Adagrad(0.01))
    return model


def _ce_terms(q, items, ids, T, c, chunk=2048):
    """The absolute terms of the in-batch soft-max cross-entropy gradients that _ce_ref_chunked sums, in row chunks:
    for the query (c p_0 + c) / T |pos| + sum_j c p_j / T |item_j| over the negatives that are not down-scored, for each
    item the same products with |q| (as positive and as negative)."""
    B = q.shape[0]
    mf = float(np.float32(O.MIN_FLOAT))
    aq, ai = torch.zeros_like(q), torch.zeros_like(items)
    qa, ia = q.abs(), items.abs()
    for s, e in _chunks(B, chunk):
        m = ids[s:e].view(-1, 1) == ids.view(1, -1)
        sn = torch.where(m, torch.full((), mf, dtype=torch.float64, device=q.device), q[s:e] @ items.T)
        z = torch.cat([(q[s:e] * items[s:e]).sum(-1, keepdim=True), sn], dim=1) / T
        p = c * torch.softmax(z, 1)
        p0 = (p[:, :1] + c) / T
        pn = p[:, 1:].masked_fill(m, 0.0) / T
        aq[s:e] = p0 * ia[s:e] + pn @ ia
        ai[s:e] += p0 * qa[s:e]
        ai += pn.T @ qa[s:e]
    return aq, ai


def _tt_reference(tr, inputs, B):
    """float64 autograd on the device of TwoTowerTrainer's step: per tower x0 from the tables, the relu tower; the
    in-batch soft-max cross-entropy with the item-id down-scoring and its gradients w.r.t. both outputs from
    _ce_ref_chunked (the (B, B) logits in row chunks), back-propagated through the towers.
    The terms of the dense gradients: the soft-max gradients are sums over the batch whose terms cancel to far less
    than their size (each query's positive term against its 16 383 negatives), and their rounding is relative to
    those terms, not to the result.  So the scale dZ_l of each layer's fp32 sums is propagated down the towers from
    the absolute soft-max terms (_ce_terms): dZ_L = relu'(z_L) |terms|, dZ_{l-1} = relu'(z_{l-1}) (dZ_l |W_l|^T), and
    the terms of dW_l are |X_l|^T dZ_l (of db_l, sum dZ_l)."""
    assert not tr.l2 and tr.downscore and tr.false_neg_score == O.MIN_FLOAT
    ref = _Ref([l for tw in tr.towers for l in tw["layers"]])
    names = {id(l): f"{tw['name']}/" for tw in tr.towers for l in tw["layers"]}
    outs, x0s, flips = [], [], []
    for tw, inp in zip(tr.towers, tr.inps):
        x0 = torch.zeros((B, inp.d), dtype=torch.float64, device=tr.device)
        for t, f in zip(inp.tidx, inp.feats):
            c, w = inp.cols[f], tr.tables[t].table.shape[1]
            x0[:, c:c + w] = tr.tables[t].table[ops.widen_index(tr._idx[t]).long()].double()
        for n in inp.cont:
            x0[:, inp.cols[n]] = inputs[n].reshape(-1).double()
        x0.requires_grad_(True)
        h = x0
        for i in range(len(tw["layers"])):
            h = ref.dense(h, tw["li0"] + i, tw["h"][i][:B], flips)
        outs.append(h)
        x0s.append(x0)
    ids = ops.widen_index(inputs[tr.item_id]).long().reshape(-1)
    q, it = outs
    loss, gq, gp, gn = _ce_ref_chunked(q.detach(), it.detach(), it.detach(), ids, ids, tr.temperature, 1.0 / B)
    torch.autograd.backward([q, it], [gq, gp + gn])
    grads, _ = ref.grads(lambda l: names[id(l)])
    pre = {li: (hin, z.detach()) for li, hin, z in ref.pre}
    terms, slice_terms = {}, [None] * len(tr.tables)
    with torch.no_grad():
        for tw, inp, dz in zip(tr.towers, tr.inps, _ce_terms(q.detach(), it.detach(), ids, tr.temperature, 1.0 / B)):
            for i in range(len(tw["layers"]) - 1, -1, -1):
                l = tw["layers"][i]
                hin, z = pre[tw["li0"] + i]
                if l.activation == "relu":
                    dz = dz * (z > 0)
                terms[f"{tw['name']}/{l.name}/kernel"] = hin.abs().t() @ dz
                if l.bias is not None:
                    terms[f"{tw['name']}/{l.name}/bias"] = dz.sum(0)
                dz = dz @ l.kernel.double().abs().t()
            for t, f in zip(inp.tidx, inp.feats):
                c, w = inp.cols[f], tr.tables[t].table.shape[1]
                slice_terms[t] = dz[:, c:c + w]
    slices = [None] * len(tr.tables)
    for inp, x0 in zip(tr.inps, x0s):
        for t, f in zip(inp.tidx, inp.feats):
            c, w = inp.cols[f], tr.tables[t].table.shape[1]
            slices[t] = x0.grad[:, c:c + w]
    return loss, grads, terms, slices, torch.stack(flips).any(0), slice_terms


def test_twotower_train_step_at_benchmark_size(device):
    """TwoTowerModel(retrieval_10m_schema(): 10 M-row item table, 1 M-row user table; towers [256, 128]) at full size,
    Adagrad, B = 16 384, Zipf ids (generate_batch's law of the benchmark), packed through HostBatch: user_id and item_id
    as 3-byte ids.  Adagrad rather than Adam: Adam divides every update by sqrt(v), so an element whose gradient
    cancels to near zero in the sum over 16 384 samples moves by about lr whatever its size, and the order of the fp32
    atomics alone then moves it by more than 1e-5 of its variable's scale in (a) (observed on an H100: 1.7e-5 in one of
    two runs); Adagrad's update is proportional to the gradient.  The Adam rules at scale are checked by
    test_dense_apply_over_many_laps and test_sparse_rows_apply_at_scale.
    (a) two graph replays against two eager steps of a twin model on int64 ids (_graph_vs_eager);
    (b) forward_backward on a third batch after two updates against float64 autograd (_tt_reference; _check_gradients
        with the slices bounded by their propagated terms; observed on an H100: dense gradients within 4.8e-5 of their
        terms, slices within 8.1e-2 of their bound, 10 samples with a relu unit on/off differently);
    (c) the Adagrad update of every table (_check_update): the 10 M-row item table and the 1 M-row user table on the
        election path, where the hottest Zipf row folds hundreds of duplicates (about 800 of 16 384 at a = 1.05);
        the split kernels in step."""
    B = TT
    ma = _tt_bench_model(device, 51)
    mb = _tt_bench_model(device, 51)
    schema = ma.schema
    widths = ma.id_bytes()
    assert widths["user_id"] == 3 and widths["item_id"] == 3
    hosts = [datasets.generate_batch(schema, B, seed=7070 + i, index_law="zipf", index_dtype=np.int32) for i in range(3)]
    names = ma.input_columns()
    hbs = [HostBatch.like(h, names, id_bytes=widths) for h in hosts]
    packed = [hb.buffer.to(device) for hb in hbs]
    static = packed[0].clone()
    inputs = {k: _view(static, hbs[0].offsets[k], shp, dt) for k, (shp, dt) in hbs[0].spec.items()}
    ta, tb = ma.trainer(B), mb.trainer(B)
    assert type(ta).__name__ == "TwoTowerTrainer" and sorted(ta._wide) == [0, 2]  # each tower's 256-unit layer
    rows = {f: t.table.shape[0] for f, t in zip(ta.feats, ta.tables)}
    assert rows["item_id"] == 10_000_000 and rows["user_id"] == 1_000_000
    _graph_vs_eager(ta, tb, packed, static, inputs, None, hosts, names)
    del tb, mb
    _free()

    # (b)
    static.copy_(packed[2])
    ta.forward_backward(inputs, None)
    _check_operands(ta, transposed=True)
    want_loss, want, terms, ref_slices, flipped, slice_terms = _tt_reference(ta, inputs, B)
    _check_gradients(ta, want_loss, want, terms, ref_slices, flipped, B, slice_terms)
    del want, terms, ref_slices, slice_terms
    _free()

    # (c)
    before = [(t.table.clone(), a.clone(), None) for t, a in zip(ta.tables, ta.tstate1)]
    slices = [s.clone() for s in ta._slices]
    ids = [ops.widen_index(i).long() for i in ta._idx]
    ta.apply_gradients()
    hottest = _check_update(ta, "adagrad", before, slices, ids, "Adagrad step")
    assert hottest["item_id"] > 500 and hottest["user_id"] > 500, f"premise: hot rows fold hundreds of duplicates: {hottest}"
    _check_operands(ta, transposed=False)


# ---------------------------------------------------------------------------------------------------------------
# D. the pipelined forward as bench.py times it
# ---------------------------------------------------------------------------------------------------------------
def _bench_forward(kind, device):
    """The model, batch size, pipeline depth, call arguments, id law and whether ids travel packed, as bench.py builds
    them for its dlrm, dcn and twotower forwards."""
    if kind == "dlrm":
        schema = datasets.criteo_schema()
        model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([128, 64]), top_block=mm.MLPBlock([128, 64, 32]),
                             embedding_options=mm.EmbeddingOptions(embeddings_initializers={"hash_seed": 4321}))
        cfg = (BIG, 3, {}, "uniform", True)
    elif kind == "dcn":
        mm.set_seed(1)
        schema = datasets.criteo_schema()
        model = mm.DCNModel(schema, depth=3, deep_block=mm.MLPBlock([256, 128]), embeddings_initializer={"hash_seed": 99})
        cfg = (BIG, 2, {}, "uniform", False)
    else:
        mm.set_seed(1)
        schema = datasets.retrieval_10m_schema()
        model = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([256, 128]),
                                 embedding_options=mm.EmbeddingOptions(embeddings_initializers={"hash_seed": 5}))
        cfg = (TT, 2, {"training": True}, "zipf", False)
    model.build(device)
    return schema, model, cfg


@pytest.mark.parametrize("kind", ["dlrm", "dcn", "twotower"])
def test_pipelined_forward_as_the_benchmark_times_it(device, kind):
    """model.pipeline(...).submit_device(...) as bench.py times it: DLRM at B = 65 536 with depth 3 (packed 1/2/3-byte
    ids), DCN-v2 at B = 65 536 with depth 2, the two-tower model at B = 16 384 with depth 2 and training=True (its
    output is the (B, 1 + B) logits).  2 depth + 1 submissions over depth + 1 rotating device batches, with no join in
    between: before a slot is reused its output is snapshotted on the slot's stream.  Each snapshot equals the eager
    forward of its own batch bit for bit, and no two slots share an output buffer."""
    schema, model, (B, depth, kw, law, packed_ids) = _bench_forward(kind, device)
    n = depth + 1
    hosts = [datasets.split_targets(schema, datasets.generate_batch(schema, B, seed=1234 + i, index_law=law, index_dtype=np.int32))[0]
             for i in range(n)]
    cols = model.input_columns()
    hbs = [HostBatch.like(h, cols, id_bytes=model.id_bytes() if packed_ids else None) for h in hosts]
    packed = [hb.buffer.to(device) for hb in hbs]
    want = []
    for h in hosts:
        out = model({k: torch.from_numpy(h[k]).to(device) for k in cols}, **kw)
        want.append((out.outputs if isinstance(out, Prediction) else out).clone())
    if kind == "twotower":
        assert want[0].shape == (B, 1 + B)
    pf = model.pipeline(hbs[0], depth=depth, **kw)
    ptrs = {pf.output(k).data_ptr() for k in range(depth)}
    assert len(ptrs) == depth, "two pipeline slots share one output buffer"
    pending, snaps = [None] * depth, []
    for i in range(2 * depth + 1):
        k = i % depth
        if pending[k] is not None:
            with torch.cuda.stream(pf.streams[k]):
                snaps.append((pending[k], pf.output(k).clone()))
        assert pf.submit_device(packed[i % n]) == k
        pending[k] = i % n
    pf.join()
    for k in range(depth):
        snaps.append((pending[k], pf.output(k).clone()))
    torch.cuda.synchronize()
    assert len(snaps) == 2 * depth + 1
    for j, (b, got) in enumerate(snaps):
        assert torch.equal(got, want[b]), f"submission {j} (batch {b}, slot {j % depth}) differs from the eager forward of its batch"
