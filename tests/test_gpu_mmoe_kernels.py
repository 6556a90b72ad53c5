"""The MMoE kernels against float64 at every compiled instantiation: mm_mmoe_mix_fwd, mm_mmoe_mix_bwd and
mm_mmoe_task_heads_fwd_bwd (the task-tower path), and the fused mm_mmoe_heads_fwd_bwd at the widths and expert counts
its own tests leave out.

Each kernel is compiled for NH x C = {1, 2, 4, 8} x {1, 2, 4, 8}: NH is the task count H rounded up to a power of two
(tasks t >= H are skipped at run time) and C the columns per lane of the width n (1: n <= 32, 2: <= 64, 4: <= 128,
8: <= 256).  CASES reaches every pair once (tests/test_mmoe_host.py checks that), with full and partial last column
groups, E in {1, 4, 16} (H E = 128: the warp's whole shared-memory row), gate logits as separate (B, E) tensors and as
column views of one stacked matrix (as MMOEBlock.gate_logits gives them), and B in {37, 1 001} (one grid-stride lap) or {65 536, 65 573} (15-16 laps of 4 SMs x 8 warps, the last one ragged).

    H  U    E   B       NH C        H  U    E   B       NH C
    1  7    4   37      1  1        3  32   16  65536   4  1
    1  64   16  1001    1  2        4  64   4   1001    4  2
    1  100  1   1001    1  4        3  100  4   37      4  4
    1  256  4   65536   1  8        4  256  1   1001    4  8
    2  32   1   1001    2  1        5  7    4   1001    8  1
    2  33   4   37      2  2        8  33   16  1001    8  2
    2  128  16  65573   2  4        8  128  4   65536   8  4
    2  129  4   1001    2  8        5  256  16  65573   8  8

Tolerances are per element and derived from the arithmetic (EPS = 2^-24): an fp32 sum of n terms is within (n - 1) EPS
of the sum of the absolute terms; the soft-max of logits of size A (after / T) is within (10 A + E + 8) EPS relative.
Sums over the batch go through one lane's laps, the CTA's 8 warps and one atomic per CTA, so their chain is
laps + 8 + CTAs long.  Output buffers carry NaN guard rows past the batch and NaN guard columns beside every strided
view; they must stay NaN."""
import pytest
import torch

from models_b200 import ops
from tests.mmoe_oracle import BCE, MSE, gate_mix, heads_loss
from tests.test_gpu_train_scale import BIG, GUARD, RAGGED, _nan, _sms, _untouched, _within

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -24
WARPS = 8  # warps (samples in flight) per CTA of every MMoE kernel

CASES = [(1, 7, 4, 37, "split"), (1, 64, 16, 1001, "view"), (1, 100, 1, 1001, "split"), (1, 256, 4, BIG, "view"),
         (2, 32, 1, 1001, "view"), (2, 33, 4, 37, "split"), (2, 128, 16, RAGGED, "view"), (2, 129, 4, 1001, "split"),
         (3, 32, 16, BIG, "view"), (4, 64, 4, 1001, "split"), (3, 100, 4, 37, "view"), (4, 256, 1, 1001, "split"),
         (5, 7, 4, 1001, "view"), (8, 33, 16, 1001, "split"), (8, 128, 4, BIG, "split"), (5, 256, 16, RAGGED, "view")]
TEMPS = (0.5, 1.0, 1.7)


def _id(c):
    return "H{}-U{}-E{}-B{}-{}".format(*c)


def _dispatch(H, n):
    """(NH, C) as MM_MOE_DISPATCH in mmoe.cu picks them."""
    return (1 if H == 1 else 2 if H == 2 else 4 if H <= 4 else 8), (1 if n <= 32 else 2 if n <= 64 else 4 if n <= 128 else 8)


def _grid(B, device):
    """(CTAs, laps, chain) of grid_for in mmoe.cu: chain is the longest sequence of fp32 additions of a batch sum."""
    ctas = min(-(-B // WARPS), 4 * _sms(device))
    laps = -(-B // (WARPS * ctas))
    if B >= BIG:
        assert laps >= 2 and B % (WARPS * ctas), f"premise: B = {B} gives {laps} lap(s) of {ctas} CTAs x {WARPS} warps, not ragged"
    return ctas, laps, laps + WARPS + ctas


def _gate_views(L, H, E):
    """Column t E .. (t + 1) E of the stacked (B, H E) gate logits for each task: the strided views MMOEBlock.gate_logits
    hands the kernels."""
    return [L[:, t * E:(t + 1) * E] for t in range(H)]


def _gates(L, H, E, form):
    """The H (B, E) gate-logit matrices: separate contiguous tensors, or column views of one stacked matrix."""
    views = _gate_views(L, H, E)
    return views if form == "view" else [v.contiguous() for v in views]


def _inputs(device, H, U, E, B, relu, seed):
    g = torch.Generator(device=device).manual_seed(seed)
    X = torch.randn((B, E * U), generator=g, device=device)
    if relu:
        X = X.clamp_min(0)  # the experts' relu outputs: about half exactly 0
    L = torch.randn((B, H * E), generator=g, device=device) * 2
    return g, X, L


def _softmax_ref(L, H, E, T):
    """float64 gate weights (B, H, E) and their relative bound (B, H, 1)."""
    a = L.double().reshape(-1, H, E) / T
    A = a.abs().amax(2, keepdim=True)
    return torch.softmax(a, 2), (10 * A + E + 8) * EPS


def _mix_forward(X, E, gl, T, B, H, U):
    """mm_mmoe_mix_fwd into NaN-filled buffers with guard rows: (p, m, m_split) and the buffers."""
    dev = X.device
    Kp = ops.tc_padded_k(U)
    P = _nan((B + GUARD, H * E), dev)
    Mf = _nan((H * B * U + GUARD * U,), dev)
    Sf = torch.full((H * B * 2 * Kp + GUARD,), float("nan"), dtype=torch.bfloat16, device=dev)
    p, m, ms = P[:B], Mf[:H * B * U].view(H, B, U), Sf[:H * B * 2 * Kp].view(H, B, 2 * Kp)
    ops.mmoe_mix_fwd(X, E, gl, T, p, m, ms)
    return p, m, ms, (P, Mf, Sf)


# ---------------------------------------------------------------------------------------------------------------
# mm_mmoe_mix_fwd
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=_id)
def test_mix_forward_matches_float64(device, case):
    """p against softmax(L_t / T), m_t against sum_e p_t,e X_e (bound (rel_p + (E + 2) EPS) sum_e p |X_e|), m_split
    bit-identical to mm_split_rows of the kernel's own m, its padding columns U..Kp exactly 0."""
    H, U, E, B, form = case
    T = TEMPS[CASES.index(case) % 3]
    _grid(B, device)
    _, X, L = _inputs(device, H, U, E, B, False, 7 * CASES.index(case))
    p, m, ms, (P, Mf, Sf) = _mix_forward(X, E, _gates(L, H, E, form), T, B, H, U)
    torch.cuda.synchronize()
    pr, rel = _softmax_ref(L, H, E, T)
    _within(p.reshape(B, H, E), pr, rel * pr + 1e-300, "p")
    X64 = X.double()
    for t in range(H):
        Lt = L[:, t * E:(t + 1) * E].double()
        mr = gate_mix(X64, Lt, E, T)
        bound = (rel[:, t] + (E + 2) * EPS) * gate_mix(X64.abs(), Lt, E, T)
        _within(m[t], mr, bound, f"m[{t}]")
    Kp = ops.tc_padded_k(U)
    for t in range(H):
        assert torch.equal(ms[t].view(torch.int16), ops.split_rows(m[t]).view(torch.int16)), f"m_split[{t}] != split_rows(m[{t}])"
    if Kp > U:
        pad = torch.cat([ms[:, :, U:Kp], ms[:, :, Kp + U:]], 2)
        assert bool((pad.view(torch.int16) == 0).all()), "m_split padding columns U..Kp are not +0"
    _untouched(P, B, H * E, "p")
    assert bool(torch.isnan(Mf[H * B * U:]).all()) and bool(torch.isnan(Sf[H * B * 2 * Kp:].float()).all()), "m / m_split guard written"


# ---------------------------------------------------------------------------------------------------------------
# mm_mmoe_mix_bwd
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "linear"])
@pytest.mark.parametrize("case", CASES, ids=_id)
def test_mix_backward_matches_float64(device, case, relu):
    """dX and dL of a random dm against float64 autograd of sum_t <m_t, dm_t>, dX and the gate-logit gradients written
    as column blocks of one NaN-filled G buffer (as MMoETrainer passes them).  Bounds: dX_e within
    sum_t (rel_p_t + (H + 1) EPS) p_t,e |dm_t|; dL_t,e within 2 p_t,e / T (rel_p_t + (U + E + 8) EPS) (a_e + sum_e p a_e)
    with a_e = sum_k |dm_t,k X_e,k|, which a lost 1 / T factor at T != 1 exceeds by orders of magnitude."""
    H, U, E, B, form = case
    T = TEMPS[CASES.index(case) % 3]
    _grid(B, device)
    g, X, L = _inputs(device, H, U, E, B, relu, 7 * CASES.index(case) + relu)
    p, _, _, _ = _mix_forward(X, E, _gates(L, H, E, form), T, B, H, U)
    dm = torch.randn((H, B, U), generator=g, device=device)
    EU = E * U
    G = _nan((B + GUARD, EU + H * E + 3), device)
    dX = G[:B, :EU]
    dgl = [G[:B, EU + t * E:EU + (t + 1) * E] for t in range(H)]
    ops.mmoe_mix_bwd(X, E, p, T, dm, dX, dgl, mask_relu=relu)
    torch.cuda.synchronize()
    Xd = X.double().requires_grad_(True)
    Ld = L.double().requires_grad_(True)
    dm64 = dm.double()
    obj = sum((gate_mix(Xd, Ld[:, t * E:(t + 1) * E], E, T) * dm64[t]).sum() for t in range(H))
    obj.backward()
    dX_ref = Xd.grad * (X > 0) if relu else Xd.grad
    pr, rel = _softmax_ref(L, H, E, T)  # (B, H, E), (B, H, 1)
    adm = dm64.abs()
    bx = torch.einsum("bte,tbu->beu", (rel + (H + 1) * EPS) * pr, adm).reshape(B, EU)
    _within(dX, dX_ref, bx, "dX")
    X3 = X.double().abs().reshape(B, E, U)
    for t in range(H):
        a = torch.einsum("bu,beu->be", adm[t], X3)
        A = (pr[:, t] * a).sum(1, keepdim=True)
        bound = 2 * pr[:, t] / T * (rel[:, t] + (U + E + 8) * EPS) * (a + A) + 1e-300
        _within(dgl[t], Ld.grad[:, t * E:(t + 1) * E], bound, f"dL[{t}]")
    _untouched(G, B, EU + H * E, "G")


# ---------------------------------------------------------------------------------------------------------------
# mm_mmoe_task_heads_fwd_bwd and mm_mmoe_heads_fwd_bwd: the loss side
# ---------------------------------------------------------------------------------------------------------------
def _targets(g, H, B, device):
    """BCE / MSE heads alternating; targets int64, int32, float32 in turn; sample weights on two of every three tasks
    (None on the rest); loss weights 0.5 + 0.25 t."""
    losses = [(BCE, MSE)[t % 2] for t in range(H)]
    ys = []
    for t, l in enumerate(losses):
        v = (torch.rand(B, generator=g, device=device) < 0.4).double() if l == BCE else \
            torch.randint(-2, 3, (B,), generator=g, device=device).double() if t % 3 != 2 else torch.randn(B, generator=g, device=device).double()
        ys.append(v.to((torch.int64, torch.int32, torch.float32)[t % 3]))
    sws = [None if t % 3 == 1 else torch.rand(B, generator=g, device=device) * 2 for t in range(H)]
    lws = [0.5 + 0.25 * t for t in range(H)]
    return losses, ys, sws, lws


def _loss_bounds(zs, ez, losses, ys, sws, lws, B, chain):
    """Per task: (dz, its bound, loss bound); and the total loss's bound, for float64 logits zs with bounds ez."""
    out, total = [], 0.0
    for z, e, l, y, sw, lw in zip(zs, ez, losses, ys, sws, lws):
        y = y.double()
        s = sw.double() if sw is not None else torch.ones_like(z)
        if l == BCE:
            lt, gt, cz = z.clamp_min(0) - z * y + torch.log1p(torch.exp(-z.abs())), torch.sigmoid(z) - y, 0.25
        else:
            lt, gt, cz = (z - y) ** 2, 2 * (z - y), 2.0
        dz = gt * s * lw / B
        edz = s * abs(lw) / B * (cz * e + 8 * EPS * (gt.abs() + 1))
        el = float((s / B * (gt.abs() * e + 4 * EPS * (lt.abs() + z.abs() + 1))).sum() + chain * EPS * (s * lt.abs()).sum() / B)
        out.append((dz, edz, el))
        total += abs(lw) * (el + len(zs) * chain * EPS * float((s * lt.abs()).sum()) / B)  # H atomics per CTA into the total
    return out, total


def _check_losses(loss, per, terms, total_bound):
    _within(loss[0], per[0].detach(), torch.tensor(total_bound, dtype=torch.float64, device=loss.device), "total loss")
    for t, (_, _, el) in enumerate(terms):
        _within(loss[1 + t], per[1][t].detach(), torch.tensor(el, dtype=torch.float64, device=loss.device), f"loss[{t}]")


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_task_heads_match_float64(device, case):
    """H Dense(K -> 1) heads, head t reading its own strided input x_t (K = the case's U): logits, [total, loss_t] with
    loss weights, dx_t (relu mask on in half the cases) as column blocks of a NaN-filled buffer with a guard column after
    each, dw and db; then the forward alone (null targets) against sigmoid / identity.  Bounds: z within
    (K + 2) EPS (sum |x w| + |b|); dz from it through the loss; dw, db and the losses along the batch-sum chain."""
    H, K, _, B, _ = case
    relu = CASES.index(case) % 2 == 0
    ctas, laps, chain = _grid(B, device)
    g = torch.Generator(device=device).manual_seed(7 * CASES.index(case) + 3)
    Xall = torch.randn((B, H * (K + 1)), generator=g, device=device)
    if relu:
        Xall = Xall.clamp_min(0)
    xs = [Xall[:, t * (K + 1):t * (K + 1) + K] for t in range(H)]
    W = torch.randn((K, H), generator=g, device=device) * 0.2
    b = torch.randn(H, generator=g, device=device) * 0.1
    losses, ys, sws, lws = _targets(g, H, B, device)
    D = _nan((B + GUARD, H * (K + 1)), device)
    dxs = [D[:B, t * (K + 1):t * (K + 1) + K] for t in range(H)]
    Z = _nan((H, B + GUARD), device)
    z = Z.view(-1)[:H * B].view(H, B)
    loss = torch.zeros(1 + H, device=device)
    dW, db = torch.zeros((K, H), device=device), torch.zeros(H, device=device)
    ops.mmoe_task_heads_fwd_bwd(xs, W, b, losses, ys, z, loss, dxs, dW, db, loss_weights=lws, mask_relu=relu, sample_weight=sws)
    torch.cuda.synchronize()
    x64 = [x.double().requires_grad_(True) for x in xs]
    W64, b64 = W.double().requires_grad_(True), b.double().requires_grad_(True)
    zr = [x64[t] @ W64[:, t] + b64[t] for t in range(H)]
    per = heads_loss(zr, losses, ys, lws, sws)
    per[0].backward()
    ez = [(K + 2) * EPS * (xs[t].double().abs() @ W[:, t].double().abs() + float(b[t].abs())) for t in range(H)]
    terms, tb = _loss_bounds([zz.detach() for zz in zr], ez, losses, ys, sws, lws, B, chain)
    for t in range(H):
        _within(z[t], zr[t].detach(), ez[t], f"z[{t}]")
    _check_losses(loss, per, terms, tb)
    for t, (dz, edz, _) in enumerate(terms):
        ref = x64[t].grad * (xs[t] > 0) if relu else x64[t].grad
        w_ = W[:, t].double().abs()
        _within(dxs[t], ref, edz[:, None] * w_[None, :] + 2 * EPS * (dz.abs()[:, None] * w_[None, :]), f"dx[{t}]")
        ax = xs[t].double().abs()
        _within(dW[:, t], W64.grad[:, t], ax.t() @ edz + chain * EPS * (ax.t() @ dz.abs()), f"dw[:, {t}]")
        _within(db[t], b64.grad[t], edz.sum() + chain * EPS * dz.abs().sum(), f"db[{t}]")
    _untouched(D, B, H * (K + 1) - 1, "dx buffer")
    for t in range(H):
        assert bool(torch.isnan(D[:B, t * (K + 1) + K]).all()), f"the guard column after dx[{t}] was written"
    assert bool(torch.isnan(Z.view(-1)[H * B:]).all()), "a logit past H B was written"
    # forward only: the activated predictions
    Pd = _nan((H * B + GUARD,), device)
    pred = Pd[:H * B].view(H, B)
    ops.mmoe_task_heads_fwd_bwd(xs, W, b, losses, None, pred)
    assert bool(torch.isnan(Pd[H * B:]).all()), "a prediction past H B was written"
    for t in range(H):
        zt = zr[t].detach()
        ref, bound = (torch.sigmoid(zt), ez[t] / 4 + 4 * EPS) if losses[t] == BCE else (zt, ez[t])
        _within(pred[t], ref, bound, f"prediction[{t}]")


@pytest.mark.parametrize("B,E,U,H,T", [(1001, 4, 100, 3, 1.7), (RAGGED, 4, 128, 2, 0.5), (37, 16, 128, 5, 1.0),
                                       (1001, 1, 64, 3, 1.0), (BIG, 1, 100, 1, 0.5), (37, 1, 256, 8, 1.7)])
def test_fused_heads_at_four_columns_and_one_expert(device, B, E, U, H, T):
    """mm_mmoe_heads_fwd_bwd at C = 4 (65 <= U <= 128) and E = 1, per element: z within the mixture's bound carried
    through w plus the dot's; dX_e = sum_t p_t,e dz_t w_t; dL_t,e = p (dz <w_t, X_e> - s) / T; dW = sum_b m dz; the
    losses and db as the task heads.  With one expert the gate weight is exactly 1, so dL must be exactly 0 and z is the
    expert's own head."""
    ctas, laps, chain = _grid(B, device)
    g, X, L = _inputs(device, H, U, E, B, True, B + E + U)
    W = torch.randn((U, H), generator=g, device=device) * 0.2
    b = torch.randn(H, generator=g, device=device) * 0.1
    losses, ys, sws, lws = _targets(g, H, B, device)
    EU = E * U
    Gb = _nan((B + GUARD, EU + H * E + 3), device)
    dX, dgl = Gb[:B, :EU], [Gb[:B, EU + t * E:EU + (t + 1) * E] for t in range(H)]
    Z = _nan((H * B + GUARD,), device)
    z = Z[:H * B].view(H, B)
    loss = torch.zeros(1 + H, device=device)
    dW, db = torch.zeros((U, H), device=device), torch.zeros(H, device=device)
    gl = _gate_views(L, H, E)
    ops.mmoe_heads_fwd_bwd(X, E, gl, T, W, b, losses, ys, z, loss, dx=dX, d_gate_logits=dgl, dw=dW, db=db, loss_weights=lws,
                           mask_relu=True, sample_weight=sws)
    torch.cuda.synchronize()
    Xd, Ld = X.double().requires_grad_(True), L.double().requires_grad_(True)
    W64, b64 = W.double().requires_grad_(True), b.double().requires_grad_(True)
    ms = [gate_mix(Xd, Ld[:, t * E:(t + 1) * E], E, T) for t in range(H)]
    zr = [ms[t] @ W64[:, t] + b64[t] for t in range(H)]
    per = heads_loss(zr, losses, ys, lws, sws)
    per[0].backward()
    pr, rel = _softmax_ref(L, H, E, T)
    X64 = X.double()
    X3 = X64.abs().reshape(B, E, U)
    aw = W.double().abs()
    em = [(rel[:, t] + (E + 2) * EPS) * gate_mix(X64.abs(), L[:, t * E:(t + 1) * E].double(), E, T) for t in range(H)]
    ez = [em[t] @ aw[:, t] + (U + 2) * EPS * (ms[t].detach().abs() @ aw[:, t] + float(b[t].abs())) for t in range(H)]
    terms, tb = _loss_bounds([zz.detach() for zz in zr], ez, losses, ys, sws, lws, B, chain)
    for t in range(H):
        _within(z[t], zr[t].detach(), ez[t], f"z[{t}]")
    _check_losses(loss, per, terms, tb)
    bx = torch.zeros((B, E, U), dtype=torch.float64, device=device)
    for t, (dz, edz, _) in enumerate(terms):
        c = pr[:, t] * (edz + dz.abs() * (rel[:, t, 0] + (H + 2) * EPS))[:, None]  # (B, E)
        bx += c[:, :, None] * aw[None, None, :, t]
        a = torch.einsum("u,beu->be", aw[:, t], X3)  # |<w_t, X_e>| bound
        A = (pr[:, t] * a).sum(1, keepdim=True)
        bl = 2 * pr[:, t] / T * ((rel[:, t] + (U + E + 8) * EPS) * dz.abs()[:, None] + edz[:, None]) * (a + A) + 1e-300
        _within(dgl[t], Ld.grad[:, t * E:(t + 1) * E], bl, f"dL[{t}]")
        if E == 1:
            assert bool((dgl[t] == 0).all()), f"dL[{t}] with one expert must be exactly 0"
        am = ms[t].detach().abs()
        _within(dW[:, t], W64.grad[:, t], am.t() @ edz + em[t].t() @ dz.abs() + chain * EPS * (am.t() @ dz.abs()), f"dw[:, {t}]")
        _within(db[t], b64.grad[t], edz.sum() + chain * EPS * dz.abs().sum(), f"db[{t}]")
    _within(dX, Xd.grad * (X > 0), bx.reshape(B, EU), "dX")
    _untouched(Gb, B, EU + H * E, "G")
    if E == 1:  # the mixture is the expert itself: z is the expert's head, to the dot's own rounding
        for t in range(H):
            zx = X64 @ W[:, t].double() + float(b[t])
            _within(z[t], zx, (U + 2) * EPS * (X64.abs() @ aw[:, t] + float(b[t].abs())), f"z[{t}] vs the expert's head")
    assert bool(torch.isnan(Z[H * B:]).all()), "a logit past H B was written"
    Pd = _nan((H * B + GUARD,), device)
    pred = Pd[:H * B].view(H, B)
    ops.mmoe_heads_fwd_bwd(X, E, gl, T, W, b, losses, None, pred)
    assert bool(torch.isnan(Pd[H * B:]).all()), "a prediction past H B was written"
    for t in range(H):
        zt = zr[t].detach()
        ref, bound = (torch.sigmoid(zt), ez[t] / 4 + 4 * EPS) if losses[t] == BCE else (zt, ez[t])
        _within(pred[t], ref, bound, f"prediction[{t}]")
