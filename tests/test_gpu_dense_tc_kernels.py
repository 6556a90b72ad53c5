"""mm_dense_tc, the general tensor-core GEMM, at every variant dense_tc_launch (models_b200/csrc/dense_tc.cu) dispatches:
the tile width BN (one wgmma instruction per BN in 16, 32, ..., 128), the ring depth (2..5 stages, from BN and Kp), the
interleaved or resident-A schedule, every epilogue (seven activations, the DCN-v2 cross with vector or scalar x0 / x
loads, the fused Dense(N -> 1) head, the in-batch scorer with no / narrow / wide id mask, logQ and temperature) and every
store (fp32 rows through interior vector, edge vector or scalar stores; the split-bf16 operand of the next layer with
or without its padding gap).  `plan` and `fp32_paths` restate the launcher; tests/test_dense_tc_host.py pins them to
the library and checks, without a GPU, that the case tables below reach every variant.

Each case makes one call and compares EVERY output element with float64 computed on the device, within a bound derived
from the arithmetic (conventions of test_gpu_train_scale and test_gpu_forward_scale, E = 2^-24):
  * one 3-pass split-bf16 product is within UNIT = 3 * 2^-16 of |a b|: a = hi + lo leaves at most 2^-8 * 2^-8 of |a|
    (bf16 rounds within 2^-8), as does b, and lo * lo is dropped.  The 2^-16 of the other modules holds for long dot
    products, where these errors do not line up, but a K = 1 GEMM reaches 1.6 * 2^-16.  A passes = 1 (plain bf16)
    product is within 2 * 2^-8 + 2^-16.  An fp32 sum of n terms is within n E sum |terms|.  So the pre-activation
    z = x W + b is within (unit + K E) (|x| @ |W| + |b|) (_chain);
  * the activation carries that error in through its Lipschitz constant L and adds its own rounding (_act):
      relu, linear: L = 1, exact;
      sigmoid  1 / (1 + expf(-v)): L = 1/4; expf within 2 ulp (4 E relative), one add, one division: under 8 E |y|;
      tanh     tanhf within 2 ulp: L = 1, 4 E |y|;
      elu      v or expm1f(v), expm1f within 1 ulp: L = 1, 2 E |y|;
      selu     scale v or (scale alpha) expm1f(v): L = scale alpha = 1.7581 < 1.76; the two fp32 constants (E each),
               their folded product (E), expm1f (2 E) and the final product (E): 6 E |y|, taken as 8 E |y|;
      gelu     0.5 v (1 + erff(v c)), c = fp32(1/sqrt 2): L = max gelu' = 1.1289 < 1.13; v c within 2 E relative moves
               erf by at most 2/sqrt(pi) e^(-v^2/2) 2 E |v| / sqrt 2 < E, erff within 2 ulp (2 E absolute near +-1),
               1 + erf rounds (2 E): 1 + erf within 5 E absolute, so y within 0.5 |v| 5 E + E |y| < 4 E |v| + E |y|;
    each own rounding is taken at the device's pre-activation, |z| + ez and |y| + L ez;
  * the cross epilogue x0 * (x W + b) + x: |x0| times the GEMM bound, then one rounded product and one rounded sum;
  * the head: an fp32 dot of N terms plus head_b (N E of the absolute terms), then head_act as above;
  * the scorer as test_gpu_forward_scale's test_inbatch_scorer_at_scale, with UNIT; a masked entry is fl(fns / T) bit
    for bit;
  * a split-bf16 output hi + lo adds at most 2^-16 of the value; with out_f32 as well it is split_rows(out_f32) bit for
    bit, and its padding columns up to Kp(N) are exact zeros.
A wrong wgmma width, a dropped bias chunk, a wrong activation constant, a lost head bias, a wrong store path or a flipped
logQ moves an element by O(1) of its scale, far above these bounds.

The data has rows of exact zeros (with a bias that is zero in every third column, the pre-activation is exactly 0:
relu's mask), rows scaled by 40 (sigmoid and tanh saturate, selu / elu / gelu reach their negative tails) and values on
both sides of 0.  Every fp32 output is a view of a NaN buffer with guard rows past M and guard columns beside the view,
and every split output a view of a NaN buffer with guard rows; nothing outside the output may be written."""
from collections import namedtuple

import pytest
import torch

from models_b200 import _cabi, ops
from tests.test_gpu_forward_scale import SPLIT, _chain, _dense_tc_laps, _nan_bf16, _scorer_schedule, _split_padding_zero, _unsplit
from tests.test_gpu_train_scale import E, GUARD, U, _nan, _sms, _untouched, _within

pytestmark = pytest.mark.gpu
ACTS = ("linear", "relu", "sigmoid", "tanh", "selu", "elu", "gelu")
UNIT = 3 * U  # relative error of one 3-pass split-bf16 product
BF16_UNIT = 2 * 2.0 ** -8 + 2.0 ** -16  # relative error of one passes = 1 product
SMEM = 227 * 1024
FNS = -655.04  # false-negative score of the scorer
SMS = 132  # SMs of an H100 SXM: the lap cases are sized for it (and asserted on the device's own count)

# fp32 output layouts: (first column of the view in its row, row stride) for N columns
LAYOUTS = ("dense", "vec", "odd", "off1")


def _c4(n):
    return (n + 3) // 4 * 4


def layout_of(layout, N):
    """dense: contiguous (M, N); vec: columns 4..4+N of rows of 4k floats (16-byte aligned); odd: columns 2..2+N of
    rows of 4k + 1 floats; off1: columns 1..1+N of rows of 4k floats (4-byte aligned)."""
    return {"dense": (0, N), "vec": (4, _c4(N) + 8), "odd": (2, _c4(N) + 5), "off1": (1, _c4(N) + 8)}[layout]


# ---------------------------------------------------------------------------------------------------------------
# the launcher, restated
# ---------------------------------------------------------------------------------------------------------------
def padded_k(K):
    return (K + 63) // 64 * 64


def padded_n(N):
    return (N + 15) // 16 * 16 if N <= 128 else (N + 127) // 128 * 128


def plan(M, K, N, score=False, sms=SMS):
    """dense_tc_launch's choices (passes 3 or 1 alike, except the resident schedule, which only the 3-pass scorer
    takes): tile width BN, n-tiles, ring depth, schedule, tiles per CTA and CTAs."""
    Kp, Np = padded_k(K), padded_n(N)
    BN = min(Np, 128)
    ntn, KB = Np // BN, Kp // 64
    resident = score and Kp <= 128 and ntn >= 8
    a_res = KB * 2 * 16384 if resident else 0
    stage = (0 if resident else 2 * 16384) + 2 * BN * 64 * 2
    image = 128 * ((BN + 31) // 32 * 32 + 4) * 4
    fixed = 1024 + a_res + image + 16 * 8 + 256 * 8 + 256 * 4
    stages = min((SMEM - fixed) // stage, 6)
    if not resident:
        stages = min(stages, 2 * KB)
    tiles = -(-M // 128) * ntn
    grid = min(tiles, sms)
    tpc = -(-tiles // grid) if tiles else 0
    if resident and tiles:
        grid = -(-tiles // tpc)
    return dict(Kp=Kp, Np=Np, BN=BN, n_tiles_n=ntn, KB=KB, stages=stages, resident=resident, tiles=tiles, grid=grid,
                tiles_per_cta=tpc)


def fp32_paths(M, N, stride, col):
    """The fp32 store paths a call takes (rows 16-byte aligned at column 0): interior / edge vector stores when the row
    stride and the first column are multiples of 4 floats, scalar stores otherwise."""
    if stride % 4 or col % 4:
        return {"scalar"}
    paths = set()
    if M >= 32 and N >= 32:
        paths.add("interior")  # some 32 x 32 chunk lies wholly inside the output
    if M % 32 or N % 32:
        paths.add("edge")
    return paths


def split_gap(N):
    """True when the split output has padding columns [Np, Kp(N)) past the single n-tile."""
    return padded_n(N) < padded_k(N)


# ---------------------------------------------------------------------------------------------------------------
# case tables (importable without CUDA)
# ---------------------------------------------------------------------------------------------------------------
Dense = namedtuple("Dense", "M K N act bias out layout passes")
Cross = namedtuple("Cross", "M d layout out")
Head = namedtuple("Head", "M K N act bias head_act")
Scorer = namedtuple("Scorer", "B N D T logq ids layout")

# N: two widths per tile width BN (16 .. 128), mostly not multiples of 16 or 4, then several n-tiles with a partial last
NS = (1, 7, 17, 30, 33, 47, 50, 63, 65, 79, 83, 90, 100, 111, 113, 128, 129, 272, 1037)
# K by k-blocks: one (ring depth 2), two (depth min(4, cap)), three or more (the cap; K >= 415 wraps the ring in a tile)
K_BY_KB = ((1, 13, 64), (65, 128), (129, 415, 1037))
MS = (1, 127, 128, 129, 1001)
OUTS = ("f32", "split", "both")

DENSE = []
for _i, _N in enumerate(NS):
    for _j, _ks in enumerate(K_BY_KB):
        _t = 3 * _i + _j
        DENSE.append(Dense(MS[_t % 5], _ks[(_i + _j) % len(_ks)], _N, ACTS[_t % 7], (_t // 7) % 2 == 0, OUTS[(_i + 2 * _j) % 3],
                           LAYOUTS[(_i + _j) % 4], 3))
DENSE += [
    # the interleaved schedule over 3 laps with a ragged last one (300 and 303 tiles on 132 SMs)
    Dense(300 * 128 - 37, 64, 100, "gelu", True, "both", "vec", 3),
    Dense(101 * 128 - 123, 415, 272, "tanh", True, "both", "odd", 3),
    # passes = 1 (plain bf16)
    Dense(1001, 415, 100, "relu", True, "both", "vec", 1),
    Dense(129, 1037, 272, "selu", False, "f32", "off1", 1),
    Dense(128, 64, 1, "sigmoid", True, "f32", "dense", 1),
]

CROSS = [
    Cross(1001, 33, "vec", "both"), Cross(129, 33, "odd", "f32"), Cross(128, 100, "off1", "both"),
    Cross(1001, 100, "vec", "split"), Cross(127, 128, "vec", "f32"), Cross(1001, 272, "odd", "both"),
    Cross(129, 1037, "vec", "both"), Cross(1001, 1037, "off1", "f32"), Cross(1, 64, "odd", "split"),
]

# every head activation at BN = 16 and BN = 32, with and without the layer's bias
HEAD = []
for _i, _ha in enumerate(ACTS):
    HEAD.append(Head((1001, 129, 127, 1)[_i % 4], (13, 129, 415, 64)[_i % 4], (1, 9, 16)[_i % 3], ACTS[(_i + 3) % 7], _i % 2 == 0, _ha))
    HEAD.append(Head((129, 1001, 1, 128)[_i % 4], (64, 1037, 65, 128)[_i % 4], (17, 24, 32)[_i % 3], ACTS[(_i + 5) % 7], _i % 2 == 1, _ha))

# N = 896 (7 n-tiles: resident schedule off) and 897 (8: on when D <= 128); ids None (no mask), "i32", "narrow" (int64
# below 2^32) or "wide" (int64, some above 2^32 sharing low words); layout "model": column 1 of (B, 1 + N) rows at
# stride N + 4 (scalar stores), "bench": column 4 (vector stores)
SCORER = [
    Scorer(1001, 897, 64, 0.05, True, "wide", "model"), Scorer(1001, 896, 64, 1.0, False, "i32", "model"),
    Scorer(300, 897, 128, 1.0, True, "narrow", "model"), Scorer(300, 896, 128, 0.05, True, "wide", "model"),
    Scorer(129, 897, 192, 0.05, False, "narrow", "model"), Scorer(129, 896, 192, 1.0, True, None, "model"),
    Scorer(1, 897, 64, 1.0, False, None, "model"), Scorer(127, 896, 128, 1.0, False, "narrow", "bench"),
    # the resident schedule over 3 tiles per CTA, the last CTA's range short (320 tiles)
    Scorer(40 * 128 - 11, 897, 64, 0.05, True, "i32", "model"),
]


def dense_id(c):
    return f"M{c.M}-K{c.K}-N{c.N}-{c.act}-{'b' if c.bias else 'nb'}-{c.out}-{c.layout}-p{c.passes}"


def scorer_out(B, N, layout):
    """(first column of the (B, 1 + N) view, row stride) of the scorer's output buffer."""
    return (0 if layout == "model" else 3), N + 4


# ---------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------
def _inputs(M, K, N, bias, seed, device):
    """x (M, K) with rows of exact zeros (every 7th) and rows scaled by 40 (every 5th), W (K, N) / sqrt(K), and the
    bias (N,) zero in every third column."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn((M, K), generator=g, device=device)
    r = torch.arange(M, device=device)
    x[r % 7 == 3] = 0.0
    x[r % 5 == 1] *= 40.0
    W = torch.randn((K, N), generator=g, device=device) / K ** 0.5
    b = None
    if bias:
        b = torch.randn(N, generator=g, device=device) * 0.5
        b[1::3] = 0.0
    return x, W, b


def _f32_out(M, N, layout, device):
    """(NaN buffer, (M, N) view, first column) in the given layout."""
    c, stride = layout_of(layout, N)
    buf = _nan((M + GUARD, stride), device)
    return buf, buf[:M, c:c + N], c


def _f32_untouched(buf, M, c, N, what):
    _untouched(buf[:, c:], M, N, what)
    assert bool(torch.isnan(buf[:, :c]).all()), f"{what}: a guard column before the output was written"


def _check_split(sb, M, N, y, ey, f32, what):
    """Rows >= M of the NaN buffer untouched, padding columns up to Kp(N) zero, and hi + lo within the bound of y or
    (with f32) split_rows(f32) bit for bit."""
    _split_padding_zero(sb, M, N, what)
    if f32 is not None:
        assert torch.equal(sb[:M], ops.split_rows(f32)), f"{what}: not split_rows(out_f32) bit for bit"
    else:
        _within(_unsplit(sb[:M], N), y, ey + SPLIT * (y.abs() + ey), what)


# ---------------------------------------------------------------------------------------------------------------
# 1. act(x W + b): every tile width, ring depth, activation and store path
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", DENSE, ids=dense_id)
def test_dense_tc_matches_float64(device, c):
    p = plan(c.M, c.K, c.N, sms=_sms(device))
    if c.M > 1001:
        laps = _dense_tc_laps(c.M, c.N, _sms(device))
        assert laps >= 3 and p["tiles"] % p["grid"], f"premise: {p['tiles']} tiles give {laps} lap(s) on {p['grid']} CTAs"
    x, W, b = _inputs(c.M, c.K, c.N, c.bias, DENSE.index(c), device)
    fb = fv = sb = None
    if c.out in ("f32", "both"):
        fb, fv, col = _f32_out(c.M, c.N, c.layout, device)
    Kp = ops.tc_padded_k(c.N)
    if c.out in ("split", "both"):
        sb = _nan_bf16((c.M + GUARD, 2 * Kp), device)
    ops.dense_tc(ops.split_rows(x), c.K, ops.split_weights(W), c.N, b, c.act, passes=c.passes, out_f32=fv,
                 out_split=None if sb is None else sb[:c.M])
    y, ey = _chain(x.double(), [(W, b, c.act)], unit=UNIT if c.passes == 3 else BF16_UNIT)
    if fv is not None:
        _f32_untouched(fb, c.M, col, c.N, "out_f32")
        _within(fv, y, ey, f"out_f32 ({c.act})")
    if sb is not None:
        _check_split(sb, c.M, c.N, y, ey, fv, "out_split")


# ---------------------------------------------------------------------------------------------------------------
# 2. the DCN-v2 cross epilogue x0 * (x W + b) + x
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", CROSS, ids=lambda c: f"M{c.M}-d{c.d}-{c.layout}-{c.out}")
def test_dense_tc_cross_matches_float64(device, c):
    """x0 and x are (M, d) views of NaN buffers in the case's layout (vector loads for "vec", scalar otherwise); the
    fp32 output takes the same layout.  Bound |x0| (UNIT + d E) (|x| @ |W| + |b|) + E (|x0 z| + |x|)."""
    M, d = c.M, c.d
    x, W, b = _inputs(M, d, d, True, 1000 + CROSS.index(c), device)
    x0 = torch.randn((M, d), generator=torch.Generator(device=device).manual_seed(d), device=device)
    views = []
    for v in (x0, x):
        buf, view, _ = _f32_out(M, d, c.layout, device)
        view.copy_(v)
        views.append(view)
    fb = fv = sb = None
    if c.out in ("f32", "both"):
        fb, fv, col = _f32_out(M, d, c.layout, device)
    if c.out in ("split", "both"):
        sb = _nan_bf16((M + GUARD, 2 * ops.tc_padded_k(d)), device)
    ops.dense_tc(ops.split_rows(x), d, ops.split_weights(W), d, b, None, out_f32=fv, out_split=None if sb is None else sb[:M],
                 x0=views[0], xres=views[1])
    xd, x0d, Wd, bd = x.double(), x0.double(), W.double(), b.double()
    z = xd @ Wd + bd
    y = x0d * z + xd
    ey = x0d.abs() * (UNIT + d * E) * (xd.abs() @ Wd.abs() + bd.abs()) + E * ((x0d * z).abs() + xd.abs())
    if fv is not None:
        _f32_untouched(fb, M, col, d, "cross out_f32")
        _within(fv, y, ey, "cross out_f32")
    if sb is not None:
        _check_split(sb, M, d, y, ey, fv, "cross out_split")


# ---------------------------------------------------------------------------------------------------------------
# 3. mm_dense_tc_head: the layer and a fused Dense(N -> 1)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", HEAD, ids=lambda c: f"M{c.M}-K{c.K}-N{c.N}-{c.act}-{'b' if c.bias else 'nb'}-head_{c.head_act}")
def test_dense_tc_head_matches_float64(device, c):
    """head_out[m] = head_act(act(x W + b)[m] . head_w + head_b) into M values of a NaN buffer with guards past M; the
    layer's bound from _chain, the head's as one more layer with fp32 products (unit 0)."""
    x, W, b = _inputs(c.M, c.K, c.N, c.bias, 2000 + HEAD.index(c), device)
    g = torch.Generator(device=device).manual_seed(c.N)
    hw = torch.randn(c.N, generator=g, device=device) / c.N ** 0.5
    hb = -0.375
    hbuf = _nan((c.M + GUARD,), device)
    ops.dense_tc_head(ops.split_rows(x), c.K, ops.split_weights(W), c.N, b, c.act, hw, hb, c.head_act, hbuf[:c.M])
    assert bool(torch.isnan(hbuf[c.M:]).all()), "head: a guard element past M was written"
    h, eh = _chain(x.double(), [(W, b, c.act)], unit=UNIT)
    y, ey = _chain(h, [(hw.view(c.N, 1), torch.tensor([hb], device=device), c.head_act)], eh, unit=0.0)
    _within(hbuf[:c.M], y[:, 0], ey[:, 0], f"head ({c.act} -> {c.head_act})")


# ---------------------------------------------------------------------------------------------------------------
# 4. mm_inbatch_scores_tc: the scorer epilogue, both schedules
# ---------------------------------------------------------------------------------------------------------------
def _scorer_ids(kind, B, N, g, device):
    """(positive ids (B,), negative ids (N,)) of the kind: 40 distinct values (many hits); "wide" adds 2^32 to about
    half of them, so ids that differ only above bit 31 sit side by side in a tile."""
    if kind is None:
        return None, None
    p = torch.randint(0, 40, (B,), generator=g, device=device)
    n = torch.randint(0, 40, (N,), generator=g, device=device)
    if kind == "wide":
        p = p + (torch.randint(0, 2, (B,), generator=g, device=device) << 32)
        n = n + (torch.randint(0, 2, (N,), generator=g, device=device) << 32)
    return (p.int(), n.int()) if kind == "i32" else (p, n)


@pytest.mark.parametrize("c", SCORER, ids=lambda c: f"B{c.B}-N{c.N}-D{c.D}-T{c.T}-{'logq' if c.logq else 'nologq'}-{c.ids}-{c.layout}")
def test_inbatch_scores_tc_matches_float64(device, c):
    """logits[m, 1 + n] = (mask ? fns : q_m . neg_n - log(p_n + 1e-16)) / T through the C entry alone, so column 0 (the
    positive, another kernel's) and every guard stay NaN.  Bound as test_inbatch_scorer_at_scale, with UNIT; masked
    entries are fl(fns / T) bit for bit and exactly as many as id hits."""
    B, N, D, T = c.B, c.N, c.D, c.T
    sms = _sms(device)
    p = plan(B, D, N, score=True, sms=sms)
    resident, tpc, _ = _scorer_schedule(B, N, D, sms)
    assert resident == p["resident"] and tpc == p["tiles_per_cta"]
    if B > 1001:
        assert resident and tpc >= 3 and p["tiles"] % tpc, f"premise: {p['tiles']} tiles, {tpc} per CTA"
    g = torch.Generator(device=device).manual_seed(B + N + D)
    q = torch.randn((B, D), generator=g, device=device)
    neg = torch.randn((N, D), generator=g, device=device)
    q[::9] *= 30.0
    prob = torch.rand(N, generator=g, device=device) * 0.5 + 1e-4 if c.logq else None
    pid, nid = _scorer_ids(c.ids, B, N, g, device)
    c0, stride = scorer_out(B, N, c.layout)
    buf = _nan((B + GUARD, stride), device)
    out = buf[:B, c0:c0 + 1 + N]
    id_dt = _cabi.MM_I32 if c.ids == "i32" else _cabi.MM_I64
    qs, ns = ops.split_rows(q), ops.split_rows(neg)  # held: the kernel reads them after the call returns
    _cabi.check(_cabi.load().mm_inbatch_scores_tc(
        qs.data_ptr(), ns.data_ptr(), B, N, D, None if pid is None else pid.data_ptr(),
        None if nid is None else nid.data_ptr(), id_dt, int(c.ids is not None), FNS, None if prob is None else prob.data_ptr(),
        T, out.data_ptr(), stride, torch.cuda.current_stream().cuda_stream), "mm_inbatch_scores_tc")
    _untouched(buf[:, c0 + 1:], B, N, "scorer")
    assert bool(torch.isnan(buf[:, :c0 + 1]).all()), "scorer: column 0 or a guard column before it was written"
    T32 = float(torch.tensor(T, dtype=torch.float32))
    fns = torch.tensor(FNS, dtype=torch.float32)
    masked = float(fns if T == 1.0 else fns / torch.tensor(T, dtype=torch.float32))
    qd, nd = q.double(), neg.double()
    dot = qd @ nd.T
    lq = -torch.log(prob.double() + 1e-16) if c.logq else torch.zeros(N, dtype=torch.float64, device=device)
    s = (dot + lq) / T32
    bound = ((UNIT + D * E) * (qd.abs() @ nd.abs().T) + 4 * E * lq.abs() + E * (dot.abs() + lq.abs())) / T32 + E * s.abs()
    got = out[:, 1:]
    if pid is None:
        _within(got, s, bound, "scorer logits")
        return
    hit = pid.long().view(-1, 1) == nid.long().view(1, -1)
    want = torch.where(hit, torch.full((), masked, dtype=torch.float64, device=device), s)
    _within(got, want, torch.where(hit, torch.zeros_like(bound), bound), "scorer logits")
    assert int((got == masked).sum()) == int(hit.sum()) > 0, "scorer: masked entries differ from the id hits"


# ---------------------------------------------------------------------------------------------------------------
# 5. M = 0
# ---------------------------------------------------------------------------------------------------------------
def test_dense_tc_zero_rows_writes_nothing(device):
    """M = 0 through the C entries (torch hands out null pointers for empty tensors, which the entries refuse): every
    output buffer, fp32 and split rows, cross, head, keeps its NaN."""
    K, N = 65, 30  # the head needs N <= 32; Np = 32 < Kp(N) = 64: the split has a padding gap
    Kp, Np, oKp = ops.tc_padded_k(K), ops.tc_padded_n(N), ops.tc_padded_k(N)
    W = ops.split_weights(torch.randn((K, N), device=device))
    b, hw = torch.randn(N, device=device), torch.randn(N, device=device)
    a = ops.split_rows(torch.randn((GUARD, K), device=device))
    fb, sb, hb = _nan((GUARD, N), device), _nan_bf16((GUARD, 2 * oKp), device), _nan((GUARD,), device)
    x0 = torch.randn((GUARD, N), device=device)
    lib, st = _cabi.load(), torch.cuda.current_stream().cuda_stream
    gelu, relu, sig = (_cabi.ACTIVATIONS[k] for k in ("gelu", "relu", "sigmoid"))
    _cabi.check(lib.mm_dense_tc(a.data_ptr(), 0, K, Kp, W.data_ptr(), N, Np, b.data_ptr(), gelu, 3, None, None, 0,
                                fb.data_ptr(), N, sb.data_ptr(), oKp, st), "mm_dense_tc")
    _cabi.check(lib.mm_dense_tc(a.data_ptr(), 0, K, Kp, W.data_ptr(), N, Np, b.data_ptr(), 0, 3, x0.data_ptr(), x0.data_ptr(),
                                N, fb.data_ptr(), N, None, 0, st), "mm_dense_tc (cross)")
    _cabi.check(lib.mm_dense_tc_head(a.data_ptr(), 0, K, Kp, W.data_ptr(), N, Np, b.data_ptr(), relu, 3, hw.data_ptr(), 0.5,
                                     sig, hb.data_ptr(), st), "mm_dense_tc_head")
    torch.cuda.synchronize()
    for t, what in ((fb, "out_f32"), (sb, "out_split"), (hb, "head_out")):
        assert bool(torch.isnan(t.float()).all()), f"M = 0 wrote {what}"
