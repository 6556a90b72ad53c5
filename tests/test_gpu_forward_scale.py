"""The forward kernels at the sizes the benchmark runs: the fused DLRM lookup + interaction and the top tower at
B = 65 536, the DCN-v2 cross layer at B = 65 536, d = 1037, and the two-tower in-batch scorer at B = N = 16 384.  Every
one of them is persistent: a CTA walks many tiles or samples, so after its first lap it runs with ring stages refilled,
mbarrier phases flipped, sample buffers rotated and (scorer) the resident query tile reloaded.  Each large-size test
asserts from the launcher's own formula and the device's SM count that the kernel makes at least two laps, and compares
EVERY output with a float64 reference computed on the device in chunks.

Bounds are per element and derived from the arithmetic (conventions of test_gpu_train_scale):
  * a 3-pass split-bf16 product is within U = 2^-16 of |a b|;
  * an fp32 sum of n terms, in any order, is within n E sum |terms| (E = 2^-24);
  * so a K-deep GEMM or dot entry is within (U + K E) (|A| @ |B|), plus the bias and epilogue roundings;
  * through a chain of layers the bound propagates element-wise (_chain):
        e_l = Lip(act_l) (e_{l-1} @ |W_l| + (U + K_l E) ((|h_{l-1}| + e_{l-1}) @ |W_l| + |b_l|)) + rounding of act_l,
    Lip = 1 for relu / linear, 1/4 for sigmoid, whose own rounding (1 / (1 + expf(-v)): expf within 2 ulp, one add,
    one division) is under 8 E |sigmoid|;
  * a split-bf16 output hi + lo adds at most 2^-16 of the value.
Every activation on the forward pass is Lipschitz, so no unit needs to be excluded.  A lost, repeated or stale lap, a
dropped bias or a wrong operand moves an output by O(1) of its scale, far above these bounds.

Output buffers carry NaN guard rows past the batch and NaN padding columns past the logical width; they must stay NaN,
and the padding columns of split-bf16 outputs must be exact zeros."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import blocks, datasets, ops
from models_b200.graph import HostBatch
from tests import twotower_train_oracle as O
from tests.test_gpu_lookup_v2 import pack_ids
from tests.test_gpu_train_scale import (BIG, CAP, E, GUARD, RAGGED, U, WIDTHS, _ids_with_oob, _nan, _sms, _untouched,
                                        _width_rows, _within)
from tests.test_gpu_train_twotower import _ce_case

pytestmark = pytest.mark.gpu
SPLIT = 2.0 ** -16  # hi + lo of a split-bf16 output against its fp32 value, relative


def _nan_bf16(shape, device):
    return torch.full(shape, float("nan"), dtype=torch.bfloat16, device=device)


def _unsplit(buf, W):
    """hi + lo of the first W columns of split-bf16 rows (M, 2 Kp), in float64."""
    Kp = buf.shape[1] // 2
    return buf[:, :W].double() + buf[:, Kp:Kp + W].double()


def _split_padding_zero(buf, rows, W, what):
    """Rows >= `rows` of a NaN-filled split-bf16 buffer were not written; columns W..Kp of hi and lo are exact zeros."""
    Kp = buf.shape[1] // 2
    assert bool(torch.isnan(buf[rows:].float()).all()), f"{what}: a guard row past the batch was written"
    if Kp > W:
        pad = torch.cat([buf[:rows, W:Kp], buf[:rows, Kp + W:]], dim=1)
        assert bool((pad.float() == 0).all()), f"{what}: a padding column of the split output is not zero"


# activation: (float64 function, Lipschitz constant L, own rounding in units of E as (a, g): a |y| + g |z|); the
# constants of tanh, selu, elu and gelu are derived in tests/test_gpu_dense_tc_kernels.py
ACT_REF = {
    None: (lambda z: z, 1.0, 0, 0), "linear": (lambda z: z, 1.0, 0, 0), "relu": (lambda z: z.clamp_min(0.0), 1.0, 0, 0),
    "sigmoid": (torch.sigmoid, 0.25, 8, 0), "tanh": (torch.tanh, 1.0, 4, 0), "selu": (torch.nn.functional.selu, 1.76, 8, 0),
    "elu": (torch.nn.functional.elu, 1.0, 2, 0), "gelu": (torch.nn.functional.gelu, 1.13, 1, 4),
}


def _act(z, ez, act):
    """float64 act(z) and the bound of the device's act at a pre-activation within ez of z: L ez for the error carried
    in, plus the activation's own rounding at that pre-activation, E (a (|y| + L ez) + g (|z| + ez))."""
    f, L, a, g = ACT_REF[act]
    y = f(z)
    e = L * ez
    if a or g:
        e = e + E * (a * (y.abs() + e) + g * (z.abs() + ez))
    return y, e


def _chain(h, layers, e=None, unit=U):
    """float64 forward of Dense layers (W (K, N) fp32, b (N,) or None, activation) from h, which is within e of the
    device's input, and the element-wise bound of the module docstring.  `unit`: the relative error of one product
    (U for 3-pass split-bf16, 0 for fp32 CUDA-core dots).  Returns (output, bound)."""
    e = torch.zeros_like(h) if e is None else e
    for W, b, act in layers:
        Wd = W.double()
        Wa = Wd.abs()
        z = h @ Wd
        ba = 0.0
        if b is not None:
            z = z + b.double()
            ba = b.double().abs()
        ez = e @ Wa + (unit + W.shape[0] * E) * ((h.abs() + e) @ Wa + ba)
        h, e = _act(z, ez, act)
    return h, e


def _chunks(M, chunk=8192):
    return [(s, min(M, s + chunk)) for s in range(0, M, chunk)]


# ---------------------------------------------------------------------------------------------------------------
# 1. mm_dlrm_lookup_interact
# ---------------------------------------------------------------------------------------------------------------
def _interact_iters(B, D, F, P, out_Kp, sms, world=1):
    """(warps per CTA, CTAs, fewest iterations of a warp) as launch<1> in interaction_v2.cu chooses them."""
    OW = P + F * (F - 1) // 2
    stage_cols = out_Kp if out_Kp else (OW + 3) & ~3
    buf = (max(F * D * 4, stage_cols * 4) + 255) & ~255
    peer = F * world * 8 if world > 1 else 0
    warps = min((227 * 1024 - peer) // (2 * buf), 16)
    grid = min(-(-B // warps), sms)
    n_cta = B // grid  # the smallest contiguous sample range of a CTA
    return warps, grid, -(-n_cta // warps)


def _interaction_fwd(rows_of_slot, F, P):
    """[bottom |] upper-triangle pairwise dots (row-major, i < j) of the (n, F, D) float64 stack, and their bound scale
    sum_d |x_i| |x_j|."""
    st = rows_of_slot
    iu = torch.triu_indices(F, F, 1, device=st.device)
    z = torch.bmm(st, st.transpose(1, 2))[:, iu[0], iu[1]]
    za = torch.bmm(st.abs(), st.abs().transpose(1, 2))[:, iu[0], iu[1]]
    return z, za


INTERACT_CASES = [(64, "f32", "f32"), (64, "f32", "split"), (64, "operand", "split")]


@pytest.mark.parametrize("D,rows_fmt,out_fmt,B", [c + (b,) for c in INTERACT_CASES for b in (BIG, RAGGED)] +
                         [(d, "f32", o, b) for d in (16, 128) for o in ("f32", "split") for b in (8192, 8192 + 37)])
def test_lookup_interact_at_scale(device, D, rows_fmt, out_fmt, B):
    """Criteo shape: 26 tables + the bottom vector at its sorted slot (as DLRM.slots() places it), P = D, ids of every
    width (1, 2, 3, 4, 8 bytes) with ~1 % outside the table; fp32 rows or (D = 64) the operand-format mirrors; fp32
    output at a row stride > OW or the split-bf16 operand of the top tower.
    Bound per pair (U + D E) sum_d |x_i| |x_j|: D split-bf16 products (U each) summed in fp32 over D / 16 MMA steps
    (D E); the split output adds 2^-16 of the value.  The prefix is a copy: the bottom itself (fp32 output) or its
    split (split output), bit for bit.  The out-of-range count is exact.  A sample is one warp's work, so windows
    launched alone (first lap, mid-batch, ragged end) equal the full run bit for bit, and (B = 65 536) so does the
    row-sharded placement (world 8, all shards on this GPU handed over as the peers, ranks 0 and 7)."""
    T = 26
    F, P = T + 1, D
    OW = P + F * (F - 1) // 2
    operand = rows_fmt == "operand"
    out_Kp = ops.tc_padded_k(OW) if out_fmt == "split" else 0
    warps, ctas, iters = _interact_iters(B, D, F, P, out_Kp, _sms(device))
    assert iters >= 2, f"premise: B = {B} gives {iters} iteration(s) per warp of {warps} warps x {ctas} CTAs"
    rng = np.random.default_rng(B + D + 3 * operand + (out_fmt == "split"))
    gen = torch.Generator(device=device).manual_seed(B + D)
    widths = [WIDTHS[t % 5] for t in range(T)]
    rows = [_width_rows(w, t) for t, w in enumerate(widths)]
    tables = [torch.randn((r, D), generator=gen, device=device) * 0.3 for r in rows]
    ids64 = [_ids_with_oob(rng, r, w, B) for r, w in zip(rows, widths)]
    ids = [torch.from_numpy(pack_ids(i, w)).to(device) for i, w in zip(ids64, widths)]
    assert [ops.index_bytes_of(i) for i in ids] == widths
    names = sorted([f"C{t}" for t in range(T)] + ["bottom_block"])
    slot_b = names.index("bottom_block")
    slots = [names.index(f"C{t}") for t in range(T)]
    bottom = torch.randn((B, D), generator=gen, device=device)
    bottom[:, ::5] = 0.0
    w_in = [ops.split_rows(w) for w in tables] if operand else tables
    b_in = ops.split_rows(bottom) if operand else bottom
    want_oob = sum(int(((i < 0) | (i >= r)).sum()) for i, r in zip(ids64, rows))
    assert want_oob >= T * (B // 100)

    def new_out(n):
        return _nan_bf16((n + GUARD, 2 * out_Kp), device) if out_Kp else _nan((n + GUARD, OW + 5), device)

    def run(buf, lo=0, hi=B, weights=None, peers=None, rank=0, world=1):
        n = hi - lo
        out = buf[:n] if out_Kp else buf[:n, :OW]
        oob = torch.zeros(1, dtype=torch.int32, device=device)
        ops.dlrm_lookup_interact(w_in if weights is None else weights, [i[lo:hi] for i in ids], slots, rows, D, b_in[lo:hi],
                                 slot_b, out, oob, peers=peers, rank=rank, world=world, operand_rows=operand)
        return int(oob.item())

    full = new_out(B)
    assert run(full) == want_oob, "out-of-range ids miscounted"
    # prefix: a copy of the bottom vector (fp32) or of its split (split output; operand rows: the rows handed in)
    if out_Kp:
        sb = b_in if operand else ops.split_rows(bottom)
        Kb = sb.shape[1] // 2
        assert torch.equal(full[:B, :D], sb[:, :D]) and torch.equal(full[:B, out_Kp:out_Kp + D], sb[:, Kb:Kb + D]), \
            "prefix is not the bottom's split"
        _split_padding_zero(full, B, OW, "split output")
    else:
        assert torch.equal(full[:B, :D], bottom), "prefix is not a copy of the bottom vector"
        _untouched(full, B, OW, "fp32 output")
    dev_ids = [torch.from_numpy(i).to(device) for i in ids64]
    for s, e in _chunks(B):
        st = torch.empty((e - s, F, D), dtype=torch.float64, device=device)
        for t in range(T):
            i = dev_ids[t][s:e]
            ok = (i >= 0) & (i < rows[t])
            st[:, slots[t]] = (tables[t][i.clamp(0, rows[t] - 1)] * ok.unsqueeze(1)).double()
        st[:, slot_b] = bottom[s:e].double()
        z, za = _interaction_fwd(st, F, P)
        bound = (U + D * E) * za
        if out_Kp:
            got = _unsplit(full[s:e], OW)[:, P:]
            bound = bound + SPLIT * z.abs()
        else:
            got = full[s:e, P:OW]
        _within(got, z, bound, f"pairs of samples [{s}, {e})")
    # position independence: windows launched alone, bit for bit
    for lo, w in ((0, 1000), (B // 2 + 3, 777), (B - 901, 901)):
        wb = new_out(w)
        run(wb, lo, lo + w)
        a, b = (wb[:w], full[lo:lo + w]) if out_Kp else (wb[:w, :OW], full[lo:lo + w, :OW])
        assert torch.equal(a, b), f"window [{lo}, {lo + w}) depends on the position"
    if B != BIG:
        return
    # row-sharded placement: row r on rank r % world at local row r // world; every fifth table replicated
    world = 8
    assert _interact_iters(B, D, F, P, out_Kp, _sms(device), world)[2] >= 2
    for rank in (0, world - 1):
        weights, peers, keep = [], [], []
        for t in range(T):
            if t % 5 == 4:
                weights.append(w_in[t])
                peers.append(None)
                continue
            pad = torch.zeros((1, w_in[t].shape[1]), dtype=w_in[t].dtype, device=device)
            shards = [torch.cat([w_in[t][k::world], pad]).contiguous() for k in range(world)]
            keep.append(shards)
            weights.append(shards[rank])
            peers.append([x.data_ptr() for x in shards])
        sh = new_out(B)
        assert run(sh, weights=weights, peers=peers, rank=rank, world=world) == want_oob
        assert torch.equal(sh[:B], full[:B]) if out_Kp else torch.equal(sh[:B, :OW], full[:B, :OW]), \
            f"rank {rank} of {world}: the sharded placement differs from the replicated run"
        del keep


# ---------------------------------------------------------------------------------------------------------------
# 2. mm_mlp_tc / mm_mlp_tc_heads: the DLRM top tower
# ---------------------------------------------------------------------------------------------------------------
def _tower_laps(M, sms):
    """Fewest tiles any consumer warpgroup of mlp_tc_kernel runs (mlp_tc_impl: one CTA per SM over 64-row tiles, which
    the CTA's two consumer warpgroups take in turn)."""
    tiles = -(-M // 64)
    return tiles // min(tiles, sms) // 2


@pytest.mark.parametrize("M", [BIG, RAGGED])
def test_top_tower_at_scale(device, M):
    """K = 415 (the interaction output), [128, 64, 32] relu, the fused Dense(32 -> 1) sigmoid head, from the split
    operand of fp32 rows.  (a) fp32 rows and the head together, (b) the head alone, (c) mm_mlp_tc_heads with three
    heads (sigmoid, linear, sigmoid) as the multi-task model runs it.  Bound: _chain over the three layers (each
    split-bf16 on the tensor cores, K = 415 / 128 / 64), then the head (an fp32 dot of 32 terms, bias, activation)."""
    laps = _tower_laps(M, _sms(device))
    assert laps >= 2, f"premise: M = {M} gives {laps} lap(s)"
    K, widths = 415, [128, 64, 32]
    acts = ["relu"] * 3
    gen = torch.Generator(device=device).manual_seed(M)
    x = torch.randn((M, K), generator=gen, device=device)
    Ws = [torch.randn((k, n), generator=gen, device=device) / k ** 0.5 for k, n in zip([K] + widths[:-1], widths)]
    bs = [torch.randn(n, generator=gen, device=device) * 0.1 for n in widths]
    hw = torch.randn(32, generator=gen, device=device) / 32 ** 0.5
    hb = 0.25
    Hw = torch.randn((32, 3), generator=gen, device=device) / 32 ** 0.5
    Hb = torch.tensor([0.1, -0.2, 0.3], device=device)
    a, ws = ops.split_rows(x), [ops.split_weights(w) for w in Ws]

    obuf, h1, h2 = _nan((M + GUARD, 36), device), _nan((M + GUARD,), device), _nan((M + GUARD,), device)
    ops.mlp_tc(a, K, ws, widths, bs, acts, out=obuf[:M, :32], head_w=hw, head_b=hb, head_act="sigmoid", head_out=h1[:M])
    ops.mlp_tc(a, K, ws, widths, bs, acts, head_w=hw, head_b=hb, head_act="sigmoid", head_out=h2[:M])
    hbuf = _nan((3 * M + GUARD,), device)
    ops.mlp_tc_heads(a, K, ws, widths, bs, acts, Hw, Hb, ["sigmoid", None, "sigmoid"], hbuf[:3 * M].view(3, M))
    _untouched(obuf, M, 32, "tower rows")
    for buf, what in ((h1, "head with rows"), (h2, "head alone"), (hbuf[2 * M:], "heads")):
        assert bool(torch.isnan(buf[-GUARD:]).all()), f"{what}: a guard element past the batch was written"
    heads = hbuf[:3 * M].view(3, M)
    tower = list(zip(Ws, bs, acts))
    for s, e in _chunks(M):
        h, eb = _chain(x[s:e].double(), tower)
        _within(obuf[s:e, :32], h, eb, f"tower rows [{s}, {e})")
        y, ey = _chain(h, [(hw.view(32, 1), torch.tensor([hb], device=device), "sigmoid")], eb)
        _within(h1[s:e], y[:, 0], ey[:, 0], f"head (with rows) [{s}, {e})")
        _within(h2[s:e], y[:, 0], ey[:, 0], f"head alone [{s}, {e})")
        for j, act in enumerate(["sigmoid", None, "sigmoid"]):
            y, ey = _chain(h, [(Hw[:, j:j + 1].contiguous(), Hb[j:j + 1], act)], eb)
            _within(heads[j, s:e], y[:, 0], ey[:, 0], f"head {j} ({act}) of mm_mlp_tc_heads [{s}, {e})")


# ---------------------------------------------------------------------------------------------------------------
# 3. mm_dense_tc at the DCN-v2 shapes
# ---------------------------------------------------------------------------------------------------------------
def _dense_tc_laps(M, N, sms):
    """Laps of dense_tc_kernel's interleaved schedule (dense_tc_launch: 128-row x BN tiles, one CTA per SM)."""
    Np = ops.tc_padded_n(N)
    tiles = -(-M // 128) * (Np // min(Np, 128))
    return -(-tiles // min(tiles, sms))


@pytest.mark.parametrize("M", [BIG, RAGGED])
def test_cross_layer_at_scale(device, M):
    """DCN-v2 cross layer x0 * (x W + b) + x at d = 1037 (9 n-tiles per 128-row m-tile, ~35 laps): out_f32 and the next
    layer's split operand, x0 / xres at row stride 1037 (scalar loads, as the model and the benchmark pass them; fp32
    rows at an odd stride) and 1040 (vector loads and stores).  Bound per element
    |x0| (U + d E) (|x| @ |W| + |b|) + E (|x0 z| + |x|): the GEMM entry and its bias, then one rounded product and one
    rounded sum; the split output adds 2^-16 of the value.  The padding columns 1037..1088 of the split are zero."""
    d = 1037
    laps = _dense_tc_laps(M, d, _sms(device))
    assert laps >= 2, f"premise: M = {M} gives {laps} lap(s)"
    gen = torch.Generator(device=device).manual_seed(M + d)
    x = torch.randn((M, d), generator=gen, device=device)
    x0 = torch.randn((M, d), generator=gen, device=device)
    W = torch.randn((d, d), generator=gen, device=device) / d ** 0.5
    b = torch.randn(d, generator=gen, device=device) * 0.1
    a, ws = ops.split_rows(x), ops.split_weights(W)
    Kp = ops.tc_padded_k(d)
    runs = []
    for xs, os_ in ((d, d + 2), (1040, 1040)):
        if xs == d:
            x0v, xv = x0, x
        else:
            x0v, xv = _nan((M, xs), device)[:, :d], _nan((M, xs), device)[:, :d]
            x0v.copy_(x0)
            xv.copy_(x)
        fb, sb = _nan((M + GUARD, os_), device), _nan_bf16((M + GUARD, 2 * Kp), device)
        ops.dense_tc(a, d, ws, d, b, None, out_f32=fb[:M, :d], out_split=sb[:M], x0=x0v, xres=xv)
        _untouched(fb, M, d, f"cross out_f32 (x_stride {xs})")
        _split_padding_zero(sb, M, d, f"cross out_split (x_stride {xs})")
        runs.append((xs, fb, sb))
        del x0v, xv
    Wd, Wa, bd = W.double(), W.double().abs(), b.double()
    for s, e in _chunks(M, 4096):
        xd, x0d = x[s:e].double(), x0[s:e].double()
        z = xd @ Wd + bd
        want = x0d * z + xd
        bound = x0d.abs() * (U + d * E) * (xd.abs() @ Wa + bd.abs()) + E * ((x0d * z).abs() + xd.abs())
        for xs, fb, sb in runs:
            _within(fb[s:e, :d], want, bound, f"cross out_f32 (x_stride {xs}) rows [{s}, {e})")
            _within(_unsplit(sb[s:e], d), want, bound + SPLIT * want.abs(), f"cross out_split (x_stride {xs}) rows [{s}, {e})")


@pytest.mark.parametrize("M", [BIG, RAGGED])
def test_dense_relu_and_head_at_scale(device, M):
    """The DCN deep tower's layers on the tensor cores: relu 1037 -> 256 (two n-tiles) into fp32 rows and the split
    operand, and mm_dense_tc_head: relu 256 -> 32 with the fused Dense(32 -> 1) sigmoid.  Bounds from _chain."""
    sms = _sms(device)
    assert min(_dense_tc_laps(M, 256, sms), _dense_tc_laps(M, 32, sms)) >= 2, "premise: a single lap"
    gen = torch.Generator(device=device).manual_seed(M + 256)
    K = 1037
    x = torch.randn((M, K), generator=gen, device=device)
    W1 = torch.randn((K, 256), generator=gen, device=device) / K ** 0.5
    b1 = torch.randn(256, generator=gen, device=device) * 0.1
    W2 = torch.randn((256, 32), generator=gen, device=device) / 16.0
    b2 = torch.randn(32, generator=gen, device=device) * 0.1
    hw = torch.randn(32, generator=gen, device=device) / 32 ** 0.5
    hb = -0.125
    fb, sb = _nan((M + GUARD, 260), device), _nan_bf16((M + GUARD, 512), device)
    ops.dense_tc(ops.split_rows(x), K, ops.split_weights(W1), 256, b1, "relu", out_f32=fb[:M, :256], out_split=sb[:M])
    _untouched(fb, M, 256, "relu layer out_f32")
    _split_padding_zero(sb, M, 256, "relu layer out_split")
    h2 = torch.randn((M, 256), generator=gen, device=device).clamp_min(0.0)  # a relu layer's output
    hbuf = _nan((M + GUARD,), device)
    ops.dense_tc_head(ops.split_rows(h2), 256, ops.split_weights(W2), 32, b2, "relu", hw, hb, "sigmoid", hbuf[:M])
    assert bool(torch.isnan(hbuf[M:]).all()), "head: a guard element past the batch was written"
    for s, e in _chunks(M, 4096):
        y, ey = _chain(x[s:e].double(), [(W1, b1, "relu")])
        _within(fb[s:e, :256], y, ey, f"relu layer out_f32 rows [{s}, {e})")
        _within(_unsplit(sb[s:e], 256), y, ey + SPLIT * y.abs(), f"relu layer out_split rows [{s}, {e})")
        y, ey = _chain(h2[s:e].double(), [(W2, b2, "relu"), (hw.view(32, 1), torch.tensor([hb], device=device), "sigmoid")])
        _within(hbuf[s:e], y[:, 0], ey[:, 0], f"dense_tc_head rows [{s}, {e})")


# ---------------------------------------------------------------------------------------------------------------
# 4. the in-batch scorer: mm_positive_scores + mm_inbatch_scores_tc, and mm_inbatch_softmax_ce
# ---------------------------------------------------------------------------------------------------------------
def _scorer_schedule(B, N, D, sms):
    """(resident-A schedule on, tiles per CTA, some CTA's contiguous tile range crosses an m-row) as dense_tc_launch
    plans mm_inbatch_scores_tc."""
    Np = ops.tc_padded_n(N)
    ntn = Np // min(Np, 128)
    tiles = -(-B // 128) * ntn
    tpc = -(-tiles // min(tiles, sms))
    resident = ops.tc_padded_k(D) <= 128 and ntn >= 8
    crosses = any((c * tpc) // ntn != (min(tiles, (c + 1) * tpc) - 1) // ntn for c in range(-(-tiles // tpc)))
    return resident, tpc, crosses


def _zipf_ids(rng, n, wide):
    """Zipf item ids (one id takes thousands of rows); `wide`: a third of them moved above 2^32 (a bijection, so the
    hits are the same) to reach the 64-bit compare of the mask."""
    z = np.minimum(rng.zipf(1.3, n) - 1, 10 ** 6).astype(np.int64)
    return z + (z % 3 == 0) * (1 << 33) if wide else z


@pytest.mark.parametrize("B,N,D,T,logq", [(16384, 16384, 128, 0.05, True), (16384, 16384, 128, 1.0, False),
                                          (16384 - 5, 16384 + 77, 64, 0.05, True)])
def test_inbatch_scorer_at_scale(device, B, N, D, T, logq):
    """Down-scoring on with Zipf item ids (int64 at B = N: the in-batch negatives are the positives; int32 in the
    ragged case).  All B (1 + N) logits against float64, in query-row chunks, in the model's layout (column 1 of a
    (B, 1 + N) buffer, 4-byte aligned: scalar stores) and the benchmark's (negatives 16-byte aligned: vector stores).
    Negatives: ((U + D E) (|q| @ |n|^T) + 4 E |log p| + E (|q n| + |log p|)) / T + E |s|: the split-bf16 dot, -logf (within
    2 ulp) added with one rounding, one IEEE division.  Column 0 (fp32 fma dot): the same with D E in place of U + D E.
    A masked entry is fl(fp32(false_neg_score) / fp32(T)) bit for bit, and there are exactly as many as id hits.
    mm_inbatch_softmax_ce for the same case: the positive logit equals column 0 bit for bit; the row max within the
    largest logit bound of the row (+ 2 E |s| for its x fl(1/T) in place of / T); log-sum-exp, 1-Lipschitz in the
    max-norm, within that plus the relative error of its fp32 sum of exponentials: each partial adds 12 rounded steps
    per 128-column tile (8 ex2.approx terms per accumulator, the rescale, the three-way combine) over its tiles of the
    item range, the merge 4 per partial over P / 32 partials per lane and a 5-step warp sum; each step within 2^-21."""
    sms = _sms(device)
    resident, tpc, crosses = _scorer_schedule(B, N, D, sms)
    assert resident and tpc >= 2 and crosses, f"premise: resident-A {resident}, {tpc} tiles per CTA, m-row crossing {crosses}"
    wide = B == N
    q, pos, neg, _, _, prob = _ce_case(device, B, N, D, True, logq, T, seed=2 if B == N else 3)
    assert (neg is pos) == (B == N)
    rng = np.random.default_rng(B + N + int(logq))
    pid = torch.from_numpy(_zipf_ids(rng, B, wide)).to(device)
    nid = pid if neg is pos else torch.from_numpy(_zipf_ids(rng, N, wide)).to(device)
    if not wide:
        pid, nid = pid.int(), nid.int()
    pprob = (prob if neg is pos else torch.rand(B, generator=torch.Generator(device=device).manual_seed(B), device=device)
             * 0.5 + 1e-4) if logq else None
    kw = dict(pos_ids=pid, neg_ids=nid, downscore=True, false_neg_score=O.MIN_FLOAT, pos_prob=pprob, neg_prob=prob, temperature=T)
    model_buf = _nan((B + GUARD, N + 4), device)
    bench_buf = _nan((B + GUARD, N + 4), device)
    layouts = (("model layout", model_buf, model_buf[:B, :1 + N], (1 + N, N + 4)),
               ("bench layout", bench_buf, bench_buf[:B, 3:4 + N], (0, 3)))
    for _, _, view, _ in layouts:
        ops.inbatch_scores(q, pos, neg, view, **kw)
    assert (bench_buf[:B, 4:].data_ptr() % 16) == 0 and (model_buf[:B, 1:].data_ptr() % 16) != 0
    for what, buf, _, (c0, c1) in layouts:
        assert bool(torch.isnan(buf[B:]).all()), f"{what}: a guard row past the batch was written"
        assert bool(torch.isnan(buf[:B, c0:c1]).all()), f"{what}: a padding column was written"
    stats = ops.inbatch_softmax_ce(q, pos, neg, pos_ids=pid, neg_ids=nid, downscore=True, false_neg_score=O.MIN_FLOAT,
                                   pos_prob=pprob, neg_prob=prob, temperature=T)
    assert torch.equal(stats[:, 2], layouts[0][2][:, 0]), "soft-max positive logit differs from column 0 of the scorer"

    T32 = float(np.float32(T))
    fns = np.float32(O.MIN_FLOAT)
    masked = float(fns if T == 1.0 else np.float32(fns / np.float32(T)))
    qd, pd, nd = q.double(), pos.double(), neg.double()
    nda = nd.abs()
    lq = -torch.log(prob.double() + 1e-16) if logq else torch.zeros(N, dtype=torch.float64, device=device)
    lp = -torch.log(pprob.double() + 1e-16) if logq else torch.zeros(B, dtype=torch.float64, device=device)
    P = (ops.catalog_workspace_bytes(B, N) - 256) // (12 * B)  # partials per row (kParts x item-range splits)
    tiles_per_split = -(-(-(-N // 128)) // (P // 4))
    depth = 12 * tiles_per_split + 4 * -(-P // 32) + 8
    hits = 0
    for s, e in _chunks(B, 1024):
        qc = qd[s:e]
        dot = qc @ nd.T
        hit = pid[s:e].view(-1, 1).long() == nid.view(1, -1).long()
        hits += int(hit.sum())
        sn = (dot + lq) / T32
        bn = ((U + D * E) * (qc.abs() @ nda.T) + 4 * E * lq.abs() + E * (dot.abs() + lq.abs())) / T32 + E * sn.abs()
        d0 = (qc * pd[s:e]).sum(1)
        s0 = (d0 + lp[s:e]) / T32
        b0 = (D * E * (qc.abs() * pd[s:e].abs()).sum(1) + 4 * E * lp[s:e].abs() + E * (d0.abs() + lp[s:e].abs())) / T32 + E * s0.abs()
        want = torch.where(hit, torch.full((), masked, dtype=torch.float64, device=device), sn)
        bound = torch.where(hit, torch.zeros((), dtype=torch.float64, device=device), bn)
        for what, _, view, _ in layouts:
            _within(view[s:e, 0], s0, b0, f"{what}: column 0 of rows [{s}, {e})")
            _within(view[s:e, 1:], want, bound, f"{what}: negatives of rows [{s}, {e})")
            n_masked = int((view[s:e, 1:] == masked).sum())
            assert n_masked == int(hit.sum()), f"{what}: {n_masked} masked entries in rows [{s}, {e}) for {int(hit.sum())} id hits"
        # soft-max statistics: x fl(1 / T) rounds once more than / T
        ce = torch.cat([s0.unsqueeze(1), torch.where(hit, torch.full((), float(fns) / T32, dtype=torch.float64, device=device), sn)], 1)
        cb = torch.cat([b0.unsqueeze(1), torch.where(hit, torch.zeros((), dtype=torch.float64, device=device), bn)], 1) + 2 * E * ce.abs()
        rmax, lse = ce.max(1).values, torch.logsumexp(ce, 1)
        bmax = cb.max(1).values
        _within(stats[s:e, 0], rmax, bmax, f"soft-max row max of rows [{s}, {e})")
        blse = bmax + depth * 2.0 ** -21 + 4 * E * (lse.abs() + ce.abs().max(1).values)
        _within(stats[s:e, 1], lse, blse, f"soft-max log-sum-exp of rows [{s}, {e})")
    assert hits > 4 * B, f"premise: only {hits} id hits"


# ---------------------------------------------------------------------------------------------------------------
# 5. the DLRM forward as bench.py runs it
# ---------------------------------------------------------------------------------------------------------------
def _layers(block_layers):
    return [(l.kernel, l.bias, l.activation) for l in block_layers]


def test_dlrm_forward_as_the_benchmark_runs_it(device):
    """Criteo schema capped at 400 000 rows (1/2/3-byte packed ids through HostBatch), embedding_dim 64 with the operand
    mirrors, bottom [128, 64], top [128, 64, 32], B = 65 536, one compiled graph.  The graph replay equals the eager
    forward on int64 ids bit for bit.  Then the three stages run eagerly with the calls of RankingModel.call's production
    path, each checked against float64 of ITS OWN device input (so every bound stays local):
      bottom: the fp32 columns -> operand rows (mm_tower2_small), _chain + 2^-16 of the split;
      interaction: the device bottom as hi + lo and the fp32 tables -> the split operand: prefix = the bottom's rows
        bit for bit, pairs within (U + 64 E) sum |x_i| |x_j| + 2^-16 of the value, padding zero;
      top tower + head: the device split operand -> the predictions, _chain over [128, 64, 32] relu + sigmoid.
    The stage-wise predictions equal the replay bit for bit."""
    B, D = BIG, 64
    mm.set_seed(33)
    schema = datasets.criteo_schema({k: min(v, CAP - 1) for k, v in datasets.CRITEO_MAX.items()})
    model = mm.DLRMModel(schema, embedding_dim=D, bottom_block=mm.MLPBlock([128, 64]), top_block=mm.MLPBlock([128, 64, 32]))
    model.build(device)
    body = model.body
    assert body.use_operand_rows(), "premise: the production path with the operand-format mirrors"
    feats, _ = datasets.split_targets(schema, datasets.generate_batch(schema, B, seed=2024, index_law="uniform", index_dtype=np.int32))
    widths = model.id_bytes()
    assert sorted(set(widths.values())) == [1, 2, 3]
    hb = HostBatch.like(feats, model.input_columns(), id_bytes=widths)
    replay = model.compile(hb)(hb).to(device)
    x = {k: torch.from_numpy(np.asarray(feats[k]).astype(np.int64) if np.asarray(feats[k]).dtype.kind in "iu"
                             else np.asarray(feats[k])).to(device) for k in model.input_columns()}
    assert torch.equal(model(x), replay), "graph replay on packed ids differs from the eager forward on int64 ids"

    # the stages, as RankingModel.call runs them
    assert model._all_onehot(x)
    bottom = body.bottom_forward(x, operand_out=True)
    assert blocks.last_dense_path() == "tower2_small"
    a = body.interaction_forward(x, bottom, as_split=True, operand_rows=True)
    layers, tail = body.top_block.chain([model.prediction.to_call])
    assert tail is None
    K = body.output_width_before_top()
    pred = blocks.run_dense_chain(None, layers, a_split=a, K=K)
    assert blocks.last_dense_path() == "mlp_tc"
    assert torch.equal(pred, replay), "stage-wise forward differs from the graph replay"

    cont = body.continuous(x)
    x0 = torch.cat([cont[k].reshape(B, -1).float() for k in sorted(cont)], dim=1)
    bl, btail = body.bottom_block.chain()
    assert btail is None
    emb = body.embeddings
    slots = body.slots()
    F = len(slots)
    OW = D + F * (F - 1) // 2
    assert K == OW
    _split_padding_zero(a, B, OW, "interaction split operand")  # no guard rows here: the model allocates (B, 2 Kp)
    Kp = a.shape[1] // 2
    assert torch.equal(a[:, :D], bottom[:, :D]) and torch.equal(a[:, Kp:Kp + D], bottom[:, D:]), "prefix is not the bottom's rows"
    top = _layers(layers)
    for s, e in _chunks(B):
        # bottom tower
        h, eh = _chain(x0[s:e].double(), _layers(bl))
        bv = _unsplit(bottom[s:e], D)
        _within(bv, h, eh + SPLIT * (h.abs() + eh), f"bottom tower rows [{s}, {e})")
        # interaction from the device bottom
        st = torch.empty((e - s, F, D), dtype=torch.float64, device=device)
        for f in emb.feature_names:
            t = emb.feature_to_table[f].table
            i = x[f][s:e].reshape(-1)
            st[:, slots[f]] = t[i].double()
        st[:, slots["bottom_block"]] = bv
        z, za = _interaction_fwd(st, F, D)
        _within(_unsplit(a[s:e], OW)[:, D:], z, (U + D * E) * za + SPLIT * z.abs(), f"interaction rows [{s}, {e})")
        # top tower + head from the device operand
        y, ey = _chain(_unsplit(a[s:e], OW), top)
        _within(pred[s:e], y, ey, f"predictions rows [{s}, {e})")
