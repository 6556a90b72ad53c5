"""The DeepFM training step on the GPU: mm_deepfm_head_fwd_bwd, mm_fm_concat_backward and mm_wide_rows_apply against
float64 references, then DeepFMTrainer against the restatement (tests/deepfm_train_oracle.py) with the Keras update rules.

Tolerances of the kernel tests are per element and derived from fp32 summation: a sum of n terms computed in fp32, in any
order, is within n u sum|terms| of the exact sum (u = 2^-24).  The pairwise term 0.5 (S^2 - sum e^2) cancels, so its bound
scales with S^2 + sum e^2, not with the result."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import ops
from tests import helpers as H
from tests.deepfm_train_oracle import BCE, MSE, deepfm_loss_and_grads
from tests.test_deepfm_train_host import CATS, CONTS, rejections, schema

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -24
TOL = 3e-4
INT32_MAX = 2 ** 31 - 1


def close(got, ref, tol=TOL, what=""):
    got = np.asarray(got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got, dtype=np.float64)
    ref = np.asarray(ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref, dtype=np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    scale = max(float(np.max(np.abs(ref))), 1e-30)
    err = float(np.max(np.abs(got - ref))) / scale
    assert err < tol, f"{what}: max |diff| / max |ref| = {err:.3e} (tol {tol})"


def within(got, ref, bound, what):
    got, ref, bound = (t.double().reshape(-1) for t in (got, ref, bound))
    bad = (got - ref).abs() > bound
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements outside the bound, e.g. got {got[bad][:3].tolist()} want {ref[bad][:3].tolist()}"


def packed_ids(ids: np.ndarray, width: int, device) -> torch.Tensor:
    """ids as the column form of `width` bytes (index_bytes_of): uint8, uint16, uint8 (B, 3), int32, int64."""
    if width == 1:
        return torch.from_numpy(ids.astype(np.uint8)).to(device)
    if width == 2:
        return torch.from_numpy(ids.astype(np.uint16)).to(device)
    if width == 3:
        u = ids.astype(np.uint32)
        return torch.from_numpy(np.stack([u & 255, (u >> 8) & 255, (u >> 16) & 255], 1).astype(np.uint8)).to(device)
    return torch.from_numpy(ids.astype(np.int32 if width == 4 else np.int64)).to(device)


# ---------------------------------------------------------------------------------------------------------------
# mm_deepfm_head_fwd_bwd
# ---------------------------------------------------------------------------------------------------------------
def _head_case(device, B, T, D, C, loss, use_sw, act_dl, U=40, seed=0):
    """Random inputs of the head kernel: x0 with T feature slices of width D at unaligned columns and a continuous column
    between features, ids of every width (about 10 % outside [0, rows): their x0 slice is zero, as the gather leaves it),
    C continuous columns of mixed dtypes."""
    g = np.random.default_rng(seed)
    widths = [(1, 2, 3, 4, 8)[f % 5] for f in range(T)]
    rows = [int(g.integers(60, 230)) for _ in range(T)]  # ids up to rows + rows // 10 < 256: the 1-byte columns hold them
    cols, c = [], 1
    for f in range(T):
        cols.append(c)
        c += D + (1 if f < C else 0)
    d = c + 2
    x0 = torch.from_numpy(g.standard_normal((B, d + 3)).astype(np.float32) * 0.5).to(device)[:, :d]
    ids_np = [g.integers(0, r + r // 10, B) for r in rows]
    for f in range(T):
        if widths[f] >= 4:
            ids_np[f][::17] = -1
        bad = torch.from_numpy((ids_np[f] < 0) | (ids_np[f] >= rows[f])).to(device)
        x0[:, cols[f]:cols[f] + D][bad] = 0.0
    ids = [packed_ids(i, w, device) for i, w in zip(ids_np, widths)]
    woff, o = [], 0
    for r in rows:
        woff.append(o)
        o += r
    coff = [o + k for k in range(C)]
    W = o + C
    wide = torch.from_numpy(g.standard_normal(W).astype(np.float32) * 0.3).to(device)
    dts = [torch.float32, torch.float64, torch.int32, torch.int64]
    cont = []
    for k in range(C):
        v = g.standard_normal(B) * 2
        cont.append(torch.from_numpy(v).to(device).to(dts[k % 4]) if dts[k % 4].is_floating_point
                    else torch.from_numpy(np.round(v).astype(np.int64)).to(device).to(dts[k % 4]))
    h = torch.from_numpy(np.maximum(g.standard_normal((B, U)), 0).astype(np.float32)).to(device)
    f32 = lambda *s: torch.from_numpy(g.standard_normal(s).astype(np.float32) * 0.4).to(device)  # noqa: E731
    p = dict(x0=x0, cols=cols, D=D, ids=ids, ids_np=ids_np, rows=rows, woff=woff, cont=cont, coff=coff, wide=wide, bw=f32(1), h=h,
             w_dl=f32(U), b_dl=f32(1), act_dl=act_dl, out_w=f32(1) + 1.0, out_b=f32(1), loss=loss)
    if loss == BCE:
        p["y"] = torch.from_numpy(g.integers(0, 2, B)).to(device)
    else:
        p["y"] = torch.from_numpy(g.standard_normal(B).astype(np.float32)).to(device)
    p["sw"] = torch.from_numpy(g.random(B).astype(np.float32) * 2).to(device) if use_sw else None
    return p


def _head_ref(p):
    """float64 head: (z, s, ds, du, loss sum, per-sample scale of s's fp32 error bound, n terms)."""
    x0, D = p["x0"].double(), p["D"]
    B = x0.shape[0]
    pair = torch.zeros(B, dtype=torch.float64, device=x0.device)
    mag = torch.zeros_like(pair)
    for c in p["cols"]:
        e = x0[:, c:c + D]
        S = e.sum(1)
        pair += 0.5 * (S * S - (e * e).sum(1))
        mag += 0.5 * (S * S + (e * e).sum(1)) + e.abs().sum(1) * S.abs()
    wide = p["bw"].double().expand(B).clone()
    for i, r, o in zip(p["ids_np"], p["rows"], p["woff"]):
        it = torch.from_numpy(i).to(x0.device)
        ok = (it >= 0) & (it < r)
        term = torch.where(ok, p["wide"].double()[(it.clamp(0, r - 1) + o)], torch.zeros_like(wide))
        wide += term
        mag += term.abs()
    for x, o in zip(p["cont"], p["coff"]):
        term = p["wide"].double()[o] * x.double().float().double()
        wide += term
        mag += term.abs()
    hw = p["h"].double() * p["w_dl"].double()
    u = hw.sum(1) + p["b_dl"].double()
    mag += hw.abs().sum(1) + p["b_dl"].double().abs() + p["bw"].double().abs()
    relu = p["act_dl"] == "relu"
    s = pair + wide + (u.clamp(min=0) if relu else u)
    wo, bo = p["out_w"].double(), p["out_b"].double()
    z = s * wo + bo
    y = p["y"].double()
    sw = p["sw"].double() if p["sw"] is not None else torch.ones_like(z)
    if p["loss"] == BCE:
        per, gz = z.clamp(min=0) - z * y + torch.log1p(torch.exp(-z.abs())), torch.sigmoid(z) - y
    else:
        per, gz = (z - y) ** 2, 2 * (z - y)
    delta = gz * sw / B
    ds = delta * wo
    du = torch.where(u > 0, ds, torch.zeros_like(ds)) if relu else ds
    n = len(p["cols"]) * D + len(p["cols"]) + len(p["cont"]) + p["h"].shape[1] + 8
    return dict(z=z, s=s, ds=ds, du=du, delta=delta, gz=gz, loss=(per * sw).sum() / B, mag=mag, n=n, sw=sw, u=u)


def _run_head(p, B, guard=2):
    dev = p["x0"].device
    U = p["h"].shape[1]
    nan = float("nan")
    logits, ds = torch.full((B + guard,), nan, device=dev), torch.full((B + guard,), nan, device=dev)
    dh = torch.full((B + guard, U), nan, device=dev)
    acc = {k: torch.zeros(n, device=dev) for k, n in (("loss", 2), ("dw_out", 1), ("db_out", 1), ("dw_dl", U), ("db_dl", 1), ("dbw", 1),
                                                      ("dcont", max(len(p["cont"]), 1)))}
    oob = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.deepfm_head_fwd_bwd(p["x0"], p["cols"], p["D"], p["ids"], p["rows"], p["woff"], p["cont"], p["coff"], p["wide"], p["bw"], p["h"],
                            True, p["w_dl"], p["b_dl"], p["act_dl"], p["out_w"], p["out_b"], p["loss"], p["y"], p["sw"], logits[:B],
                            acc["loss"], ds[:B], dh[:B], dw_out=acc["dw_out"], db_out=acc["db_out"], dw_dl=acc["dw_dl"], db_dl=acc["db_dl"],
                            d_wide_bias=acc["dbw"], d_cont=acc["dcont"][:len(p["cont"])] if p["cont"] else None, oob=oob)
    assert torch.isnan(logits[B:]).all() and torch.isnan(ds[B:]).all() and torch.isnan(dh[B:]).all(), "a guard row was written"
    return logits[:B], ds[:B], dh[:B], acc, oob


def _check_head(p, B):
    r = _head_ref(p)
    logits, ds, dh, acc, oob = _run_head(p, B)
    want_oob = sum(int(((i < 0) | (i >= rw)).sum()) for i, rw in zip(p["ids_np"], p["rows"]))
    assert int(oob.item()) == want_oob
    wo = p["out_w"].double().abs()
    # s and z: n u (sum of |terms|), the pairwise terms counted at S^2 + sum e^2
    err_s = r["n"] * U32 * r["mag"] + 1e-30
    err_z = err_s * wo + 4 * U32 * r["z"].abs()
    within(logits, r["z"], err_z, "z")
    # ds = delta w_out, dl/dz Lipschitz in z with constant 1/4 (BCE) or 2 (MSE)
    lip = 0.25 if p["loss"] == BCE else 2.0
    err_ds = (lip * err_z + 8 * U32 * (r["delta"].abs() * p["x0"].shape[0] + 1)) * r["sw"] / p["x0"].shape[0] * wo + 4 * U32 * r["ds"].abs()
    within(ds, r["ds"], err_ds, "ds")
    relu = p["act_dl"] == "relu"
    flip = (r["u"].abs() <= err_s) if relu else torch.zeros_like(r["u"], dtype=torch.bool)  # u within its error of 0
    h = p["h"].double()
    want_dh = r["du"][:, None] * p["w_dl"].double()[None, :] * (h > 0)
    err_dh = err_ds[:, None] * p["w_dl"].double().abs()[None, :] + 4 * U32 * want_dh.abs()
    keep = ~flip
    within(dh[keep], want_dh[keep], err_dh[keep], "dh")
    # reductions over the batch: sum of per-sample bounds + B u sum |terms|
    Bn = p["x0"].shape[0]

    def red(got, terms, errs, what):
        within(got, terms.sum(0), errs.sum(0) + Bn * U32 * terms.abs().sum(0) + 1e-30, what)

    red(acc["dw_out"], r["delta"] * r["s"], (err_ds / wo) * r["s"].abs() + r["delta"].abs() * err_s, "dW_out")
    red(acc["db_out"], r["delta"], err_ds / wo, "db_out")
    red(acc["dbw"], r["ds"], err_ds, "d wide bias")
    if not relu or not bool(flip.any()):
        red(acc["dw_dl"], r["du"][:, None] * h, err_ds[:, None] * h, "dw_dl")
        red(acc["db_dl"], r["du"], err_ds, "db_dl")
    if p["cont"]:
        xs = torch.stack([x.double().float().double() for x in p["cont"]], 1)
        red(acc["dcont"], r["ds"][:, None] * xs, err_ds[:, None] * xs.abs(), "d continuous rows")
    # loss: per sample |dl/dz| err_z + lip err_z^2 (+ the log1p / square rounding), summed in fp32
    err_l = ((r["gz"].abs() * err_z + lip * err_z ** 2) * r["sw"]).sum() / Bn
    for k in (0, 1):  # the total and the output's loss: the same sums, accumulated in different atomic orders
        assert abs(float(acc["loss"][k]) - float(r["loss"])) <= float(err_l) + 8 * Bn * U32 * abs(float(r["loss"])) + 1e-12


@pytest.mark.parametrize("T,D", [(1, 4), (26, 16), (32, 64), (5, 128)])
@pytest.mark.parametrize("B", [1, 37, 1000])
@pytest.mark.parametrize("C", [0, 13])
def test_head_matches_float64(device, T, D, B, C):
    for k, (loss, sw, act) in enumerate([(BCE, False, "linear"), (MSE, True, "relu")]):
        _check_head(_head_case(device, B, T, D, C, loss, sw, act, seed=T * 1000 + D + B + C + k), B)


@pytest.mark.parametrize("loss,sw,act", [(BCE, True, "relu"), (MSE, False, "linear")])
def test_head_other_losses_and_deep_logits(device, loss, sw, act):
    _check_head(_head_case(device, 500, 26, 16, 13, loss, sw, act, seed=3), 500)


# ---------------------------------------------------------------------------------------------------------------
# mm_fm_concat_backward
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [4, 12, 16, 64, 128])
@pytest.mark.parametrize("n_add", [0, 1, 2])
def test_fm_input_backward_matches_float64(device, D, n_add):
    """Unaligned column offsets with a continuous column between features; continuous columns are never written."""
    g = np.random.default_rng(D + n_add)
    T, B = 7, 301
    cols, c = [], 0
    for _ in range(T):
        c += 1
        cols.append(c)
        c += D
    d = c + 1
    x0 = torch.from_numpy(g.standard_normal((B, d + 5)).astype(np.float32)).to(device)[:, :d]
    adds = [torch.from_numpy(g.standard_normal((B, d + 4 * i)).astype(np.float32)).to(device)[:, :d] for i in range(n_add)]
    ds = torch.from_numpy(g.standard_normal(B).astype(np.float32)).to(device)
    dst = [torch.full((B + 1, D + 4), float("nan"), device=device) for _ in range(T)]
    ops.fm_concat_backward(adds, x0, ds, [(t[:B, :D], col) for t, col in zip(dst, cols)])
    for t, col in zip(dst, cols):
        e = x0[:, col:col + D].double()
        want = ds.double()[:, None] * (e.sum(1, keepdims=True) - e) + sum((a[:, col:col + D].double() for a in adds), torch.zeros_like(e))
        # S: D terms, then one product and n_add additions
        bound = (D + n_add + 2) * U32 * (ds.double().abs()[:, None] * (e.abs().sum(1, keepdims=True) + e.abs())
                                         + sum((a[:, col:col + D].double().abs() for a in adds), torch.zeros_like(e)))
        within(t[:B, :D], want, bound + 1e-30, f"slice at column {col}")
        assert torch.isnan(t[B:]).all() and torch.isnan(t[:, D:]).all(), "a guard row / column was written"


# ---------------------------------------------------------------------------------------------------------------
# mm_wide_rows_apply
# ---------------------------------------------------------------------------------------------------------------
def _sparse_ref(opt, w, ids, vals, state, lr, step):
    from oracle import oracle_train

    return oracle_train.sparse_update(opt, w, ids, vals, state, lr, beta_1=float(np.float32(0.9)), beta_2=float(np.float32(0.999)),
                                      epsilon=float(np.float32(1e-7)), step=step)


def _wide_setup(device, opt, block_rows, id_widths, n_cont=2, seed=0):
    g = np.random.default_rng(seed)
    offs, o, coff = [], 0, []
    for r in block_rows:
        offs.append(o)
        o += r
        if len(coff) < n_cont:
            coff.append(o)
            o += 1
    W = o
    w0 = g.standard_normal(W).astype(np.float32)
    f32 = dict(dtype=torch.float32, device=device)
    st = dict(w=torch.from_numpy(w0).to(device), s1=None, s2=None, bias=torch.tensor([0.3], **f32), bs1=None, bs2=None)
    if opt != "sgd":
        st["s1"] = torch.full((W,), 0.1, **f32) if opt == "adagrad" else torch.zeros(W, **f32)
        st["bs1"] = torch.full((1,), 0.1, **f32) if opt == "adagrad" else torch.zeros(1, **f32)
    if opt == "adam":
        st["s2"], st["bs2"] = torch.zeros(W, **f32), torch.zeros(1, **f32)
    st.update(acc=torch.zeros(W, **f32), rep=ops.fill_i32(torch.empty(W, dtype=torch.int32, device=device), INT32_MAX), offs=offs, coff=coff,
              W=W, rows=list(block_rows), widths=list(id_widths), dgrad=torch.zeros(n_cont + 1, **f32))
    hyper = torch.zeros(8, **f32)
    hyper[0], hyper[1], hyper[2], hyper[3] = 0.05, 0.9, 0.999, 1e-7
    return st, hyper, g


def _wide_ids(g, B, rows, law, width):
    if law == "zipf":
        ids = np.minimum(g.zipf(1.2, B) - 1, rows + 3)
    else:
        ids = g.integers(0, rows, B)
    ids[5] = rows + 2  # outside [0, rows): dropped
    if width >= 4:
        ids[6] = -1
    return ids


def _wide_steps(device, opt, law, block_rows, widths, B, steps=2, seed=0):
    st, hyper, g = _wide_setup(device, opt, block_rows, widths, seed=seed)
    W = st["W"]
    ref_w = st["w"].double().cpu().numpy().copy()
    slots = {"a": np.full(W, 0.1)} if opt == "adagrad" else ({"m": np.zeros(W), "v": np.zeros(W)} if opt == "adam" else {})
    bslots = {k: np.asarray(v[:1]).copy() for k, v in slots.items()}
    ref_b = np.array([0.3])
    w_start = st["w"].clone()
    s_start = [None if s is None else s.clone() for s in (st["s1"], st["s2"])]
    touched = np.zeros(W, dtype=bool)
    for step in range(1, steps + 1):
        ops.opt_tick(hyper)
        ids_np = [_wide_ids(g, B, r, law, w) for r, w in zip(block_rows, widths)]
        ids = [packed_ids(np.where(i < 0, 0, i) if w < 4 else i, w, device) for i, w in zip(ids_np, widths)]
        grad = g.standard_normal(B).astype(np.float32)
        dg = g.standard_normal(len(st["coff"]) + 1).astype(np.float32)
        st["dgrad"].copy_(torch.from_numpy(dg))
        ops.wide_rows_apply(opt, st["w"], st["s1"], st["s2"], ids, st["rows"], st["offs"], torch.from_numpy(grad).to(device), st["acc"], st["rep"],
                            st["coff"], st["dgrad"], st["bias"], st["bs1"], st["bs2"], hyper)
        # reference: one (rows, 1) IndexedSlices per block over the full kernel, then the dense rows
        all_ids, all_vals = [], []
        for i, r, o, w in zip(ids_np, block_rows, st["offs"], widths):
            ok = (i >= 0) & (i < r)
            all_ids.append(i[ok] + o)
            all_vals.append(grad[ok])
        all_ids = np.concatenate(all_ids)
        touched[all_ids] = True
        # the slot arrays are updated in place through these (W, 1) views
        ref_w = _sparse_ref(opt, ref_w[:, None], all_ids, np.concatenate(all_vals)[:, None], {k: v[:, None] for k, v in slots.items()},
                            0.05, step)[:, 0]
        for c, o in enumerate(st["coff"]):  # every step, by the dense rule
            touched[o] = True
            ref_w = _sparse_ref(opt, ref_w[:, None], np.array([o]), np.array([[dg[c]]]), {k: v[:, None] for k, v in slots.items()},
                                0.05, step)[:, 0]
        ref_b = _sparse_ref(opt, ref_b[:, None], np.array([0]), np.array([[dg[-1]]]), {k: v[:, None] for k, v in bslots.items()},
                            0.05, step)[:, 0]
    w = st["w"]
    unt = torch.from_numpy(~touched).to(device)
    assert torch.equal(w[unt], w_start[unt]), "an untouched row moved"
    for s, s0 in zip((st["s1"], st["s2"]), s_start):
        if s is not None:
            assert torch.equal(s[unt], s0[unt]), "an untouched row's slot moved"
    upd, upd_ref = (w.double() - w_start.double()).cpu().numpy(), ref_w - w_start.double().cpu().numpy()
    for o, r in zip(st["offs"], block_rows):
        close(upd[o:o + r], upd_ref[o:o + r], 2e-4, f"{opt} {law} update of the block of {r} rows")
    close(upd[st["coff"]], upd_ref[st["coff"]], 1e-5, "continuous rows")
    close(st["bias"].double() - 0.3, ref_b - 0.3, 1e-5, "bias")
    if opt == "adagrad":
        close(st["s1"], slots["a"], 2e-4, "accumulator")
    assert not st["acc"].any() and torch.equal(st["rep"], torch.full_like(st["rep"], INT32_MAX)), "scratch not left idle"
    assert not st["dgrad"].any(), "the dense gradients were not cleared"
    return st


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
@pytest.mark.parametrize("law", ["uniform", "zipf"])
def test_wide_update_all_size_classes(device, opt, law):
    """Blocks of 3 and 1 500 rows (shared-memory pre-reduction), 60 000 (dense accumulator) and 300 000 (election) in one call,
    ids of 1, 2, 3 and 8 bytes with out-of-range ids, two steps; untouched rows and their slots stay bit-identical."""
    _wide_steps(device, opt, law, [3, 1500, 60000, 300000], [1, 2, 3, 8], B=5000)


# ---------------------------------------------------------------------------------------------------------------
# the training step
# ---------------------------------------------------------------------------------------------------------------
def _deepfm(seed=3, D=16, deep=(32, 16), logit=None, target="click"):
    mm.set_seed(seed)
    kw = {} if logit is None else dict(deep_logit_block=logit)
    return mm.DeepFMModel(schema(target=target), embedding_dim=D, deep_block=mm.MLPBlock(list(deep)), **kw)


def _batch(B, seed):
    g = np.random.default_rng(seed)
    f = {n: g.integers(0, mx + 1, B).astype(np.int64) for n, mx in CATS}
    f.update({n: g.standard_normal(B).astype(np.float32) for n in CONTS})
    y = (g.random(B) < 0.4).astype(np.int64)
    return f, y


def _state(model):
    body = model.body
    tables, f2t = H.emb_tables(body.input_block.embeddings)
    tables = {f: tables[t].astype(np.float64) for f, t in f2t.items()}
    fm = body.fm

    def lay(m):
        return [dict(l, kernel=l["kernel"].astype(np.float64), bias=l["bias"].astype(np.float64)) for l in H.mlp_layers(m)]

    hl = model.prediction.to_call
    head = {"kernel": H.to_numpy(hl.kernel).astype(np.float64), "bias": H.to_numpy(hl.bias).astype(np.float64),
            "loss": MSE if isinstance(model.prediction, mm.RegressionOutput) else BCE}
    return dict(tables=tables, wk=H.to_numpy(fm.wide.kernel).astype(np.float64), wb=H.to_numpy(fm.wide.bias).astype(np.float64),
                deep=lay(body.deep), logit=lay(body.deep_logit), head=head, offsets=dict(fm.wide_offsets))


def _clear_batch(st, B, seed):
    """The first batch from `seed` on whose relu pre-activations (float64, restated weights) all lie outside their device
    error bound: the split-bf16 products are within 2^-16 of sum |x||w| per element, and the input's own error (of the same
    relative size) adds about as much again; 2^-14 sum |x||w| is taken.  A pre-activation within that bound of 0 may take the other side of the relu on
    the device and move the deep layers' gradients by one sample's share — a property of the input, not of the kernels."""
    for s in range(seed, seed + 400):
        feats, y = _batch(B, s)
        cols = {n: st["tables"][n][feats[n]] for n in st["tables"]}
        cols.update({n: feats[n].astype(np.float64)[:, None] for n in CONTS})
        h = np.concatenate([cols[n] for n in sorted(cols)], 1)
        ok = True
        for l in st["deep"] + st["logit"][:-1]:
            W, b = l["kernel"], l["bias"]
            pre = h @ W + b
            err = 2.0 ** -14 * (np.abs(h) @ np.abs(W) + np.abs(b))
            ok = ok and (l["activation"] != "relu" or bool(((np.abs(pre) > err) | (err == 0)).all()))  # err 0: exact on the device too
            h = np.maximum(pre, 0) if l["activation"] == "relu" else pre
        if ok:
            return feats, y
    raise AssertionError("no batch without relu inputs within their error bound of 0")


def _restated(st, feats, y, sw=None):
    return deepfm_loss_and_grads(feats, st["tables"], CONTS, st["offsets"], st["wk"], st["wb"], st["deep"], st["logit"], st["head"], y,
                                 sample_weight=sw)


@pytest.mark.parametrize("case", ["bce", "mse-sw", "relu-logit"])
def test_step_gradients_match_the_restatement(device, case):
    """Loss and every gradient of one step at 3e-4 of each tensor's scale: tables, wide kernel, wide bias, deep layers, deep
    logit, output layer."""
    B = 160
    if case == "mse-sw":
        model = _deepfm(target="rating")
    elif case == "relu-logit":
        model = _deepfm(logit=mm.MLPBlock([8, 1], activation="relu"))
    else:
        model = _deepfm()
    model.build(device)
    st = _state(model)
    feats, y = _clear_batch(st, B, 11)
    sw = None
    if case == "mse-sw":
        y = np.random.default_rng(1).random(B).astype(np.float32) * 3
        sw = np.random.default_rng(2).random(B).astype(np.float32)
    model.compile(optimizer=mm.SGD(0.0))
    tr = model.trainer(B)
    assert type(tr).__name__ == "DeepFMTrainer"
    tr.forward_backward(H.device_batch(feats, device), torch.from_numpy(y).to(device),
                        None if sw is None else torch.from_numpy(sw).to(device))
    loss, z, grads = _restated(st, feats, y, sw)
    np.testing.assert_allclose(tr.loss[0].item(), loss, rtol=1e-5)
    close(tr.logits[:B], z, what="logits")
    got = tr.gradients()
    names = [("deep", i) for i in range(len(st["deep"]))] + [("deep_logit", i) for i in range(len(st["logit"]))]
    for l, (grp, i) in zip(tr.arena.layers[:-1], names):
        close(got[f"{l.name}/kernel"], grads[f"{grp}/kernel_{i}"], what=f"{grp} kernel {i}")
        close(got[f"{l.name}/bias"], grads[f"{grp}/bias_{i}"], what=f"{grp} bias {i}")
    hl = model.prediction.to_call
    close(got[f"{hl.name}/kernel"], grads["head/kernel"], what="output kernel")
    close(got[f"{hl.name}/bias"], grads["head/bias"], what="output bias")
    wg = tr.wide_gradients()
    close(wg["wide/kernel"], grads["wide/kernel"], what="wide kernel")
    close(wg["wide/bias"], grads["wide/bias"], what="wide bias")
    for t, f in enumerate(tr.feats):
        dense = torch.zeros(tr.tables[t].table.shape, dtype=torch.float64, device=device)
        dense.index_add_(0, tr._idx[t].long(), tr._slices[t].double())
        close(dense, grads[f"table/{f}"], what=f"table {f}")


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
def test_three_steps_match_the_restatement(device, opt):
    """Three optimizer steps (the last on a smaller batch) against the restatement + the Keras rules in float64; every
    variable's update in the Frobenius norm (0.1) and elementwise at 0.5 of its largest element, as the DCN step."""
    from oracle import oracle_train

    model = _deepfm()
    model.build(device)
    st = _state(model)
    lr = {"sgd": 0.5, "adagrad": 0.05, "adam": 0.01}[opt]
    eps = 1e-6 if opt == "adam" else 1e-7
    model.compile(optimizer={"sgd": mm.SGD(lr), "adagrad": mm.Adagrad(lr), "adam": mm.Adam(lr, epsilon=eps)}[opt])
    model.trainer(300)

    def slots(shape):
        if opt == "adagrad":
            return {"a": np.full(shape, 0.1)}
        return {"m": np.zeros(shape), "v": np.zeros(shape)} if opt == "adam" else {}

    def flat(s):
        out = [s["tables"][f] for f in sorted(s["tables"])] + [s["wk"], s["wb"]]
        for l in s["deep"] + s["logit"]:
            out += [l["kernel"], l["bias"]]
        return out + [s["head"]["kernel"], s["head"]["bias"]]

    before = [np.array(v) for v in flat(st)]
    tslots = {f: slots(t.shape) for f, t in st["tables"].items()}
    wslots, bslots, dslots = slots(st["wk"].shape), slots(st["wb"].shape), {}
    cont_rows = np.array([st["offsets"][c] for c in CONTS])
    for step, B in ((1, 300), (2, 300), (3, 170)):
        feats, y = _batch(B, 100 + step)
        m = model.train_step((H.device_batch(feats, device), torch.from_numpy(y).to(device)))
        loss, _, grads = _restated(st, feats, y)
        np.testing.assert_allclose(m["loss"].item(), loss, rtol=1e-4)
        kw = dict(beta_1=0.9, beta_2=0.999, epsilon=eps, step=step)
        for f in st["tables"]:
            uniq = np.unique(feats[f])
            st["tables"][f] = oracle_train.sparse_update(opt, st["tables"][f], uniq, grads[f"table/{f}"][uniq], tslots[f], lr, **kw)
        rows = np.unique(np.concatenate([feats[f] + st["offsets"][f] for f in st["tables"]] + [cont_rows]))
        st["wk"] = oracle_train.sparse_update(opt, st["wk"], rows, grads["wide/kernel"][rows], wslots, lr, **kw)
        st["wb"] = oracle_train.dense_update(opt, st["wb"], grads["wide/bias"], bslots, lr, **kw)
        for grp, ls in (("deep", st["deep"]), ("deep_logit", st["logit"])):
            for i, l in enumerate(ls):
                for what in ("kernel", "bias"):
                    key = f"{grp}/{what}_{i}"
                    dslots.setdefault(key, slots(l[what].shape))
                    l[what] = oracle_train.dense_update(opt, l[what], grads[key], dslots[key], lr, **kw)
        for what in ("kernel", "bias"):
            key = f"head/{what}"
            dslots.setdefault(key, slots(st["head"][what].shape))
            st["head"][what] = oracle_train.dense_update(opt, st["head"][what], grads[key], dslots[key], lr, **kw)
    after = [np.asarray(v, dtype=np.float64) for v in flat(_state(model))]
    want = flat(st)
    for i, (a, w, b0) in enumerate(zip(after, want, before)):
        upd_ref = np.asarray(w, dtype=np.float64) - b0
        upd = a - b0
        if not np.any(upd_ref):
            assert not np.any(upd), i
            continue
        fro = float(np.linalg.norm(upd - upd_ref) / np.linalg.norm(upd_ref))
        assert fro < 0.1, f"update of variable {i} after 3 {opt} steps: relative Frobenius error {fro:.3e}"
        close(upd, upd_ref, 0.5, f"update of variable {i} after 3 {opt} steps")


def _packed(feats, device):
    """The categorical columns as the host batch packs them: 1-byte C3 / C7, 2-byte C1, 3-byte C5."""
    out = H.device_batch(feats, device)
    for n, w in (("C3", 1), ("C7", 1), ("C1", 2), ("C5", 3)):
        out[n] = packed_ids(feats[n], w, device)
    return out


def test_graph_replay_on_packed_ids_equals_eager_steps(device):
    ma, mb = _deepfm(seed=12), _deepfm(seed=12)
    ma.build(device), mb.build(device)
    ma.compile(optimizer=mm.Adagrad(0.05))
    mb.compile(optimizer=mm.Adagrad(0.05))
    B = 256
    batches = [_batch(B, 20 + s) for s in range(3)]
    ta, tb = ma.trainer(B), mb.trainer(B)
    w0 = mb.body.fm.wide.kernel.clone()
    tb.capture(_packed(batches[0][0], device), torch.from_numpy(batches[0][1]).to(device))
    assert tb.launches_per_step > 0
    assert torch.equal(mb.body.fm.wide.kernel, w0), "capture moved the wide kernel"
    for f, y in batches:
        la = ta.step(H.device_batch(f, device), torch.from_numpy(y).to(device)).clone()
        lb = tb.replay(_packed(f, device), torch.from_numpy(y).to(device)).clone()
        close(la, lb, 1e-5, "loss")
    for (na, va), (nb, vb) in zip(sorted(ma.weights().items()), sorted(mb.weights().items())):
        close(va, vb, 1e-4, na)


def test_trained_model_forward_save_and_load(device, tmp_path):
    """After training steps the model's forward (eager and a compiled graph) reads the trained variables, wide kernel
    included: it equals the trainer's logits on the next batch; save / load round-trips them."""
    from models_b200.graph import HostBatch

    model = _deepfm(seed=4)
    model.compile(optimizer=mm.Adam(0.01))
    for s in range(3):
        f, y = _batch(256, 40 + s)
        model.train_step((H.device_batch(f, device), torch.from_numpy(y).to(device)))
    w = model.body.fm.wide.kernel.clone()
    f, y = _batch(256, 50)
    tr = model.trainer(256)
    tr.forward_backward(H.device_batch(f, device), torch.from_numpy(y).to(device))
    p = model(H.device_batch(f, device)).reshape(-1)
    close(p, torch.sigmoid(tr.logits.double()), 1e-4, "forward vs the trainer's logits")
    close(p.cpu().numpy(), H.oracle_deepfm(model, f).reshape(-1), 2e-4, "forward vs the oracle")
    hb = HostBatch.like(f, model.input_columns())
    cf = model.compile(hb)
    close(np.asarray(cf(hb)).reshape(-1), p.cpu().numpy(), 1e-4, "compiled forward")
    model.save(tmp_path / "export")
    loaded = mm.Model.load(tmp_path / "export")
    assert torch.equal(loaded.body.fm.wide.kernel.to(device), w)
    np.testing.assert_array_equal(loaded(H.device_batch(f, device)).cpu().numpy().reshape(-1), p.cpu().numpy())


def test_fit_learns_a_planted_rule(device, tmp_path):
    import pyarrow as pa
    import pyarrow.parquet as pq

    n = 16000
    feats, _ = _batch(n, 1)
    rng = np.random.default_rng(0)
    s = (feats["C7"] % 2 == 0).astype(np.float32) * 2.0 + feats["C2"] * 1.5 - 1.0
    cols = dict(feats, click=(rng.random(n) < 1 / (1 + np.exp(-3 * s))).astype(np.int64))
    d = tmp_path / "data"
    d.mkdir()
    pq.write_table(pa.table(cols), d / "train.parquet")
    loader = mm.Loader(str(d), batch_size=2000, shuffle=True, schema=schema(), device=device)
    model = _deepfm(seed=5)
    model.compile(optimizer=mm.Adam(0.01))
    hist = model.fit(loader, epochs=5).history["loss"]
    assert len(hist) == 5 and hist[-1] < 0.9 * hist[0], hist
    held, _ = _batch(4000, 2)
    sh = (held["C7"] % 2 == 0).astype(np.float32) * 2.0 + held["C2"] * 1.5 - 1.0
    p = model(H.device_batch(held, device)).cpu().numpy().reshape(-1)
    assert np.corrcoef(p, sh)[0, 1] > 0.6


def test_unsupported_configurations_name_their_cause(device):
    f, y = _batch(64, 3)
    x, yt = H.device_batch(f, device), torch.from_numpy(y).to(device)
    for model, match, group in rejections(device):
        model.build(device)
        model.compile(optimizer="sgd")
        with pytest.raises(NotImplementedError, match=match):
            if group is None:
                model.train_step((x, yt))
            else:
                model.trainer(64, group=group)
    from models_b200.blocks import set_dense_engine

    set_dense_engine("fp32")
    try:
        m = _deepfm()
        m.compile(optimizer="sgd")
        with pytest.raises(NotImplementedError, match="fp32"):
            m.train_step((x, yt))
    finally:
        set_dense_engine("auto")
    m = _deepfm()
    m.compile(optimizer="sgd")
    with pytest.raises(NotImplementedError, match="'C3'.*multi-hot"):
        m.train_step((dict(x, C3=torch.zeros((64, 3), dtype=torch.int64, device=device)), yt))


# ---------------------------------------------------------------------------------------------------------------
# at the benchmark's batch: several laps of every grid-stride loop
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [65536, 65536 + 37])
def test_head_and_wide_update_at_scale(device, B):
    """The Criteo shape (26 features, D = 16, 13 continuous columns) at the benchmark's batch; each kernel takes at least two
    laps of its grid-stride loop (from the launch formulas and the SM count)."""
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    head_warps = min((B + 7) // 8, 8 * sms) * 8
    assert (B + head_warps - 1) // head_warps >= 2
    _check_head(_head_case(device, B, 26, 16, 13, BCE, True, "linear", seed=B), B)
    T = 26
    chunks = (B + 2047) // 2048
    sx = min(chunks, max(1, 2 * sms // T))
    ax = min((B + 255) // 256, max(1, 4 * sms // T))
    assert (chunks + sx - 1) // sx >= 2 and (B + 256 * ax - 1) // (256 * ax) >= 2
    rows = [3, 4, 10, 100, 500, 1500, 2100, 5000, 8000, 20000, 60000, 131072, 140000, 300000, 1000000] + [2000] * 11
    widths = [1, 1, 1, 1, 2, 2, 2, 2, 2, 2, 3, 3, 3, 3, 8] + [2] * 11
    _wide_steps(device, "adagrad", "zipf", rows, widths, B=B, steps=1, seed=B)
