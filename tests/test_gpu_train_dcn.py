"""The DCN-v2 training step on the GPU: mm_cross_backward, mm_concat_backward and mm_sparse_rows_apply at the widths
InputBlockV2 infers against float64 restatements, then DCNTrainer against the reference's torch DCNModel step
(tests/golden/dcn_train/ref_torch_dcn_train.npz) and against tests/dcn_train_oracle.py with the Keras update rules."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import ops
from models_b200.schema import ColumnSchema, Schema, Tags
from tests import helpers as H

pytestmark = pytest.mark.gpu
TOL = 3e-4
GOLDEN = __import__("pathlib").Path(__file__).parent / "golden" / "dcn_train" / "ref_torch_dcn_train.npz"


def close(got, ref, tol=TOL, what=""):
    got = np.asarray(got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got, dtype=np.float64)
    ref = np.asarray(ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref, dtype=np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    scale = max(float(np.max(np.abs(ref))), 1e-30)
    err = float(np.max(np.abs(got - ref))) / scale
    assert err < tol, f"{what}: max |diff| / max |ref| = {err:.3e} (tol {tol})"


def _strided(B, d, device, g, extra=4):
    """(B, d) fp32 view of a (B, round4(d) + extra) buffer: a row stride that is a multiple of 4 but not d."""
    ld = (d + 3) // 4 * 4 + extra
    buf = torch.from_numpy(g.standard_normal((B, ld)).astype(np.float32)).to(device)
    return buf[:, :d]


# ---------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [1, 7, 37, 1037])
@pytest.mark.parametrize("B", [1, 33, 4096])
@pytest.mark.parametrize("top", [True, False])
def test_cross_backward_matches_float64(device, d, B, top):
    g_ = np.random.default_rng(d * 7 + B)
    x0, z, g, acc, p = (_strided(B, d, device, g_, extra=4 * i) for i in range(5))
    dz = _strided(B, d, device, g_)
    Kp = ops.tc_padded_k(d)
    dz_split = torch.full((B, 2 * Kp), 7.0, dtype=torch.bfloat16, device=device)  # padding must be overwritten with zeros
    g0, acc0 = g.double().clone(), acc.double().clone()
    ops.cross_backward(x0, z, g, None if top else p, acc, top, dz, dz_split)
    want_g = g0 if top else g0 + p.double()
    close(g, want_g, 1e-6, "g")
    close(dz, want_g * x0.double(), 1e-6, "dz")
    close(acc, want_g * z.double() + (0 if top else acc0), 1e-6, "acc")
    assert torch.equal(dz_split, ops.split_rows(dz)), "dz_split is not mm_split_rows(dz)"


@pytest.mark.parametrize("n_add", [1, 3, 4])
def test_concat_backward_odd_offsets_every_width(device, n_add):
    """Every width 4..128 at odd column offsets (a width-1 continuous column before each table), continuous dropped."""
    g_ = np.random.default_rng(n_add)
    widths = list(range(4, 129, 4))
    cols, c = [], 0
    for w in widths:
        c += 1  # a continuous column
        cols.append(c)
        c += w
    d, B = c + 1, 65
    adds = [_strided(B, d, device, g_, extra=4 * i) for i in range(n_add)]
    dsts = [torch.full((B, w), float("nan"), device=device) for w in widths]
    ops.concat_backward(adds, list(zip(dsts, cols)))
    tot = sum(a.double() for a in adds)
    for dst, col, w in zip(dsts, cols, widths):
        close(dst, tot[:, col:col + w], 1e-6, f"width {w} at column {col}")


def _sparse_ref(opt, w, ids, vals, state, lr, step):
    from oracle import oracle_train

    # the device holds the hyper-parameters as fp32: 1 - fp32(0.999) differs from 0.001 by 1.3e-5 relative
    return oracle_train.sparse_update(opt, w, ids, vals, state, lr, beta_1=float(np.float32(0.9)), beta_2=float(np.float32(0.999)),
                                      epsilon=float(np.float32(1e-7)), step=step)


@pytest.mark.parametrize("D", [12, 24, 40, 48, 96, 120])
@pytest.mark.parametrize("path", ["elect", "mid", "small"])
@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
def test_sparse_apply_inferred_widths(device, D, path, opt):
    g_ = np.random.default_rng(D)
    rows = 50 if path == "small" else 5000
    B = 700
    w0 = g_.standard_normal((rows, D)).astype(np.float32)
    ids = g_.integers(0, rows, B).astype(np.int64)
    ids[:40] = ids[0]  # duplicates
    ids[40] = rows + 3  # out of range: dropped
    ids[41] = -2
    vals = g_.standard_normal((B, D)).astype(np.float32)
    w = torch.from_numpy(w0).to(device)
    s1 = None if opt == "sgd" else (torch.full_like(w, 0.1) if opt == "adagrad" else torch.zeros_like(w))
    s2 = torch.zeros_like(w) if opt == "adam" else None
    hyper = torch.zeros(8, dtype=torch.float32, device=device)
    hyper[0], hyper[1], hyper[2], hyper[3] = 0.05, 0.9, 0.999, 1e-7
    ops.opt_tick(hyper)
    rep = ops.fill_i32(torch.empty(rows, dtype=torch.int32, device=device), 2**31 - 1)
    tab = dict(weights=w, indices=torch.from_numpy(ids).to(device), grad_rows=torch.from_numpy(vals).to(device), rep_map=rep,
               state1=s1, state2=s2, dense_grad=torch.zeros_like(w) if path != "elect" else None)
    ops.sparse_rows_apply(opt, [tab], B, D, hyper)
    state = {"a": np.full((rows, D), 0.1)} if opt == "adagrad" else ({"m": np.zeros((rows, D)), "v": np.zeros((rows, D))} if opt == "adam" else {})
    want = _sparse_ref(opt, w0, ids, vals, state, 0.05, 1)
    close(w, want, 1e-5, f"weights D={D} {path} {opt}")
    if opt == "adagrad":
        close(s1, state["a"], 1e-5, "accumulator")
    if opt == "adam":
        close(s1, state["m"], 1e-5, "m")
        close(s2, state["v"], 1e-5, "v")
    assert torch.equal(rep, torch.full_like(rep, 2**31 - 1)) or path != "elect"  # the election map is left idle


def test_malformed_arguments_are_rejected_before_any_launch(device):
    """Every one of these fails a host-side check of the entry point, so no kernel ever sees the bad arguments."""
    f32 = dict(dtype=torch.float32, device=device)
    B, d = 8, 10
    x = torch.zeros((B, 12), **f32)[:, :d]
    dz_split = torch.zeros((B, 2 * ops.tc_padded_k(d)), dtype=torch.bfloat16, device=device)
    odd = torch.zeros((B, 13), **f32)[:, :d]  # row stride 13: not a multiple of 4
    n0 = ops.launch_count()
    with pytest.raises(ValueError, match="multiples of 4"):
        ops.cross_backward(x, x, x, None, x, True, odd, dz_split)
    lib = ops._lib()
    rc = lib.mm_cross_backward(x.data_ptr(), 12, x.data_ptr(), 12, x.data_ptr(), 12, None, 0, x.data_ptr(), 12, 1, B, d,
                               x.data_ptr(), 12, dz_split.data_ptr(), 128, None)  # Kp != mm_tc_padded_k(d)
    assert rc != 0
    with pytest.raises(ValueError, match="multiple of 4"):
        ops.concat_backward([x], [(torch.zeros((B, 6), **f32), 0)])  # width 6
    with pytest.raises(ValueError, match="outside"):
        ops.concat_backward([x], [(torch.zeros((B, 8), **f32), 4)])  # columns 4..12 > d
    hyper = torch.zeros(8, **f32)
    for D, mirror in ((6, False), (132, False), (24, True)):
        w = torch.zeros((16, D), **f32)
        tab = dict(weights=w, indices=torch.zeros(B, dtype=torch.int64, device=device), grad_rows=torch.zeros((B, D), **f32),
                   rep_map=torch.zeros(16, dtype=torch.int32, device=device),
                   mirror=torch.zeros((16, 2 * D), dtype=torch.bfloat16, device=device) if mirror else None)
        with pytest.raises((ValueError, RuntimeError), match="mirror" if mirror else "D="):
            ops.sparse_rows_apply("sgd", [tab], B, D, hyper)
    assert ops.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------
# the training step
# ---------------------------------------------------------------------------------------------------------------
# widths 16, 24, 32, 8, 48 (inferred), interleaved with continuous columns: unaligned table offsets, d = 132
CATS = [("C1", 300), ("C3", 5000), ("C5", 40000), ("C7", 7), ("C9", 200000)]
CONTS = ["C2", "C4", "C6", "C8"]


def _schema(targets=("click",)):
    cols = [ColumnSchema(n, tags=(Tags.CATEGORICAL,), dtype="int64", properties={"domain": {"min": 0, "max": mx, "name": n}})
            for n, mx in CATS]
    cols += [ColumnSchema(n, tags=(Tags.CONTINUOUS,), dtype="float32") for n in CONTS]
    for t in targets:
        if t in ("rating", "dwell", "watch_time"):
            cols.append(ColumnSchema(t, tags=(Tags.TARGET, Tags.REGRESSION), dtype="float32"))
        else:
            cols.append(ColumnSchema(t, tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"))
    return Schema(cols)


def _batch(B, seed, hot=True):
    g = np.random.default_rng(seed)
    f = {n: (g.integers(0, min(mx, 60) + 1, B) if hot else g.integers(0, mx + 1, B)).astype(np.int64) for n, mx in CATS}
    f.update({n: g.standard_normal(B).astype(np.float32) for n in CONTS})
    y = (g.random(B) < 0.4).astype(np.int64)
    return f, y


def _dcn(stacked=True, seed=3, depth=2, deep=(32, 16), targets=("click",), **kw):
    mm.set_seed(seed)
    schema = _schema(targets)
    pt = mm.OutputBlock(schema) if len(targets) > 1 else None
    return mm.DCNModel(schema, depth=depth, deep_block=mm.MLPBlock(list(deep)), stacked=stacked, prediction_tasks=pt, **kw)


def _oracle_state(model):
    body = model.body
    tables, f2t = H.emb_tables(body.input_block.embeddings)
    cross = [{"kernel": H.to_numpy(l.dense.kernel).astype(np.float64),
              "bias": None if l.dense.bias is None else H.to_numpy(l.dense.bias).astype(np.float64), "activation": "linear"}
             for l in body.cross.cross_layers]
    deep = [dict(l, kernel=l["kernel"].astype(np.float64), bias=l["bias"].astype(np.float64)) for l in H.mlp_layers(body.deep)]
    return {f: tables[t].astype(np.float64) for f, t in f2t.items()}, cross, deep


def test_dcn_widths_are_inferred_as_expected(device):
    model = _dcn()
    model.build(device)
    dims = model.body.input_block.embeddings.output_dims()
    assert dims == {"C1": 16, "C3": 24, "C5": 32, "C7": 8, "C9": 48}
    assert model.body.input_block.layout()[2] == 132


@pytest.mark.parametrize("tag", ["stacked", "parallel"])
def test_step_matches_the_reference_torch_dcn(device, tag):
    """Loss, prediction and every gradient of ONE step of the reference's torch DCNModel (inferred widths 16 / 24 / 48 / 8,
    unaligned table offsets) at 3e-4 of each tensor's scale."""
    z = np.load(GOLDEN)
    cats = [str(n) for n in z["cat_names"]]
    cols = [ColumnSchema(n, tags=(Tags.CATEGORICAL,), dtype="int64", properties={"domain": {"min": 0, "max": int(mx), "name": n}})
            for n, mx in zip(cats, z["cat_max"])]
    cols += [ColumnSchema(str(n), tags=(Tags.CONTINUOUS,), dtype="float32") for n in z["cont_names"]]
    cols.append(ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"))
    depth = 2 if tag == "stacked" else 1
    model = mm.DCNModel(Schema(cols), depth=depth, deep_block=mm.MLPBlock([16, 8]), stacked=tag == "stacked")
    model.build(device)
    emb = model.body.input_block.embeddings
    for f in cats:
        t = emb.feature_to_table[f]
        ids = torch.from_numpy(z[f"{tag}_table_{f}_ids"]).to(device)
        t.table[ids] = torch.from_numpy(z[f"{tag}_table_{f}_rows"]).to(device)
    for i, c in enumerate(model.body.cross.cross_layers):
        c.dense.set_weights(z[f"{tag}_cross_kernel_{i}"], z[f"{tag}_cross_bias_{i}"])
    for i, l in enumerate(model.body.deep.dense_layers):
        l.set_weights(z[f"{tag}_deep_kernel_{i}"], z[f"{tag}_deep_bias_{i}"])
    model.prediction.to_call.set_weights(z[f"{tag}_head_kernel_0"], z[f"{tag}_head_bias_0"])
    if tag == "parallel":
        model.body.concat_order = ("cross", "deep") if str(z[f"{tag}_order"]) == "cross_deep" else ("deep", "cross")
    model.compile(optimizer=mm.SGD(0.0))
    batch = {k[len("batch_"):]: torch.from_numpy(z[k]).to(device) for k in z if k.startswith("batch_")}
    y = torch.from_numpy(z["targets"]).to(device)
    tr = model.trainer(len(y))
    assert type(tr).__name__ == "DCNTrainer"
    tr.forward_backward(batch, y)
    np.testing.assert_allclose(tr.loss[0].item(), float(z[f"{tag}_loss"]), rtol=1e-5)
    close(torch.sigmoid(tr.logits.double()), z[f"{tag}_out"].reshape(-1), 2e-4, "prediction")
    got = tr.gradients()
    names = [("cross", i) for i in range(depth)] + [("deep", 0), ("deep", 1), ("head", 0)]
    for l, (grp, i) in zip(tr.arena.layers, names):
        close(got[f"{l.name}/kernel"], z[f"{tag}_grad_{grp}_kernel_{i}"], what=f"{grp} kernel {i}")
        close(got[f"{l.name}/bias"], z[f"{tag}_grad_{grp}_bias_{i}"], what=f"{grp} bias {i}")
    for t, f in enumerate(tr.feats):
        rows = tr.tables[t].table.shape[0]
        dense = torch.zeros((rows, tr.tables[t].table.shape[1]), dtype=torch.float64, device=device)
        dense.index_add_(0, tr._idx[t].long(), tr._slices[t].double())
        ids = torch.from_numpy(z[f"{tag}_table_{f}_ids"]).to(device)
        close(dense[ids], z[f"{tag}_grad_table_{f}_rows"], what=f"table {f}")


# explicit widths that make a parallel body's head input [cross | deep] 340 + 16 = 356 wide: beyond the 256 inputs of the
# fused loss kernel (the wide-head composition)
WIDE = dict(dim={"C1": 64, "C3": 120, "C5": 96, "C7": 8, "C9": 48})


@pytest.mark.parametrize("opt,stacked,wide", [("sgd", True, False), ("adagrad", True, False), ("adam", True, False),
                                              ("adagrad", False, False), ("adam", False, False), ("adam", False, True)])
def test_three_steps_match_the_restatement(device, opt, stacked, wide):
    """Three optimizer steps against autograd of the restated step + the Keras update rules in float64; every variable's
    UPDATE compared in the Frobenius norm (0.1 relative) and elementwise at 0.5 of its largest element (a relu whose
    input sits near 0 may flip between fp32 and float64: DESIGN.md §4c)."""
    from oracle import oracle_train
    from tests import dcn_train_oracle as DO

    model = _dcn(stacked=stacked, **(WIDE if wide else {}))
    model.build(device)
    assert (model.prediction.to_call.input_dim > 256) == wide
    tables, cross, deep = _oracle_state(model)
    hl = model.prediction.to_call
    heads = [{"name": "click", "kernel": H.to_numpy(hl.kernel).astype(np.float64), "bias": H.to_numpy(hl.bias).astype(np.float64),
              "loss": DO.BCE}]
    order = model.body.branch_order()

    def flat(m):
        t, cr, dp = _oracle_state(m)
        out = [t[f] for f in sorted(t)]
        for l in cr + dp:
            out += [l["kernel"], l["bias"]]
        return out + [H.to_numpy(m.prediction.to_call.kernel), H.to_numpy(m.prediction.to_call.bias)]

    before = [np.array(v, dtype=np.float64) for v in flat(model)]
    lr = {"sgd": 0.5, "adagrad": 0.05, "adam": 0.01}[opt]
    eps = 1e-6 if opt == "adam" else 1e-7
    model.compile(optimizer={"sgd": mm.SGD(lr), "adagrad": mm.Adagrad(lr), "adam": mm.Adam(lr, epsilon=eps)}[opt])

    def slots(shape):
        if opt == "adagrad":
            return {"a": np.full(shape, 0.1)}
        return {"m": np.zeros(shape), "v": np.zeros(shape)} if opt == "adam" else {}

    tslots = {f: slots(t.shape) for f, t in tables.items()}
    dslots = {}
    B = 300
    for step in (1, 2, 3):
        feats, y = _batch(B, 100 + step)
        m = model.train_step((H.device_batch(feats, device), torch.from_numpy(y).to(device)))
        loss, _, _, grads = DO.dcn_loss_and_grads(feats, tables, CONTS, cross, deep, heads, [y], stacked=stacked, order=order)
        np.testing.assert_allclose(m["loss"].item(), loss, rtol=1e-4)
        kw = dict(beta_1=0.9, beta_2=0.999, epsilon=eps, step=step)
        for f in tables:
            uniq = np.unique(feats[f])
            tables[f] = oracle_train.sparse_update(opt, tables[f], uniq, grads[f"table/{f}"][uniq], tslots[f], lr, **kw)
        for grp, ls in (("cross", cross), ("deep", deep)):
            for i, l in enumerate(ls):
                for what in ("kernel", "bias"):
                    key = f"{grp}/{what}_{i}"
                    dslots.setdefault(key, slots(l[what].shape))
                    l[what] = oracle_train.dense_update(opt, l[what], grads[key], dslots[key], lr, **kw)
        for hd in heads:
            for what in ("kernel", "bias"):
                key = f"head/{hd['name']}/{what}"
                dslots.setdefault(key, slots(hd[what].shape))
                hd[what] = oracle_train.dense_update(opt, hd[what], grads[key], dslots[key], lr, **kw)
    want = [tables[f] for f in sorted(tables)]
    for l in cross + deep:
        want += [l["kernel"], l["bias"]]
    want += [heads[0]["kernel"], heads[0]["bias"]]
    after = flat(model)
    assert len(after) == len(want) == len(before)
    for i, (a, w, b0) in enumerate(zip(after, want, before)):
        upd_ref = np.asarray(w, dtype=np.float64) - b0
        if not np.any(upd_ref):
            assert not np.any(np.asarray(a, dtype=np.float64) - b0), i
            continue
        upd = np.asarray(a, dtype=np.float64) - b0
        fro = float(np.linalg.norm(upd - upd_ref) / np.linalg.norm(upd_ref))
        assert fro < 0.1, f"update of variable {i} after 3 {opt} steps: relative Frobenius error {fro:.3e}"
        close(upd, upd_ref, 0.5, f"update of variable {i} after 3 {opt} steps")
    # the forward paths read the trained variables: eager call and a CUDA-graph compiled forward
    from models_b200.graph import HostBatch

    feats, _ = _batch(257, 9)
    want_p = H.oracle_dcn(model, feats).reshape(-1)
    got = model(H.device_batch(feats, device))
    assert H.rel_err(got.cpu().numpy().reshape(-1), want_p) < 2e-4
    hb = HostBatch.like(feats, model.input_columns())
    cf = model.compile(hb)
    assert H.rel_err(np.asarray(cf(hb)).reshape(-1), want_p) < 2e-4


def _many_tables(n):
    """n categorical columns of 31 rows (inferred width 8) and two continuous ones."""
    cols = [ColumnSchema(f"T{i:02d}", tags=(Tags.CATEGORICAL,), dtype="int64", properties={"domain": {"min": 0, "max": 30, "name": f"T{i:02d}"}})
            for i in range(n)]
    cols += [ColumnSchema(n_, tags=(Tags.CONTINUOUS,), dtype="float32") for n_ in ("I1", "I2")]
    cols.append(ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"))
    return Schema(cols)


@pytest.mark.parametrize("case", ["parallel-wide", "stacked-wide", "cross-without-bias", "70-tables"])
def test_step_gradients_match_the_restatement(device, case):
    """Loss and every gradient of one step against autograd of the restatement, at 3e-4 of each tensor's scale:
    a head input wider than the fused loss kernel's 256 (parallel [cross | deep] of 356, and a stacked 272-unit relu deep
    output), full-rank Cross layers without bias, and more tables than one mm_concat_backward call takes."""
    from tests import dcn_train_oracle as DO

    B = 300
    if case == "70-tables":
        mm.set_seed(7)
        schema = _many_tables(70)
        model = mm.DCNModel(schema, depth=2, deep_block=mm.MLPBlock([16, 8]))
        g = np.random.default_rng(70)
        feats = {c.name: g.integers(0, 31, B).astype(np.int64) for c in schema.select_by_tag(Tags.CATEGORICAL)}
        feats.update({n: g.standard_normal(B).astype(np.float32) for n in ("I1", "I2")})
        y, conts = (g.random(B) < 0.4).astype(np.int64), ["I1", "I2"]
    else:
        if case == "parallel-wide":
            model = _dcn(stacked=False, **WIDE)
        elif case == "stacked-wide":
            model = _dcn(deep=(32, 272))
        else:
            model = _dcn()
            for c in model.body.cross.cross_layers:
                c.use_bias = False
        feats, y = _batch(B, 11)
        conts = CONTS
    model.build(device)
    if case.endswith("wide"):
        assert model.prediction.to_call.input_dim > 256
    if case == "cross-without-bias":
        assert all(c.dense.bias is None for c in model.body.cross.cross_layers)
    tables, cross, deep = _oracle_state(model)
    hl = model.prediction.to_call
    heads = [{"name": "click", "kernel": H.to_numpy(hl.kernel).astype(np.float64), "bias": H.to_numpy(hl.bias).astype(np.float64),
              "loss": DO.BCE}]
    model.compile(optimizer=mm.SGD(0.0))
    tr = model.trainer(B)
    tr.forward_backward(H.device_batch(feats, device), torch.from_numpy(y).to(device))
    loss, _, _, grads = DO.dcn_loss_and_grads(feats, tables, conts, cross, deep, heads, [y], stacked=model.body.stacked,
                                              order=model.body.branch_order())
    np.testing.assert_allclose(tr.loss[0].item(), loss, rtol=1e-5)
    got = tr.gradients()
    L = len(cross)
    for i, l in enumerate(tr.arena.layers[:-1]):
        grp, j = ("cross", i) if i < L else ("deep", i - L)
        close(got[f"{l.name}/kernel"], grads[f"{grp}/kernel_{j}"], what=f"{grp} kernel {j}")
        if f"{grp}/bias_{j}" in grads:
            close(got[f"{l.name}/bias"], grads[f"{grp}/bias_{j}"], what=f"{grp} bias {j}")
        else:
            assert f"{l.name}/bias" not in got
    close(got[f"{hl.name}/kernel"], grads["head/click/kernel"], what="head kernel")
    close(got[f"{hl.name}/bias"], grads["head/click/bias"], what="head bias")
    for t, f in enumerate(tr.feats):
        dense = torch.zeros(tr.tables[t].table.shape, dtype=torch.float64, device=device)
        dense.index_add_(0, tr._idx[t].long(), tr._slices[t].double())
        close(dense, grads[f"table/{f}"], what=f"table {f}")


def test_binary_and_regression_outputs(device):
    """An OutputBlock with a binary and a regression head and loss weights: losses and every gradient against the
    restatement after one step's forward / backward."""
    from tests import dcn_train_oracle as DO

    model = _dcn(targets=("click", "rating"))
    model.build(device)
    tables, cross, deep = _oracle_state(model)
    W, b = H.to_numpy(model.prediction.to_call.kernel).astype(np.float64), H.to_numpy(model.prediction.to_call.bias).astype(np.float64)
    heads = [{"name": n, "kernel": W[:, h:h + 1], "bias": b[h:h + 1], "loss": l}
             for h, (n, l) in enumerate(zip(model.prediction.names, model.prediction.losses))]
    lws = [1.0, 0.3]
    model.compile(optimizer=mm.SGD(0.0), loss_weights=lws)
    feats, y = _batch(400, 5)
    rating = np.random.default_rng(5).random(400).astype(np.float32) * 4
    ys = {"click": y, "rating": rating}
    tr = model.trainer(400)
    targets = [ys[n.split("/")[0]] for n in model.prediction.names]
    tr.forward_backward(H.device_batch(feats, device), [torch.from_numpy(t).to(device) for t in targets])
    loss, per, _, grads = DO.dcn_loss_and_grads(feats, tables, CONTS, cross, deep, heads, targets, loss_weights=lws)
    np.testing.assert_allclose(tr.loss[0].item(), loss, rtol=1e-5)
    np.testing.assert_allclose(tr.loss[1:].cpu().numpy(), per, rtol=1e-5)
    got = tr.gradients()
    L = len(cross)
    for i, l in enumerate(tr.arena.layers[:-1]):
        grp, j = ("cross", i) if i < L else ("deep", i - L)
        close(got[f"{l.name}/kernel"], grads[f"{grp}/kernel_{j}"], what=f"{grp} kernel {j}")
        close(got[f"{l.name}/bias"], grads[f"{grp}/bias_{j}"], what=f"{grp} bias {j}")
    hk = tr.arena.layers[-1].name
    close(got[f"{hk}/kernel"], np.concatenate([grads[f"head/{h['name']}/kernel"] for h in heads], axis=1), what="heads kernel")
    for t, f in enumerate(tr.feats):
        dense = torch.zeros(tr.tables[t].table.shape, dtype=torch.float64, device=device)
        dense.index_add_(0, tr._idx[t].long(), tr._slices[t].double())
        close(dense, grads[f"table/{f}"], what=f"table {f}")


@pytest.mark.parametrize("n_out", [4, 8])
def test_several_outputs_on_a_wide_head_input_are_refused(device, n_out):
    """Several outputs read the head input from registers in the forward (at most 256 units), so a parallel body whose
    [cross | deep] is 356 wide is refused when the model is built, naming the limit: the trainer's wide-head composition
    (tensor-core logits, then mm_heads_fwd_bwd on the (B, H) logits with an identity kernel) runs with one output only."""
    targets = ("click", "rating", "conversion", "dwell", "like", "watch_time", "share", "follow")[:n_out]
    model = _dcn(stacked=False, targets=targets, **WIDE)
    with pytest.raises(NotImplementedError, match="at most 256 units, got 356"):
        model.build(device)


@pytest.mark.parametrize("stacked,wide", [(True, False), (False, False), (False, True)])
def test_graph_replay_equals_eager(device, stacked, wide):
    kw = WIDE if wide else {}
    ma, mb = _dcn(stacked=stacked, seed=12, **kw), _dcn(stacked=stacked, seed=12, **kw)
    ma.build(device), mb.build(device)
    ma.compile(optimizer=mm.Adagrad(0.05))
    mb.compile(optimizer=mm.Adagrad(0.05))
    B = 256
    batches = []
    for s in range(3):
        f, y = _batch(B, 20 + s)
        batches.append((H.device_batch(f, device), torch.from_numpy(y).to(device)))
    ta, tb = ma.trainer(B), mb.trainer(B)
    tb.capture(*batches[0])
    assert tb.launches_per_step > 0
    for x, y in batches:
        la = ta.step(x, y).clone()
        lb = tb.replay(x, y).clone()
        close(la, lb, 1e-5, "loss")
    for (na, va), (nb, vb) in zip(sorted(ma.weights().items()), sorted(mb.weights().items())):
        close(va, vb, 1e-4, na)


def test_fit_learns_a_planted_rule(device, tmp_path):
    import pyarrow as pa
    import pyarrow.parquet as pq

    n = 16000
    feats, _ = _batch(n, 1)
    rng = np.random.default_rng(0)
    s = (feats["C1"] % 2 == 0).astype(np.float32) * 2.0 + feats["C2"] * 1.5 - 1.0
    cols = dict(feats, click=(rng.random(n) < 1 / (1 + np.exp(-3 * s))).astype(np.int64))
    d = tmp_path / "data"
    d.mkdir()
    pq.write_table(pa.table(cols), d / "train.parquet")
    schema = _schema()
    loader = mm.Loader(str(d), batch_size=2000, shuffle=True, schema=schema, device=device)
    model = _dcn(seed=5)
    model.compile(optimizer=mm.Adam(0.01))
    hist = model.fit(loader, epochs=5).history["loss"]
    assert len(hist) == 5 and hist[-1] < 0.9 * hist[0], hist


def test_unsupported_configurations_name_their_cause(device):
    f, y = _batch(64, 3)
    x, yt = H.device_batch(f, device), torch.from_numpy(y).to(device)

    def fails(model, match, step=False, group=None):
        model.build(device)
        model.compile(optimizer="sgd")
        with pytest.raises(NotImplementedError, match=match):
            if step:
                model.train_step((xx, yt))
            else:
                model.trainer(64, group=group)

    xx = x
    m = _dcn()
    for c in m.body.cross.cross_layers:
        c.low_rank_dim = 4
    fails(m, "low_rank_dim")
    fails(_dcn(), "process group", group=object())
    fails(_dcn(dim={"C3": 6}), "'C3'.*width 6")
    fails(_dcn(dim={"C3": 136}), "'C3'.*width 136")
    m = _dcn()
    m.build(device)
    emb = m.body.input_block.embeddings
    emb.feature_to_table["C7"].trainable = False
    fails(m, "frozen")
    m = _dcn()
    m.build(device)
    emb = m.body.input_block.embeddings
    emb.feature_to_table["C7"] = emb.feature_to_table["C1"]
    fails(m, "shared")
    mm.set_seed(1)
    fails(mm.DCNModel(_schema(), depth=1, deep_block=mm.MLPBlock([16], dropout=0.2)), "normalization / dropout")
    fails(mm.DCNModel(_schema(), depth=1, deep_block=mm.MLPBlock([16], normalization="batch_norm")), "normalization / dropout")
    xx = dict(x, C3=torch.zeros((64, 3), dtype=torch.int64, device=device))  # a (B, L) multi-hot feature
    fails(_dcn(), "'C3'.*multi-hot", step=True)
