"""Training step of the DLRM path (SURVEY §8(f)-4) on the GPU, through the C ABI (include/mm_b200.h K14):
every backward / optimizer kernel against a float64 torch restatement of the same op, the whole step against
oracle/oracle_train.py (autograd of the restated forward + Keras update rules) and against the gradients the
reference's own torch DLRMModel produced in the build container (tests/golden/ref_torch_dlrm_train.npz).

Tolerances: the GEMM-shaped kernels multiply split-bf16 (hi, lo) pairs in three passes (|err| ~ 2^-16 relative per
product, fp32 accumulation, atomics in arbitrary order): gradients are asserted at 3e-4 of the tensor's scale
(max |reference|), the loss at 1e-5 relative.
"""
from pathlib import Path

import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets, ops
from oracle import oracle_train
from tests import helpers as H
from tests.golden import replay
from tests.test_gpu_lookup_v2 import pack_ids

pytestmark = pytest.mark.gpu
G = Path(__file__).parent / "golden"
TOL = 3e-4


def close(got, ref, tol=TOL, what=""):
    got = np.asarray(got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got, dtype=np.float64)
    ref = np.asarray(ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref, dtype=np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    scale = max(float(np.max(np.abs(ref))), 1e-30)
    err = float(np.max(np.abs(got - ref))) / scale
    assert err < tol, f"{what}: max |diff| / max |ref| = {err:.3e} (tol {tol})"


# ---------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------
def test_dense_dgrad_rejects_wide_layers(device):
    with pytest.raises(ValueError, match="N=256"):
        ops.dense_dgrad(torch.zeros((4, 256), device=device), torch.zeros((8, 256), device=device), torch.zeros((4, 8), device=device))


@pytest.mark.parametrize("M,K", [(1, 32), (1000, 32), (4099, 8), (513, 200), (37, 24), (100, 128), (65, 64), (9, 16)])
@pytest.mark.parametrize("tdtype", [torch.int64, torch.float32])
def test_one_bce_head_forward_backward(device, M, K, tdtype):
    """BinaryOutput's Dense(1) + BCE as the training step runs it: heads_fwd_bwd with H = 1, against float64 autograd."""
    g = torch.Generator().manual_seed(M + K)
    x = torch.randn((M, K), generator=g).clamp_min(0.0).to(device)
    w = (torch.randn(K, generator=g) * 0.5).to(device)
    b = torch.tensor([0.3], device=device)
    y = torch.randint(0, 2, (M,), generator=g).to(tdtype).to(device)
    sw = (torch.rand(M, generator=g) + 0.5).to(device)
    for weights in (None, sw):
        loss = torch.zeros(2, device=device)
        dx = torch.empty((M, K), device=device)
        dw = torch.zeros(K, device=device)
        db = torch.zeros(1, device=device)
        logits = torch.empty(M, device=device)
        ops.heads_fwd_bwd(x, w.view(K, 1), b, ["binary_crossentropy"], [y], logits.view(1, M), loss, dx, dw.view(K, 1), db,
                          mask_relu=True, sample_weight=weights)
        xd = x.double().requires_grad_(True)
        wd = w.double().requires_grad_(True)
        bd = b.double().requires_grad_(True)
        z = xd @ wd + bd
        per = torch.nn.functional.binary_cross_entropy_with_logits(z, y.double(), reduction="none")
        ref = (per * (1.0 if weights is None else weights.double())).sum() / M
        ref.backward()
        np.testing.assert_allclose(loss[0].item(), ref.item(), rtol=1e-5)
        close(logits, z, 1e-5, "logits")
        close(dx, xd.grad * (x > 0), 1e-5, "dx")
        close(dw, wd.grad, 1e-5, "dw")
        close(db, bd.grad, 1e-5, "db")


def _interaction_ref(rows, bottom, dA, slot_b, P):
    """float64 autograd of stack -> bmm -> upper triangle -> [bottom | pairs] (oracle_torch.dlrm_forward's staging)."""
    leaves = [r.double().requires_grad_(True) for r in rows]
    bt = bottom.double().requires_grad_(True)
    seq = leaves[:slot_b] + [bt] + leaves[slot_b:]
    st = torch.stack(seq, dim=1)
    z = torch.bmm(st, st.transpose(1, 2))
    Fn = st.shape[1]
    mask = torch.triu(torch.ones(Fn, Fn, dtype=torch.bool, device=st.device), diagonal=1)
    out = torch.cat([bt, z[:, mask]], dim=1) if P else z[:, mask]
    out.backward(dA.double())
    return [l.grad for l in leaves], bt.grad


@pytest.mark.parametrize("D", [16, 32, 64, 128])
@pytest.mark.parametrize("T,B", [(26, 300), (5, 37), (31, 65), (1, 9)])
def test_interact_backward(device, D, T, B):
    g = torch.Generator().manual_seed(D * 100 + T)
    rows_n = [3, 200, 70000, 300][: min(T, 4)] + [50 + 7 * i for i in range(max(0, T - 4))]
    tables = [(torch.randn((r, D), generator=g) * 0.3).to(device) for r in rows_n]
    ids64 = [torch.randint(0, r, (B,), generator=g) for r in rows_n]
    # every id width the forward kernel takes
    ids = []
    for t, (i, r) in enumerate(zip(ids64, rows_n)):
        if r <= 256 and t % 2 == 0:
            ids.append(i.to(torch.uint8).to(device))
        elif r <= 65536 and t % 3 == 0:
            ids.append(i.to(torch.uint16).to(device))
        elif t % 5 == 0:
            b3 = torch.stack([i & 255, (i >> 8) & 255, (i >> 16) & 255], dim=1).to(torch.uint8)
            ids.append(b3.contiguous().to(device))
        elif t % 2:
            ids.append(i.to(torch.int32).to(device))
        else:
            ids.append(i.to(device))
    Fn = T + 1
    names = sorted([f"C{t}" for t in range(T)] + ["bottom_block"])  # string order, as the model's slots
    slot_b = names.index("bottom_block")
    slots = [s for s in range(Fn) if s != slot_b]
    bottom = torch.randn((B, D), generator=g).to(device)
    bottom[:, ::3] = 0.0  # relu zeros: the mask matters
    OW = D + Fn * (Fn - 1) // 2
    ld = (OW + 3) // 4 * 4
    dAb = torch.randn((B, ld), generator=g).to(device)
    dA = dAb[:, :OW]
    grads = torch.full((T, B, D), 9.0, device=device)
    d_bottom = torch.empty((B, D), device=device)
    ops.dlrm_interact_backward(tables, ids, slots, rows_n, D, bottom, slot_b, dA, [grads[t] for t in range(T)], d_bottom, mask_bottom=True)
    looked = [tables[t][ids64[t].to(device)] for t in range(T)]
    ref_rows, ref_bottom = _interaction_ref(looked, bottom, dA, slot_b, D)
    for t in range(T):
        close(grads[t], ref_rows[t], what=f"slices of table {t}")
    close(d_bottom, ref_bottom * (bottom > 0), what="d_bottom (masked)")
    ops.dlrm_interact_backward(tables, ids, slots, rows_n, D, bottom, slot_b, dA, [grads[t] for t in range(T)], d_bottom, mask_bottom=False)
    close(d_bottom, ref_bottom, what="d_bottom")
    if D == 64:
        # operand-format rows (the tables' split-bf16 mirrors + the bottom vector as split rows): same gradients
        mirrors = [ops.split_rows(w) for w in tables]
        bsplit = ops.split_rows(bottom)
        for mask in (True, False):
            grads.fill_(9.0)
            d_bottom.fill_(9.0)
            ops.dlrm_interact_backward(mirrors, ids, slots, rows_n, D, bsplit, slot_b, dA, [grads[t] for t in range(T)], d_bottom,
                                       mask_bottom=mask, operand_rows=True)
            for t in range(T):
                close(grads[t], ref_rows[t], what=f"operand rows: slices of table {t}")
            close(d_bottom, ref_bottom * (bottom > 0) if mask else ref_bottom, what="operand rows: d_bottom")


def test_interact_backward_out_of_range_ids_read_zero_rows(device):
    D, B = 16, 8
    tab = [torch.randn((10, D), device=device), torch.randn((20, D), device=device)]
    ids = [torch.tensor([0, 1, 2, 99, 4, -1, 6, 7], dtype=torch.int32, device=device), torch.arange(8, dtype=torch.int64, device=device)]
    bottom = torch.randn((B, D), device=device)
    OW = D + 3
    dA = torch.randn((B, OW), device=device)
    grads = torch.empty((2, B, D), device=device)
    d_bottom = torch.empty((B, D), device=device)
    ops.dlrm_interact_backward(tab, ids, [0, 1], [10, 20], D, bottom, 2, dA, [grads[0], grads[1]], d_bottom, mask_bottom=False)
    safe = ids[0].clamp(0, 9).long()
    rows0 = tab[0][safe] * ((ids[0] >= 0) & (ids[0] < 10)).unsqueeze(1)
    ref_rows, ref_bottom = _interaction_ref([rows0, tab[1][ids[1]]], bottom, dA, 2, D)
    close(grads[1], ref_rows[1], what="other table")
    close(d_bottom, ref_bottom, what="bottom")


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
@pytest.mark.parametrize("D", [16, 64, 128])
@pytest.mark.parametrize("dense_path", [False, True])
def test_sparse_rows_apply_sums_duplicates_and_updates_once(device, opt, D, dense_path):
    """Election path (dense_grad = None) and dense-accumulator path (sort + run sums for the 7-, 300- and 200-row tables,
    vector reds for the 5 000-row ones) give the same update, at every id width (int32, int64, uint16, and the packed
    uint8 and 3-byte columns of a host batch) in one call."""
    rng = np.random.default_rng(5)
    B = 3000
    rows = [7, 5000, 300, 200, 5000, 300]  # 7 rows: every id repeats hundreds of times
    W = [rng.normal(size=(r, D)).astype(np.float32) for r in rows]
    ids = [rng.integers(0, r, B) for r in rows]
    ids[1][:10] = [-3, 5000, 6000, 1, 1, 1, 2, 2, 4999, 0]  # out of range ids are dropped
    ids[4][:10] = [(1 << 24) - 3, 5000, 6000, 1, 1, 1, 2, 2, 4999, 0]  # (-3 as a 3-byte id)
    ids[3][:3] = [200, 255, 199]  # 1-byte ids past the table's 200 rows
    vals = [rng.normal(size=(B, D)).astype(np.float32) for _ in rows]
    hyper_cfg = dict(lr=0.05, beta_1=0.9, beta_2=0.999, epsilon=1e-7)
    o = {"sgd": mm.SGD(0.05), "adagrad": mm.Adagrad(0.05), "adam": mm.Adam(0.05)}[opt]
    hyper = torch.from_numpy(o.hyper()).to(device)
    dev_w = [torch.from_numpy(w.copy()).to(device) for w in W]
    s1 = [torch.full_like(w, o.initial_accumulator_value) if o.slots >= 1 else None for w in dev_w]
    s2 = [torch.zeros_like(w) if o.slots >= 2 else None for w in dev_w]
    rep = [ops.fill_i32(torch.empty(r, dtype=torch.int32, device=device), 2**31 - 1) for r in rows]
    mirror = [ops.split_rows(w) if D == 64 else None for w in dev_w]
    dense = [torch.zeros_like(w) if dense_path else None for w in dev_w]
    widths = [4, 8, 2, 1, 3, 3]  # id bytes per table
    st = [{"a": np.full(w.shape, o.initial_accumulator_value), "m": np.zeros(w.shape), "v": np.zeros(w.shape)} for w in W]
    st = [{k: v for k, v in s.items() if (opt == "adagrad" and k == "a") or (opt == "adam" and k in "mv")} for s in st]
    ref = [w.astype(np.float64) for w in W]
    n = len(rows)
    for step in (1, 2):
        ops.opt_tick(hyper)
        tabs = [dict(weights=dev_w[t], indices=torch.from_numpy(pack_ids(ids[t], widths[t])).to(device),
                     grad_rows=torch.from_numpy(vals[t].copy()).to(device), rep_map=rep[t], state1=s1[t], state2=s2[t], mirror=mirror[t],
                     dense_grad=dense[t]) for t in range(n)]
        assert [ops.index_bytes_of(tb["indices"]) for tb in tabs] == widths
        ops.sparse_rows_apply(opt, tabs, B, D, hyper)
        for t in range(n):
            kw = dict(hyper_cfg, step=step)
            lr = kw.pop("lr")
            ref[t] = oracle_train.sparse_update(opt, ref[t], ids[t], vals[t], st[t], lr, **kw)
            close(dev_w[t], ref[t], 2e-5, f"{opt} step {step} table {t}")
            assert int((rep[t] != 2**31 - 1).sum()) == 0  # the map is idle again
            assert dense[t] is None or float(dense[t].abs().max()) == 0.0  # and so is the accumulator
            if mirror[t] is not None:
                assert torch.equal(mirror[t], ops.split_rows(dev_w[t]))  # operand-format copy kept in step
    assert float(hyper[4]) == 2.0


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
def test_dense_apply(device, opt):
    rng = np.random.default_rng(9)
    n = 10007
    w = rng.normal(size=n).astype(np.float32)
    o = {"sgd": mm.SGD(0.1), "adagrad": mm.Adagrad(0.1), "adam": mm.Adam(0.1)}[opt]
    hyper = torch.from_numpy(o.hyper()).to(device)
    dw = torch.from_numpy(w.copy()).to(device)
    s1 = torch.full_like(dw, o.initial_accumulator_value) if o.slots >= 1 else None
    s2 = torch.zeros_like(dw) if o.slots >= 2 else None
    st = {"a": np.full(n, o.initial_accumulator_value)} if opt == "adagrad" else {"m": np.zeros(n), "v": np.zeros(n)} if opt == "adam" else {}
    ref = w.astype(np.float64)
    for step in (1, 2, 3):
        g = rng.normal(size=n).astype(np.float32)
        dg = torch.from_numpy(g.copy()).to(device)
        ops.opt_tick(hyper)
        ops.dense_apply(opt, dw, dg, s1, s2, hyper, grad_scale=0.5)
        ref = oracle_train.dense_update(opt, ref, 0.5 * g.astype(np.float64), st, 0.1, step=step)
        close(dw, ref, 2e-5, f"{opt} step {step}")
        assert float(dg.abs().max()) == 0.0  # gradients are cleared for the next accumulation


# ---------------------------------------------------------------------------------------------------------------
# whole step
# ---------------------------------------------------------------------------------------------------------------
def _ref_schema(z):
    from models_b200.schema import ColumnSchema, Schema

    cols = [ColumnSchema(str(n), tags=("categorical",), dtype="int64", properties={"domain": {"min": 0, "max": int(mx), "name": str(n)}})
            for n, mx in zip(z["cat_names"], z["cat_max"])]
    cols += [ColumnSchema(str(n), tags=("continuous",), dtype="float32") for n in z["cont_names"]]
    cols.append(ColumnSchema("click", tags=("target", "binary_classification"), dtype="int64"))
    return Schema(cols)


def _load_weights(model, z, device):
    for name, t in model.body.embeddings.tables.items():
        t.table = torch.from_numpy(z[f"table_{name}"]).to(device).contiguous()
        t.built = True
    for blk, tag in ((model.body.bottom_block, "bottom"), (model.body.top_block, "top")):
        for l, w in zip(blk.dense_layers, replay.unpack_layers(z, tag)):
            l.set_weights(w["kernel"], w["bias"])
    h = replay.unpack_layers(z, "head")[0]
    model.prediction.to_call.set_weights(h["kernel"], h["bias"])


def _table_grad(tr, t, rows):
    """IndexedSlices of table t -> dense gradient (what autograd reports for the table variable)."""
    ids = ops.widen_index(tr._idx[t]).long()
    dense = torch.zeros((rows, tr.D), dtype=torch.float64, device=ids.device)
    dense.index_add_(0, ids, tr._slices[t].double())
    return dense


def test_train_step_gradients_match_the_reference_torch_backend(device):
    """Loss and every gradient of ONE step against what merlin.models.torch's DLRMModel + its default BinaryOutput loss
    + torch.autograd produced in the build container (oracle/make_golden_from_reference_torch.py §9a)."""
    z = replay.load(G / "ref_torch_dlrm_train.npz")
    dim = int(z["dim"])
    model = mm.DLRMModel(_ref_schema(z), embedding_dim=dim, bottom_block=mm.MLPBlock([32, dim]), top_block=mm.MLPBlock([24, 8]))
    model.build(device)
    _load_weights(model, z, device)
    batch = {k[len("batch_"):]: torch.from_numpy(z[k]).to(device) for k in z if k.startswith("batch_")}
    y = torch.from_numpy(z["targets"]).to(device)
    model.compile(optimizer=mm.SGD(0.0))
    tr = model.trainer(len(z["targets"]))
    tr.forward_backward(batch, y)
    np.testing.assert_allclose(tr.loss.item(), float(z["loss"]), rtol=1e-5)
    np.testing.assert_allclose(torch.sigmoid(tr.logits).cpu().numpy(), z["out"].reshape(-1), rtol=2e-4, atol=2e-6)
    got = tr.gradients()
    layers = tr.arena.layers
    names = [("bottom", 0), ("bottom", 1), ("top", 0), ("top", 1), ("head", 0)]
    assert len(layers) == len(names)
    for l, (tag, i) in zip(layers, names):
        close(got[f"{l.name}/kernel"], z[f"grad_{tag}_kernel_{i}"], what=f"{tag} kernel {i}")
        close(got[f"{l.name}/bias"], z[f"grad_{tag}_bias_{i}"], what=f"{tag} bias {i}")
    for t, f in enumerate(tr.feats):
        close(_table_grad(tr, t, z[f"table_{f}"].shape[0]), z[f"grad_table_{f}"], what=f"table {f}")


def _small_model(device, seed=3, D=64, cap=300, bottom=(128, 64), top=(128, 64, 32)):
    mm.set_seed(seed)
    schema = datasets.criteo_schema({k: min(v, cap) for k, v in datasets.CRITEO_MAX.items()})
    bottom = list(bottom[:-1]) + [D]
    model = mm.DLRMModel(schema, embedding_dim=D, bottom_block=mm.MLPBlock(bottom), top_block=mm.MLPBlock(list(top)))
    model.build(device)
    return schema, model


def _oracle_state(model):
    tables, f2t = H.emb_tables(model.body.embeddings)
    return dict(tables={k: v.astype(np.float64) for k, v in tables.items()}, f2t=f2t, cont=model.body.continuous.features,
                bottom=H.mlp_layers(model.body.bottom_block), top=H.mlp_layers(model.body.top_block), head=H.head_layer(model.prediction))


def _flat_state(model):
    """Every variable in structural order (tables by name, bottom, top, head) — names differ between two models."""
    st = _oracle_state(model)
    out = [st["tables"][n] for n in sorted(st["tables"])]
    for tag in ("bottom", "top"):
        for l in st[tag]:
            out += [l["kernel"], l["bias"]]
    return out + [st["head"]["kernel"], st["head"]["bias"]]


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
@pytest.mark.parametrize("D", [16, 64])
def test_training_steps_match_oracle(device, opt, D):
    """Three optimizer steps (different batches, heavy id duplication: tables of <= 300 rows) against autograd of the
    restated forward + the Keras update rules in float64.  What is compared is the UPDATE of every variable (after -
    before): 0.1 in the Frobenius norm (observed: <= 2.4e-2), 0.5 of the largest element (observed: <= 8e-2; a wrong
    rule or sign gives >= 1).  A relu unit whose pre-activation is within rounding
    of zero may be on in one implementation and off in the other (about one unit per step at this size); that changes ONE
    sample's gradient by a few percent — visible in the rows that sample touched (max norm), negligible in the
    Frobenius norm.  The kernels' own accuracy (3e-4) is asserted by the tests above and by the reference golden."""
    schema, model = _small_model(device, D=D)
    st = _oracle_state(model)
    before = [np.array(v, dtype=np.float64) for v in _flat_state(model)]
    lr = {"sgd": 1.0, "adagrad": 0.05, "adam": 0.01}[opt]
    # Adam's update is lr * sign(g) wherever |g| >> epsilon: with the Keras default 1e-7 an element whose gradient is
    # below the kernels' rounding noise could flip sign and move by 2 lr; 1e-6 keeps the update a smooth function of g
    # at this test's gradient scale (~1e-4) while sqrt(v) still matters
    eps = 1e-6 if opt == "adam" else 1e-7
    o = {"sgd": mm.SGD(lr), "adagrad": mm.Adagrad(lr), "adam": mm.Adam(lr, epsilon=eps)}[opt]
    model.compile(optimizer=o)
    B = 300

    def slots(shape):
        if opt == "adagrad":
            return {"a": np.full(shape, 0.1)}
        return {"m": np.zeros(shape), "v": np.zeros(shape)} if opt == "adam" else {}

    tslots = {n: slots(t.shape) for n, t in st["tables"].items()}
    dslots = {}
    for step in (1, 2, 3):
        batch = datasets.generate_batch(schema, B, seed=100 + step, index_law="uniform")
        feats, targets = datasets.split_targets(schema, batch)
        y = next(iter(targets.values())) if isinstance(targets, dict) else targets
        m = model.train_step((H.device_batch(feats, device), torch.from_numpy(np.asarray(y)).to(device)))
        loss, _, grads = oracle_train.dlrm_loss_and_grads(feats, st["tables"], st["f2t"], st["cont"], st["bottom"], st["top"], st["head"], y)
        np.testing.assert_allclose(m["loss"].item(), loss, rtol=1e-4)
        assert m["loss_batch"].item() == m["loss"].item() and m["regularization_loss"].item() == 0.0
        kw = dict(beta_1=0.9, beta_2=0.999, epsilon=eps, step=step)
        for f, tname in st["f2t"].items():
            # IndexedSlices of feature f: the dense gradient restricted to the looked-up rows (each table has one feature here)
            uniq = np.unique(np.asarray(feats[f]).reshape(-1))
            st["tables"][tname] = oracle_train.sparse_update(opt, st["tables"][tname], uniq, grads[f"table/{tname}"][uniq], tslots[tname], lr, **kw)
        for tag in ("bottom", "top"):
            for i, l in enumerate(st[tag]):
                for what in ("kernel", "bias"):
                    key = f"{tag}/{what}_{i}"
                    dslots.setdefault(key, slots(l[what].shape))
                    l[what] = oracle_train.dense_update(opt, l[what], grads[key], dslots[key], lr, **kw)
        for what in ("kernel", "bias"):
            key = f"head/{what}"
            dslots.setdefault(key, slots(st["head"][what].shape))
            st["head"][what] = oracle_train.dense_update(opt, st["head"][what], grads[key], dslots[key], lr, **kw)
    want = [st["tables"][n] for n in sorted(st["tables"])]
    for tag in ("bottom", "top"):
        for l in st[tag]:
            want += [l["kernel"], l["bias"]]
    want += [st["head"]["kernel"], st["head"]["bias"]]
    after = _flat_state(model)
    assert len(after) == len(want) == len(before)
    for i, (a, w, b0) in enumerate(zip(after, want, before)):
        upd_ref = np.asarray(w, dtype=np.float64) - b0
        assert np.max(np.abs(upd_ref)) > 0, i  # every variable trains
        upd = np.asarray(a, dtype=np.float64) - b0
        fro = float(np.linalg.norm(upd - upd_ref) / np.linalg.norm(upd_ref))
        assert fro < 0.1, f"update of variable {i} after 3 {opt} steps: relative Frobenius error {fro:.3e}"
        close(upd, upd_ref, 0.5, f"update of variable {i} after 3 {opt} steps")
    # rows no batch looked up did not move (lazy / sparse semantics), nor did their slots matter
    tr = model._trainer
    for t, f in enumerate(tr.feats):
        tab = tr.tables[t].table.cpu().numpy()
        tname = st["f2t"][f]
        idx0 = sorted(st["tables"]).index(tname)
        untouched = np.all(want[idx0] == before[idx0], axis=1)
        assert np.array_equal(tab[untouched], before[idx0][untouched].astype(np.float32))
    # the forward path of the same model sees the trained variables (operand copies were refreshed in place)
    batch = datasets.generate_batch(schema, 200, seed=55, index_law="uniform")
    feats, _ = datasets.split_targets(schema, batch)
    got = model(H.device_batch(feats, device)).cpu().numpy()
    assert H.rel_err(got, H.oracle_dlrm(model, feats)) < 2e-4


def test_wide_towers_train_through_the_tensor_core_dgrad(device):
    """Layers wider than 128 units (mm_dense_dgrad's limit) take dX = dZ W^T through mm_dense_tc on the transposed kernel +
    mm_relu_mask: one step's loss and every gradient against the oracle."""
    schema, model = _small_model(device, seed=9, D=16, cap=200, bottom=(160, 16), top=(256, 192, 32))
    st = _oracle_state(model)
    model.compile(optimizer=mm.SGD(0.0))
    B = 200
    batch = datasets.generate_batch(schema, B, seed=77, index_law="uniform")
    feats, targets = datasets.split_targets(schema, batch)
    y = np.asarray(next(iter(targets.values())))
    tr = model.trainer(B)
    assert sorted(tr._wide) == [2, 3]  # the two wide top layers (a wide FIRST bottom layer needs no input gradient)
    tr.forward_backward(H.device_batch(feats, device), torch.from_numpy(y).to(device))
    loss, _, grads = oracle_train.dlrm_loss_and_grads(feats, st["tables"], st["f2t"], st["cont"], st["bottom"], st["top"], st["head"], y)
    np.testing.assert_allclose(tr.loss.item(), loss, rtol=2e-5)
    got = tr.gradients()

    def fro(a, b, what):  # Frobenius norm: a relu unit within rounding of zero may flip and move ONE sample's contribution
        a = a.detach().cpu().numpy().astype(np.float64)
        err = float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))
        assert err < 1e-2, f"{what}: relative Frobenius error {err:.3e}"

    names = [("bottom", 0), ("bottom", 1), ("top", 0), ("top", 1), ("top", 2)]
    for l, (tag, i) in zip(tr.arena.layers[:-1], names):
        fro(got[f"{l.name}/kernel"], grads[f"{tag}/kernel_{i}"], f"{tag} kernel {i}")
        fro(got[f"{l.name}/bias"], grads[f"{tag}/bias_{i}"], f"{tag} bias {i}")
    fro(got[f"{tr.arena.layers[-1].name}/kernel"], grads["head/kernel"], "head kernel")
    for t, f in enumerate(tr.feats):
        tname = st["f2t"][f]
        fro(_table_grad(tr, t, st["tables"][tname].shape[0]), grads[f"table/{tname}"], f"table {f}")


def test_relu_mask_kernel(device):
    x = torch.randn((37, 50), device=device)
    big = torch.randn((37, 64), device=device)
    m = big[:, :50]  # strided mask
    want = torch.where(m > 0, x, torch.zeros_like(x))
    assert torch.equal(ops.relu_mask(x.clone(), m), want)


def test_graph_replay_equals_eager_steps_and_partial_batches(device):
    schema, model_a = _small_model(device, seed=11, D=32, top=(64, 32))
    _, model_b = _small_model(device, seed=11, D=32, top=(64, 32))
    B = 512
    batches = []
    for s in range(4):
        b = datasets.generate_batch(schema, B, seed=s, index_law="uniform")
        f, t = datasets.split_targets(schema, b)
        y = next(iter(t.values())) if isinstance(t, dict) else t
        batches.append((H.device_batch(f, device), torch.from_numpy(np.asarray(y)).to(device)))
    model_a.compile(optimizer=mm.Adagrad(0.05))
    model_b.compile(optimizer=mm.Adagrad(0.05))
    ta, tb = model_a.trainer(B), model_b.trainer(B)
    tb.capture(*batches[0])
    assert tb.launches_per_step >= 20
    # capture must not train: both models still hold identical variables
    for i, (va, vb) in enumerate(zip(_flat_state(model_a), _flat_state(model_b))):
        assert np.array_equal(va, vb), i
    for x, y in batches:
        la = ta.step(x, y).item()
        lb = tb.replay(x, y).item()
        np.testing.assert_allclose(la, lb, rtol=1e-6)
    for i, (va, vb) in enumerate(zip(_flat_state(model_a), _flat_state(model_b))):
        close(va, vb, 1e-5, f"variable {i}")  # same kernels; only the order of the atomics differs
    # a smaller (last) batch runs in the leading rows of the same buffers
    x, y = batches[1]
    xs, ys = {k: v[:100] for k, v in x.items()}, y[:100]
    st = _oracle_state(model_a)
    loss_small = ta.step(xs, ys).item()
    feats = {k: v.cpu().numpy() for k, v in xs.items()}
    ref_loss, _, _ = oracle_train.dlrm_loss_and_grads(feats, st["tables"], st["f2t"], st["cont"], st["bottom"], st["top"], st["head"], ys.cpu().numpy())
    np.testing.assert_allclose(loss_small, ref_loss, rtol=2e-5)
    with pytest.raises(ValueError, match="up to 512"):
        ta.step({k: torch.cat([v, v]) for k, v in x.items()}, torch.cat([y, y]))


def test_fit_with_loader_learns_a_planted_rule(device, tmp_path):
    """model.compile(optimizer) + model.fit(mm.Loader(...)): the loss of a learnable synthetic target goes down and the
    model ranks held-out positives above negatives (models/base.py `fit` contract, examples/03)."""
    import pyarrow as pa
    import pyarrow.parquet as pq

    rng = np.random.default_rng(0)
    n = 20000
    schema = datasets.criteo_schema({k: min(v, 50) for k, v in datasets.CRITEO_MAX.items()})
    batch = datasets.generate_batch(schema, n, seed=1, index_law="uniform")
    feats, _ = datasets.split_targets(schema, batch)
    score = (feats["C1"] % 2 == 0).astype(np.float32) * 1.5 + feats["I1"].reshape(-1) * 2.0 - (feats["C2"] % 3 == 0) * 1.0 - 1.0
    click = (rng.random(n) < 1 / (1 + np.exp(-3 * score))).astype(np.int64)
    cols = {k: np.asarray(v).reshape(-1) for k, v in feats.items()}
    cols["label"] = click
    d = tmp_path / "data"
    d.mkdir()
    pq.write_table(pa.table({k: v[:16000] for k, v in cols.items()}), d / "train.parquet")
    loader = mm.Loader(str(d), batch_size=2000, shuffle=True, schema=schema, device=device)
    assert loader.label_names == ["label"]
    mm.set_seed(5)
    model = mm.DLRMModel(schema, embedding_dim=16, bottom_block=mm.MLPBlock([32, 16]), top_block=mm.MLPBlock([32, 16]))
    model.compile(optimizer=mm.Adam(0.02))
    hist = model.fit(loader, epochs=8)
    losses = hist.history["loss"]
    assert len(losses) == 8 and losses[-1] < losses[0] - 0.03, losses
    held = {k: torch.from_numpy(np.ascontiguousarray(v[16000:])).to(device) for k, v in cols.items() if k != "label"}
    p = model(held).cpu().numpy().reshape(-1)
    y = click[16000:]
    auc_pairs = (p[y == 1][:, None] > p[y == 0][None, :]).mean()
    assert auc_pairs > 0.6, auc_pairs
    # a trained (compiled) model goes through the checkpoint boundary like any other: variables are views of the
    # trainer's arena, the optimizer and the History object ride along in the structure file
    model.save(tmp_path / "export")
    loaded = mm.Model.load(tmp_path / "export")
    np.testing.assert_array_equal(loaded(held).cpu().numpy().reshape(-1), p)
    assert loaded.optimizer.kind == "adam" and loaded.history.history["loss"] == losses


def test_out_of_range_ids_are_counted_and_reported(device):
    schema, model = _small_model(device, D=16)
    model.compile(optimizer="sgd")
    b = datasets.generate_batch(schema, 64, seed=2, index_law="uniform")
    feats, targets = datasets.split_targets(schema, b)
    feats["C1"] = feats["C1"].copy()
    feats["C1"][3] = 10**6
    y = torch.from_numpy(np.asarray(next(iter(targets.values())))).to(device)
    before = model.body.embeddings.feature_to_table["C1"].embeddings.clone()
    model.train_step((H.device_batch(feats, device), y))
    assert torch.isfinite(model._trainer.loss).all()
    with pytest.raises(IndexError, match="1 indices out of range"):
        model._trainer.check_indices()
    model._trainer.check_indices()  # the counter was reset
    assert before.shape == model.body.embeddings.feature_to_table["C1"].embeddings.shape  # no row was added or touched out of bounds


def test_compile_validation(device):
    schema, model = _small_model(device, D=16)
    with pytest.raises(ValueError, match="Unknown optimizer"):
        model.compile(optimizer="rmsprop")
    with pytest.raises(NotImplementedError, match="binary"):
        model.compile(optimizer="sgd", loss="mse")
    model._trainer = None
    model.optimizer = None
    with pytest.raises(RuntimeError, match="compile"):
        model.train_step(({}, torch.zeros(1)))
