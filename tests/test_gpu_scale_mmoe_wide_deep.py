"""The MMoE training step and the Wide&Deep wide kernels at the sizes their benchmarks train with, and the MMoETrainer
paths its first tests left out.

MMoETrainer against the restatement (tests/mmoe_oracle.py, through tests/test_gpu_mmoe._check_gradients with the
device's relu decisions): the benchmark's leg (b) (E = 4, U = 64, towers [32], gate blocks [16]) and the tower-only leg
at B = 65 536 on the Criteo schema (d = 941); a batch smaller than the compiled size on the tower path; per-task sample
weights; one-layer towers on a shared bottom, towers on the input block alone, E = 12 and five outputs with towers.

mm_wide_deep_head_fwd_bwd, mm_wide_bag_grad and mm_wide_rows_apply at B = 65 536 and 65 573 with fixed bags of the
MLPerf DLRM-DCNv2 lengths (L = 27 and 100) over a 40-row domain, so a bag of 100 is full of repeats and the multi_hot
deduplication scan runs its longest: per-element float64 bounds (EPS = 2^-24; an fp32 sum of n terms is within
(n - 1) EPS of the sum of the absolute terms), the bag gradient's (id, value) pairs exactly, the out-of-range counter
exactly, and the rows no id touched bit for bit."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets, ops
from models_b200.schema import ColumnSchema, Schema, Tags
from tests import helpers as Hp
from tests.mmoe_oracle import BCE
from tests.test_gpu_mmoe import _batch, _check_gradients, close
from tests.test_gpu_train_scale import BIG, RAGGED, _sms, _within
from tests.test_mmoe_host import mmoe_model, schema

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -24


def _criteo_multitask():
    """The MMoE benchmark's schema: Criteo with tables capped at 20 000 rows and click / conversion / rating targets."""
    base = datasets.criteo_schema({k: min(v, 20000) for k, v in datasets.CRITEO_MAX.items()})
    cols = [c for c in base if c.name != "label"]
    cols += [ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"),
             ColumnSchema("conversion", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"),
             ColumnSchema("rating", tags=(Tags.TARGET, Tags.REGRESSION), dtype="float32")]
    return Schema(cols)


# ---------------------------------------------------------------------------------------------------------------
# MMoETrainer at the benchmark's size
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("leg", ["towers_gates", "towers_only"])
def test_benchmark_size_tower_legs(device, leg):
    """One step at B = 65 536: the benchmark's leg (b) (MMOEBlock of 4 experts of MLPBlock([64]), task_blocks
    MLPBlock([32]), gate_block MLPBlock([16]), Adagrad(0.01)), and the towers on a shared bottom without an MMOEBlock.
    The mixture and task-head kernels run 15.5 grid-stride laps of 4 SMs x 8 warps here."""
    B = BIG
    ctas = min(-(-B // 8), 4 * _sms(device))
    assert -(-B // (8 * ctas)) >= 2 and B % (8 * ctas), "premise: more than one lap, the last one ragged"
    s = _criteo_multitask()
    mm.set_seed(4)
    if leg == "towers_gates":
        model = mmoe_model(s, E=4, U=64, towers=[32], gate=[16])
    else:
        model = mm.Model(mm.InputBlockV2(s), mm.MLPBlock([32, 16]), mm.OutputBlock(s, task_blocks=mm.MLPBlock([32])))
    model.build(device)
    assert model.body.input_block.layout()[2] > 256  # d = 941: the input gradient takes the transposed-kernel GEMM
    model.compile(optimizer=mm.Adagrad(0.01))
    feats, targs = _batch(s, B, 19)
    _check_gradients(model, model.trainer(B), feats, targs)


# ---------------------------------------------------------------------------------------------------------------
# MMoETrainer: partial batches, sample weights, configurations
# ---------------------------------------------------------------------------------------------------------------
def _towers_gates(s):
    return mmoe_model(s, E=4, U=16, bottom=[32], T=0.9, towers=[12], gate=[8])


def test_partial_batch_on_the_tower_path(device):
    """A trainer compiled for 512 rows fed 300: the mixture, its split operand and dm live in the leading H b rows of
    their buffers.  The tails past H b (and the gate weights past b) are NaN before the step and stay NaN; the gradients
    match the restatement on the 300 rows, are finite, and agree with a trainer compiled for 300 rows."""
    s = schema()
    models = []
    for _ in range(2):
        mm.set_seed(31)
        m = _towers_gates(s)
        m.build(device)
        m.compile(optimizer="sgd", loss_weights=[1.0, 0.5, 2.0])
        models.append(m)
    b = 300
    feats, targs = _batch(s, b, 8)
    ta, tb = models[0].trainer(512), models[1].trainer(b)
    H = ta.H
    tails = [t.view(-1)[H * b * t.shape[2]:] for t in (ta.M, ta.M_split, ta.dM)] + [ta.P[b:]]
    for t in tails:
        t.fill_(float("nan"))
    _check_gradients(models[0], ta, feats, targs)
    assert bool(torch.isfinite(ta.arena.grad).all()), "a gradient is not finite"
    for t, name in zip(tails, ("M", "M_split", "dM", "P")):
        assert bool(torch.isnan(t.float()).all()), f"{name} was written past the batch"
    tb.forward_backward(Hp.device_batch(feats, device), [torch.from_numpy(np.asarray(targs[o.target])).to(device)
                                                         for o in models[1].output_blocks()])
    close(ta._loss_all, tb._loss_all, 1e-5, "loss vs the 300-row trainer")
    aa, ab = ta.arena, tb.arena  # the two trainers sum their atomics in different orders: per tensor, at its own scale
    for li in range(len(aa.layers)):
        for part in ("kernel", "bias"):
            if aa.view(aa.grad, li, part) is not None:
                close(aa.view(aa.grad, li, part), ab.view(ab.grad, li, part), 1e-5, f"layer {li} {part} vs the 300-row trainer")


@pytest.mark.parametrize("path", ["fused_heads", "towers"])
def test_sample_weights_match_the_restatement(device, path):
    """Per-task sample weights (the second task's None) through forward_backward, on the fused-head path
    (mm_mmoe_heads_fwd_bwd) and on the tower path (mm_mmoe_task_heads_fwd_bwd)."""
    s = schema()
    mm.set_seed(12)
    model = mmoe_model(s, E=3, U=16, bottom=[32], T=0.8) if path == "fused_heads" else _towers_gates(s)
    model.build(device)
    model.compile(optimizer="sgd", loss_weights=[1.0, 0.5, 2.0])
    B = 300
    feats, targs = _batch(s, B, 6)
    rng = np.random.default_rng(3)
    sw = [(rng.random(B) * 2).astype(np.float32), None, (rng.random(B) * 3).astype(np.float32)]
    _check_gradients(model, model.trainer(B), feats, targs, sample_weight=sw)


FIVE = (("click", "bin"), ("conversion", "bin"), ("rating", "reg"), ("like", "bin"), ("watch", "reg"))


@pytest.mark.parametrize("case", ["bottom_one_layer_towers", "input_towers", "twelve_experts", "five_outputs_towers"])
def test_more_configurations_match_the_restatement(device, case):
    """One-layer towers on a shared bottom without an MMOEBlock (the head kernel's dx lands straight in G's strided
    columns), towers on the input block alone, E = 12 experts with gate blocks, and five outputs with towers (the
    kernels' NH = 8 instantiations with three tasks skipped)."""
    s = schema(targets=FIVE) if case == "five_outputs_towers" else schema()
    mm.set_seed(17)
    if case == "bottom_one_layer_towers":
        model = mm.Model(mm.InputBlockV2(s), mm.MLPBlock([32, 16]), mm.OutputBlock(s, task_blocks=mm.MLPBlock([8])))
    elif case == "input_towers":
        model = mm.Model(mm.InputBlockV2(s), mm.OutputBlock(s, task_blocks=mm.MLPBlock([16, 8])))
    elif case == "twelve_experts":
        model = mmoe_model(s, E=12, U=16, bottom=[32], T=1.2, gate=[8])
    else:
        model = mmoe_model(s, E=4, U=16, T=0.9, towers=[12], gate=[8])
    model.build(device)
    model.compile(optimizer="sgd")
    B = 300
    feats, targs = _batch(s, B, 5)
    _check_gradients(model, model.trainer(B), feats, targs)


# ---------------------------------------------------------------------------------------------------------------
# the wide kernels at B = 65 536 with bags of 27 and 100 ids
# ---------------------------------------------------------------------------------------------------------------
def _bag_ids(rng, B, L, rows, dtype):
    """(B, L) ids over [0, rows + 2): about 5 % out of range (int64: some negative too), every 50th bag one id
    repeated L times."""
    v = rng.integers(0, rows + 2, (B, L))
    v[::50] = rng.integers(0, rows, (len(v[::50]), 1))
    if dtype == torch.int64:
        v[rng.random((B, L)) < 0.01] = -3
    return v


def _encoding(v, rows, mode):
    """(B, rows) float64 encoding of fixed bags, vectorised, and the first-occurrence mask of every position."""
    B, L = v.shape
    ok = (v >= 0) & (v < rows)
    enc = np.zeros((B, rows))
    r = np.repeat(np.arange(B), L).reshape(B, L)
    np.add.at(enc, (r[ok], v[ok]), 1.0)
    key = np.where(ok, r * (rows + 1) + np.where(ok, v, 0), -1 - np.arange(B * L).reshape(B, L))
    _, first = np.unique(key.reshape(-1), return_index=True)
    is_first = np.zeros(B * L, bool)
    is_first[first] = True
    is_first = is_first.reshape(B, L) & ok
    return (np.minimum(enc, 1.0) if mode == "multi_hot" else enc), ok, is_first


@pytest.mark.parametrize("mode", ["multi_hot", "count"])
@pytest.mark.parametrize("B,L", [(BIG, 27), (RAGGED, 100), (BIG, 100), (RAGGED, 27)])
def test_wide_kernels_at_benchmark_bag_sizes(device, B, L, mode):
    """Two fixed (B, L) bag blocks (int32 and int64 ids) and three one-hot blocks, a deep part of 256 units:
    z, ds, dh, the loss and the five Dense gradients within their bounds, the out-of-range counter equal to the
    reference count; the forward alone; then mm_wide_bag_grad's (id, value) per position exactly (-1 / 0 where no term
    sits: out of range, or a repeat under multi_hot) and an SGD mm_wide_rows_apply: touched rows within the bound of
    their summed gradient, every other row bit for bit."""
    sms = _sms(device)
    ctas = min(-(-B // 16), 8 * sms)  # the head: 16 lanes per sample, 16 samples per CTA
    assert -(-B // (16 * ctas)) >= 2 and B % (16 * ctas), "premise: the head runs more than one lap, the last one ragged"
    nnz = B * L
    gctas = min(-(-nnz // 256), 16 * sms)
    assert -(-nnz // (256 * gctas)) >= 2 and nnz % (256 * gctas), "premise: the bag gradient runs more than one lap"
    rng = np.random.default_rng(L + B % 7 + (mode == "count"))
    f32 = lambda *s: torch.from_numpy(rng.standard_normal(s).astype(np.float32) * 0.4).to(device)  # noqa: E731
    onehot, oh_np, off = [], [], 0
    for w, rows in ((1, 200), (2, 3000), (4, 70)):
        ids = rng.integers(0, rows + rows // 20, B)
        onehot.append((torch.from_numpy(ids.astype({1: np.uint8, 2: np.uint16, 4: np.int32}[w])).to(device), rows, off))
        oh_np.append((ids, rows, off))
        off += rows
    bags, bag_np = [], []
    for rows, dt in ((40, torch.int32), (37, torch.int64)):
        v = _bag_ids(rng, B, L, rows, dt)
        bags.append((torch.from_numpy(v).to(device).to(dt), None, rows, off, mode))
        bag_np.append((v, rows, off))
        off += rows
    W, U = off, 256
    wide, bw = f32(W), f32(1)
    h = torch.from_numpy(np.maximum(rng.standard_normal((B, U)), 0).astype(np.float32)).to(device)
    w_dl, b_dl, out_w, out_b = f32(U), f32(1), f32(1) + 1.0, f32(1)
    y = torch.from_numpy(rng.integers(0, 2, B)).to(device)
    sw = torch.from_numpy((rng.random(B) * 2).astype(np.float32)).to(device) if mode == "count" else None
    # float64 reference
    wk = wide.double().cpu().numpy()
    wsum, wabs, n_bad, encs = np.zeros(B), np.zeros(B), 0, []
    for ids, rows, o in oh_np:
        ok = ids < rows
        n_bad += int((~ok).sum())
        t = np.where(ok, wk[o + np.minimum(ids, rows - 1)], 0.0)
        wsum, wabs = wsum + t, wabs + np.abs(t)
    for v, rows, o in bag_np:
        enc, ok, first = _encoding(v, rows, mode)
        encs.append((enc, ok, first))
        n_bad += int((~ok).sum())
        wsum, wabs = wsum + enc @ wk[o:o + rows], wabs + enc @ np.abs(wk[o:o + rows])
    D = lambda a: torch.from_numpy(np.asarray(a, np.float64)).to(device)  # noqa: E731
    h64 = h.double()
    u = h64 @ w_dl.double() + b_dl.double()
    s = D(wsum) + bw.double() + u
    es = (2 * L + len(oh_np) + 4) * EPS * (D(wabs) + bw.double().abs()) + (U + 4) * EPS * (h64 @ w_dl.double().abs() + b_dl.double().abs())
    wo = out_w.double()
    z = s * wo + out_b.double()
    ez = wo.abs() * es + 2 * EPS * z.abs()
    sw64 = sw.double() if sw is not None else torch.ones_like(z)
    y64 = y.double()
    l, g = z.clamp_min(0) - z * y64 + torch.log1p(torch.exp(-z.abs())), torch.sigmoid(z) - y64
    delta = g * sw64 / B
    ed = sw64 / B * (ez / 4 + 8 * EPS * (g.abs() + 1))
    ds, eds = delta * wo, ed * wo.abs() + EPS * (delta * wo).abs()
    chain = -(-B // (16 * ctas)) + 2 + 8 + ctas
    f = dict(dtype=torch.float32, device=device)
    r = dict(out=torch.zeros(B, **f), loss=torch.zeros(2, **f), ds=torch.zeros(B, **f), dh=torch.zeros((B, U), **f),
             dw_out=torch.zeros(1, **f), db_out=torch.zeros(1, **f), dw_dl=torch.zeros(U, **f), db_dl=torch.zeros(1, **f),
             dbw=torch.zeros(1, **f), oob=torch.zeros(1, dtype=torch.int32, device=device))
    ops.wide_deep_head_fwd_bwd(onehot, bags, wide, bw, h, True, w_dl, b_dl, "linear", out_w, out_b, r["out"], loss=BCE, targets=y,
                               sample_weight=sw, loss_buf=r["loss"], ds=r["ds"], dh=r["dh"], dw_out=r["dw_out"], db_out=r["db_out"],
                               dw_dl=r["dw_dl"], db_dl=r["db_dl"], d_wide_bias=r["dbw"], oob=r["oob"])
    torch.cuda.synchronize()
    _within(r["out"], z, ez, "z")
    _within(r["ds"], ds, eds, "ds")
    aw = w_dl.double().abs()
    _within(r["dh"], ds[:, None] * w_dl.double()[None, :] * (h > 0), eds[:, None] * aw[None, :] + EPS * (ds.abs()[:, None] * aw[None, :]), "dh")
    el = (sw64 / B * (g.abs() * ez + 4 * EPS * (l.abs() + z.abs() + 1))).sum() + chain * EPS * (sw64 * l.abs()).sum() / B
    ref_loss = (l * sw64).sum() / B
    _within(r["loss"], torch.stack([ref_loss, ref_loss]), el.expand(2), "loss")
    batch_sum = lambda v, ev: (ev.sum() + chain * EPS * v.abs().sum()).reshape(1)  # noqa: E731
    _within(r["dw_out"], (delta * s).sum().reshape(1), batch_sum(delta * s, ed * s.abs() + delta.abs() * es), "dw_out")
    _within(r["db_out"], delta.sum().reshape(1), batch_sum(delta, ed), "db_out")
    _within(r["db_dl"], ds.sum().reshape(1), batch_sum(ds, eds), "db_dl")
    _within(r["dbw"], ds.sum().reshape(1), batch_sum(ds, eds), "d_wide_bias")
    _within(r["dw_dl"], h64.t() @ ds, h64.t() @ eds + chain * EPS * (h64.t() @ ds.abs()), "dw_dl")
    assert int(r["oob"]) == n_bad, f"out-of-range counter {int(r['oob'])}, {n_bad} ids out of range"
    pred, oob = torch.zeros(B, **f), torch.zeros(1, dtype=torch.int32, device=device)
    ops.wide_deep_head_fwd_bwd(onehot, bags, wide, bw, h, True, w_dl, b_dl, "linear", out_w, out_b, pred, out_act="sigmoid", oob=oob)
    _within(pred, torch.sigmoid(z), ez / 4 + 4 * EPS, "forward")
    assert int(oob) == n_bad
    # mm_wide_bag_grad from the kernel's own ds, then an SGD step of the wide kernel
    hyper = torch.from_numpy(mm.train.get_optimizer("sgd").hyper()).to(device)
    ops.opt_tick(hyper)
    lr = float(hyper[0])
    w_new = wide.clone()
    acc = torch.zeros(W, **f)
    rep = ops.fill_i32(torch.empty(W, dtype=torch.int32, device=device), 2 ** 31 - 1)
    ds_k = r["ds"].double().cpu().numpy()
    touched = np.zeros(W, bool)
    for (bag, (v, rows, o), (enc, ok, first)) in zip(bags, bag_np, encs):
        ids = torch.empty(nnz, dtype=torch.int64, device=device)
        vals = torch.empty(nnz, **f)
        ops.wide_bag_grad(bag, B, r["ds"], ids, vals)
        term = first if mode == "multi_hot" else ok
        want_ids = np.where(term, v, -1).reshape(-1)
        want_vals = np.where(term, ds_k[:, None], 0.0).reshape(-1)
        got_ids, got_vals = ids.cpu().numpy(), vals.double().cpu().numpy()
        bad = np.nonzero((got_ids != want_ids) | (got_vals != want_vals))[0]
        assert bad.size == 0, (f"bag block ({rows} rows): {bad.size} of {nnz} pairs differ, first at position {bad[0]} "
                               f"(sample {bad[0] // L}): got ({got_ids[bad[0]]}, {got_vals[bad[0]]}), want ({want_ids[bad[0]]}, "
                               f"{want_vals[bad[0]]})")
        before = w_new.clone()
        ops.wide_rows_apply("sgd", w_new, None, None, [ids], [rows], [o], vals, acc, rep, [], None, None, None, None, hyper)
        torch.cuda.synchronize()
        gsum = enc.T @ ds_k
        gabs = enc.T @ np.abs(ds_k)
        cnt = enc.sum(0)
        ref = before[o:o + rows].double() - lr * D(gsum)
        _within(w_new[o:o + rows], ref, lr * (D(cnt) + 1) * EPS * D(gabs) + EPS * ref.abs(), f"sgd rows of block {o}")
        touched[o:o + rows] |= cnt > 0
        assert float(acc.abs().sum()) == 0 and int((rep != 2 ** 31 - 1).sum()) == 0, "scratch not cleared"
    keep = torch.from_numpy(~touched).to(device)
    assert torch.equal(w_new[keep].view(torch.int32), wide[keep].view(torch.int32)), "a row no id touched changed"


# ---------------------------------------------------------------------------------------------------------------
# WideAndDeepTrainer at the benchmark's size, against the sparse restatement
# ---------------------------------------------------------------------------------------------------------------
BAG_SIZES = [3, 2, 1, 2, 6, 1, 1, 1, 1, 7, 3, 8, 1, 6, 9, 5, 1, 1, 1, 12, 100, 27, 10, 3, 1, 1]  # C1..C26, MLPerf DLRM-DCNv2


@pytest.mark.parametrize("leg", ["one_hot", "multi_hot"])
def test_wide_and_deep_benchmark_size_step(device, leg):
    """One step at B = 65 536 on the Criteo schema (tables capped at 20 000 rows), deep_block MLPBlock([1024, 512, 256]),
    the 26 categorical columns on the wide side, Adagrad(0.01): one-hot ids at inferred embedding widths, or fixed
    (B, L) bags of the MLPerf sizes on both sides (multi_hot, deep embedding width 32).  Loss, logits, every dense
    gradient, the tables' gradients and the wide kernel / bias gradients against the sparse float64 restatement (with the
    device's relu decisions: a table row gathers the gradient of a few samples, so one pre-activation on the other side
    of the kink would show); then the update: wide rows no id touched keep their bits."""
    from tests.test_gpu_wide_deep import TOL as WTOL, _oracle_state
    from tests.wide_deep_train_oracle import encode_sparse, wide_deep_loss_and_grads

    B = BIG
    multihot = leg == "multi_hot"
    s = datasets.criteo_schema({k: min(v, 20000) for k, v in datasets.CRITEO_MAX.items()})
    cats = list(s.select_by_tag(Tags.CATEGORICAL))
    ws = s.select_by_name([c.name for c in cats])
    mm.set_seed(6)
    deep_in = mm.InputBlockV2(s, categorical=mm.Embeddings(s.select_by_tag(Tags.CATEGORICAL), dim=32)) if multihot else None
    model = mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([1024, 512, 256]), wide_schema=ws, deep_input_block=deep_in,
                                wide_preprocess=mm.CategoryEncoding(ws, output_mode="multi_hot" if multihot else "one_hot"),
                                prediction_tasks=mm.BinaryOutput(s.select_by_tag(Tags.TARGET).column_names[0]))
    model.build(device)
    model.compile(optimizer=mm.Adagrad(0.01))
    rng = np.random.default_rng(21 + multihot)
    f = {}
    for i, c in enumerate(cats):
        L = BAG_SIZES[i] if multihot else 1
        f[c.name] = rng.integers(0, c.int_domain.max + 1, (B, L) if L > 1 else B).astype(np.int32)
    f.update({c.name: rng.random(B).astype(np.float32) for c in s.select_by_tag(Tags.CONTINUOUS)})
    y = (rng.random(B) < 0.3).astype(np.float32)
    tr = model.trainer(B)
    tr.forward_backward({k: torch.from_numpy(v).to(device) for k, v in f.items()}, torch.from_numpy(y).to(device))
    torch.cuda.synchronize()
    wide, deep, head = _oracle_state(model)
    masks = {f"deep_{i}": (tr.h[i][:B] > 0).cpu().numpy() for i in range(len(model.body.deep.dense_layers))}
    L_, z, g = wide_deep_loss_and_grads(f, wide, deep, head, y, sparse=True, masks=masks)
    close(tr.loss[0], L_, 1e-5, "loss")
    close(tr.logits[:B], z, 1e-4, "logits")
    grads = tr.gradients()
    name = model.prediction.to_call.name
    close(grads[f"{name}/kernel"], g["head/kernel"], WTOL, "head/kernel")
    close(grads[f"{name}/bias"], g["head/bias"], WTOL, "head/bias")
    for i, l in enumerate(model.body.deep.dense_layers):
        close(grads[f"{l.name}/kernel"], g[f"deep/kernel_{i}"], WTOL, f"deep/kernel_{i}")
        close(grads[f"{l.name}/bias"], g[f"deep/bias_{i}"], WTOL, f"deep/bias_{i}")
    dl = model.body.deep_logit.dense_layers[0]
    close(grads[f"{dl.name}/kernel"], g["deep_logit/kernel"], WTOL, "deep_logit/kernel")
    close(grads[f"{dl.name}/bias"], g["deep_logit/bias"], WTOL, "deep_logit/bias")
    tr._bag_grads()
    for t, fname in enumerate(tr.feats):  # IndexedSlices (one-hot) or the bags' expanded rows, scattered in float64
        rows, D = tr.tables[t].table.shape
        bag = tr._bags.get(t)
        ids, sl = (bag["apply_ids"], bag["rows"]) if bag is not None else (tr._idx[t], tr._slices[t])
        ids = ops.widen_index(ids).reshape(-1).long()
        ok = (ids >= 0) & (ids < rows)
        dense = torch.zeros((rows, D), dtype=torch.float64, device=device)
        dense.index_add_(0, ids[ok], sl.reshape(-1, D)[ok].double())
        close(dense, g[f"table/{fname}"], WTOL, f"table/{fname}")
    wg = tr.wide_gradients()
    close(wg["wide/kernel"], g["wide/kernel"], WTOL, "wide/kernel")
    close(wg["wide/bias"], g["wide/bias"], WTOL, "wide/bias")
    # the update: rows of the wide kernel that no id of the batch encodes keep their bits
    hit = np.concatenate([np.asarray(encode_sparse(f[n], wide["cards"][n], wide["mode"]).sum(0)).reshape(-1) > 0
                          for n in sorted(wide["cards"])])
    assert not hit.all()
    wk0 = model.body.wide.dense.kernel.detach().clone().reshape(-1)
    tr.apply_gradients()
    tr._after_step()
    torch.cuda.synchronize()
    wk1 = model.body.wide.dense.kernel.detach().reshape(-1)
    keep = torch.from_numpy(~hit).to(device)
    assert torch.equal(wk1[keep].view(torch.int32), wk0[keep].view(torch.int32)), "a wide row no id touched changed"
    assert not torch.equal(wk1[~keep], wk0[~keep]), "no touched wide row moved"
