"""Learning-rate schedules and MultiOptimizer in every trainer's update stage: after each step every parameter and slot
equals the float64 Keras update at lr(s) of that step's gradients, eagerly and as graph replays; a MultiOptimizer whose
groups all use the same optimizer updates the dense arena and the tied table bit-identically to that optimizer (sparse
rows up to the fold order of duplicate ids); the session-based example's optimizer and the LazyAdam use case train."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets, ops, train
from models_b200.blocks import WideLinear
from models_b200.optimizer import block_variables_owners
from oracle.oracle_train import dense_update
from tests import catalog_model_oracle as O
from tests import test_gpu_mmoe as MM
from tests import test_gpu_ncf as NCF
from tests import test_gpu_train as DL
from tests import test_gpu_train_dcn as DCN
from tests import test_gpu_train_deepfm as DFM
from tests import test_gpu_train_twotower as TT
from tests import test_gpu_wide_deep as WD
from tests.test_mmoe_host import mmoe_model, schema as mmoe_schema

pytestmark = pytest.mark.gpu

B = 256


def _dev(f, device):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in f.items()}


# ---- the nine families: (model, batches of (inputs, targets), the block holding a wide kernel or None) --------------
def _dlrm(device):
    schema, model = DL._small_model(device, D=16, bottom=(32, 16), top=(32, 16))
    out = []
    for i in range(4):
        f, t = datasets.split_targets(schema, datasets.generate_batch(schema, B, seed=40 + i, index_law="uniform"))
        out.append((_dev(f, device), model._targets_by_output(_dev(t, device))))
    return model, out, None


def _dcn(device):
    model = DCN._dcn()
    return model, [(_dev(f, device), torch.from_numpy(y).to(device)) for f, y in (DCN._batch(B, 40 + i) for i in range(4))], None


def _deepfm(device):
    model = DFM._deepfm()
    return model, [(_dev(f, device), torch.from_numpy(y).to(device)) for f, y in (DFM._batch(B, 40 + i) for i in range(4))], \
        lambda m: m.body.fm.wide


def _wide_deep(device):
    model = WD._model(3)
    return model, [(_dev(f, device), torch.from_numpy(y).to(device)) for f, y in (WD._batch(B, 40 + i) for i in range(4))], \
        lambda m: block_variables_owners(m, (WideLinear,))[0]


def _mmoe(device):
    mm.set_seed(3)
    s = mmoe_schema()
    model = mmoe_model(s, bottom=[32])
    out = []
    for i in range(4):
        f, t = MM._batch(s, B, 40 + i)
        out.append((_dev(f, device), model._targets_by_output(MM._targets(model, t, device))))
    return model, out, None


def _ncf(device):
    model = NCF._random_model(3)
    return model, [NCF._dev_batch(u, i, y) for u, i, y in NCF._random_batches(4, B, 300, 500, seed=40)], None


def _twotower(device):
    schema, model = TT._ml1m_model(dims=(32, 16))
    return model, [(_dev(TT._batch(schema, B, 40 + i), device), None) for i in range(4)], None


def _mf(device):
    mm.set_seed(3)
    schema = datasets.movielens_1m_schema()
    model = mm.MatrixFactorizationModel(schema, dim=32)
    return model, [(_dev(TT._batch(schema, B, 40 + i), device), None) for i in range(4)], None


def _catalog(device):
    model, s, _ = O.build(900, 32, "list", T=0.5, seed=5, n_users=300)
    out = []
    for i in range(4):
        f, y = O.batch(s, 900, B, seed=40 + i, hot=3)
        out.append((_dev(f, device), torch.from_numpy(y).to(device)))
    return model, out, None


# the MovieLens schema's ragged `genres` trains eagerly only: those families are checked eagerly, without graph replays
EAGER_ONLY = {"twotower", "mf"}

FAMILIES = {"dlrm": _dlrm, "dcn": _dcn, "deepfm": _deepfm, "wide_deep": _wide_deep, "mmoe": _mmoe, "ncf": _ncf,
            "twotower": _twotower, "mf": _mf, "catalog": _catalog}


def _tables(model):
    """Every embedding table of the model (the item table of the catalog model included), largest last."""
    ts = {id(t): t for e in model.embedding_blocks() for t in e.tables.values()}
    return sorted(ts.values(), key=lambda t: t.input_dim)


# ---- the float64 Keras update of one step --------------------------------------------------------------------------
def _lr(g, s):
    sch = g.opt.schedule
    return sch(s) if sch is not None else g.opt.learning_rate


def _upd(g, w, grad, s1, s2, s):
    """(w, s1, s2) after one float64 Keras update of `grad` with group g at step index s."""
    st = {}
    if g.kind == "adagrad":
        st["a"] = s1
    elif g.kind == "adam":
        st["m"], st["v"] = s1, s2
    o = g.opt
    w = dense_update(g.kind, w, grad, st, _lr(g, s), beta_1=float(np.float32(o.beta_1)), beta_2=float(np.float32(o.beta_2)),
                     epsilon=float(np.float32(o.epsilon)), step=s + 1)
    return w, st.get("a", st.get("m")), st.get("v")


def _np(t):
    return None if t is None else t.detach().double().cpu().numpy()


def _expected_update(tr, s):
    """What apply_gradients must leave, from the state and the gradients after forward_backward: [(what, tensor, want)]."""
    out = []
    a = tr.arena
    idx, slices, rows, scale = tr._gradients_to_apply()
    for lo, hi, g in a.runs:
        w, s1, s2 = _upd(g, _np(a.w[lo:hi]), _np(a.grad[lo:hi]) * scale, _np(None if a.state1 is None else a.state1[lo:hi]),
                         _np(None if a.state2 is None else a.state2[lo:hi]), s)
        out += [(f"arena[{lo}:{hi}] {g.kind}", a.w[lo:hi], w)]
        if g.slots >= 1:
            out.append((f"arena[{lo}:{hi}] slot 1", a.state1[lo:hi], s1))
        if g.slots >= 2:
            out.append((f"arena[{lo}:{hi}] slot 2", a.state2[lo:hi], s2))
    for t, tb in enumerate(tr.tables):
        if t == getattr(tr, "tt", None):  # the weight-tied table trains densely below
            continue
        g = tr.tgroup[t]
        bag = tr._bags.get(t)
        ids, vals = (bag["apply_ids"], bag["rows"]) if bag is not None else (idx[t][:rows], slices[t][:rows])
        ids = ops.widen_index(ids).reshape(-1).long().cpu().numpy()
        vals = _np(vals).reshape(len(ids), -1)
        W = _np(tb.table)
        ok = (ids >= 0) & (ids < W.shape[0])
        G = np.zeros_like(W)
        np.add.at(G, ids[ok], vals[ok])
        touched = np.unique(ids[ok])
        s1, s2 = _np(tr.tstate1[t]), _np(tr.tstate2[t])
        w_t, a_t, v_t = _upd(g, W[touched], G[touched], None if s1 is None else s1[touched], None if s2 is None else s2[touched], s)
        W[touched] = w_t
        out.append((f"table {tb.table_name} {g.kind}", tb.table, W))
        if s1 is not None:
            s1[touched] = a_t
            out.append((f"table {tb.table_name} slot 1", tr.tstate1[t], s1))
        if s2 is not None:
            s2[touched] = v_t
            out.append((f"table {tb.table_name} slot 2", tr.tstate2[t], s2))
    wk = tr.wk
    if isinstance(wk, train._WideKernel):
        g = wk.group
        assert g.kind != "adam", "the check updates every wide row; lazy Adam would move only the touched ones"
        grads = wk.gradients()
        w, s1, _ = _upd(g, _np(wk.dense.kernel).reshape(-1), _np(grads["wide/kernel"]).reshape(-1), _np(wk.wk_s1), None, s)
        out.append(("wide kernel", wk.dense.kernel.reshape(-1), w))
        if wk.dense.bias is not None:
            b, _, _ = _upd(g, _np(wk.dense.bias), _np(grads["wide/bias"]), _np(wk.wb_s1), None, s)
            out.append(("wide bias", wk.dense.bias, b))
    elif isinstance(wk, train._TiedTable):
        w, s1, s2 = _upd(wk.gE, _np(wk.E), _np(wk.dE), _np(wk.s1), _np(wk.s2), s)
        out += [("tied table", wk.E, w)] + ([("tied table slot 1", wk.s1, s1)] if s1 is not None else []) + \
            ([("tied table slot 2", wk.s2, s2)] if s2 is not None else [])
        if wk.bias is not None:
            b, _, _ = _upd(wk.gb, _np(wk.bias), _np(wk.db), _np(wk.b_s1), _np(wk.b_s2), s)
            out.append(("tied bias", wk.bias, b))
    return out


def _close(what, got, want):
    got = _np(got).reshape(want.shape)
    scale = max(1.0, float(np.abs(want).max()) if want.size else 1.0)
    err = float(np.abs(got - want).max()) if want.size else 0.0
    assert err <= 2e-6 * scale, f"{what}: max |err| {err:.3e} (scale {scale:.3e})"


def _state(tr):
    return {k: v.detach().clone() for k, v in tr._state().items() if v is not None}


def _train(family, opt, device, graph: bool, check: bool):
    """4 steps of the family's model under opt; the state after each step (eager: checked against float64)."""
    model, batches, _ = FAMILIES[family](device)
    model.build(device)
    model.compile(optimizer=opt() if callable(opt) else opt)
    tr = model.trainer(B)
    states = []
    if graph:
        tr.capture(*batches[0])
        for x, y in batches:
            tr.replay(x, y)
            states.append(_state(tr))
        return tr, states
    for s, (x, y) in enumerate(batches):
        tr.forward_backward(x, y)
        want = _expected_update(tr, s) if check else []
        tr.apply_gradients()
        tr._after_step()
        for what, got, w in want:
            _close(f"{family} step {s}: {what}", got, w)
        for g in tr._groups.groups:  # each group's own step counter and lr(s) on the device
            assert float(g.hyper[4]) == s + 1 and float(g.hyper[0]) == pytest.approx(_lr(g, s), rel=1e-6)
        states.append(_state(tr))
    return tr, states


def _same(a, b, rel):
    assert a.keys() == b.keys()
    for k in a:
        x, y = a[k].double(), b[k].double()
        if y.numel():
            scale = max(1.0, float(y.abs().max()))
            assert float((x - y).abs().max()) <= rel * scale, k


# ---- a schedule on one optimizer -----------------------------------------------------------------------------------
SCHEDULED = {f: (lambda: mm.Adagrad(mm.schedules.ExponentialDecay(0.05, 2, 0.5, staircase=True)))
             if i % 2 == 0 else (lambda: mm.SGD(mm.schedules.PiecewiseConstantDecay([0, 2], [0.05, 0.02, 0.01])))
             for i, f in enumerate(FAMILIES)}


@pytest.mark.parametrize("family", list(FAMILIES))
def test_schedule_eager_and_graph_replay_follow_keras(device, family):
    tr, eager = _train(family, SCHEDULED[family], device, graph=False, check=True)
    assert [g.sched is not None for g in tr._groups.groups] == [True]
    if family in EAGER_ONLY:
        return
    tr_g, replay = _train(family, SCHEDULED[family], device, graph=True, check=False)
    for s, (e, r) in enumerate(zip(eager, replay)):
        _same(r, e, 1e-5)
    assert float(tr_g.hyper[0]) == np.float32(SCHEDULED[family]().schedule(3))


# ---- a MultiOptimizer split --------------------------------------------------------------------------------------
def _split(model, wide):
    """Tables by size between Adagrad and Adam, every other variable under SGD with a schedule, the wide kernel (where
    there is one) under its own Adagrad."""
    ts = _tables(model)
    large, small = mm.split_embeddings_on_size(model.embedding_blocks()[0], ts[-1].input_dim) \
        if len(model.embedding_blocks()) == 1 else ([ts[-1]], ts[:-1])
    pairs = [mm.OptimizerBlocks(mm.Adagrad(0.05), large)]
    if small:
        pairs.append(mm.OptimizerBlocks(mm.Adam(0.01, epsilon=1e-3), small))
    if wide is not None:
        pairs.append(mm.OptimizerBlocks(mm.Adagrad(0.02, initial_accumulator_value=0.3), wide(model)))
    return mm.MultiOptimizer(pairs, default_optimizer=mm.SGD(mm.schedules.ExponentialDecay(0.05, 2, 0.5, staircase=True)))


@pytest.mark.parametrize("family", list(FAMILIES))
def test_multi_optimizer_split_follows_keras(device, family):
    model2, batches, wide = FAMILIES[family](device)
    model2.build(device)
    model2.compile(optimizer=_split(model2, wide))
    tr2 = model2.trainer(B)
    kinds = sorted(g.kind for g in tr2._groups.groups)
    assert "adagrad" in kinds and "adam" in kinds, kinds
    if tr2.arena.runs:  # matrix factorization has no Dense layer: nothing falls to the scheduled SGD default
        assert "sgd" in kinds and any(g.sched is not None for g in tr2._groups.groups)
    eager = []
    for s, (x, y) in enumerate(batches):
        tr2.forward_backward(x, y)
        want = _expected_update(tr2, s)
        tr2.apply_gradients()
        tr2._after_step()
        for what, got, w in want:
            _close(f"{family} step {s}: {what}", got, w)
        eager.append(_state(tr2))
    if family in EAGER_ONLY:
        return
    model3, batches3, _ = FAMILIES[family](device)
    model3.build(device)
    model3.compile(optimizer=_split(model3, wide))
    tr3 = model3.trainer(B)
    tr3.capture(*batches3[0])
    for s, (x, y) in enumerate(batches3):
        tr3.replay(x, y)
        _same(_state(tr3), eager[s], 1e-5)


# ---- every group the same optimizer: bit-identical to that optimizer ----------------------------------------------
def _grad_buffers(tr):
    out = [tr.arena.grad]
    out += list(tr.slices) if isinstance(tr.slices, list) else [tr.slices]
    out += [b["rows"] for b in tr._bag_bufs.values() if b["rows"] is not None]
    wk = tr.wk
    if isinstance(wk, train._WideKernel):
        out += [wk.grad] + [c[3] for c in wk.calls]
    elif isinstance(wk, train._TiedTable):
        out.append(wk.grad)
    return out


@pytest.mark.parametrize("family", list(FAMILIES))
def test_multi_optimizer_of_one_kind_is_bit_identical(device, family):
    trs = []
    for multi in (False, True):
        model, batches, wide = FAMILIES[family](device)
        model.build(device)
        if multi:
            ts = _tables(model)
            opt = mm.MultiOptimizer([mm.OptimizerBlocks(mm.Adagrad(0.05), ts[-1:]), mm.OptimizerBlocks(mm.Adagrad(0.05), ts[:-1])]
                                    + ([mm.OptimizerBlocks(mm.Adagrad(0.05), wide(model))] if wide else []),
                                    default_optimizer=mm.Adagrad(0.05))
        else:
            opt = mm.Adagrad(0.05)
        model.compile(optimizer=opt)
        trs.append((model.trainer(B), batches))
    (t1, batches), (t2, _) = trs
    assert len(t1._groups.groups) == 1 and len(t2._groups.groups) >= 2
    for x, y in batches[:3]:
        t1.forward_backward(x, y)
        t2.forward_backward(x, y)
        for a, b in zip(_grad_buffers(t1), _grad_buffers(t2)):  # the same gradients into both update stages
            b.copy_(a)
        t1.apply_gradients()
        t2.apply_gradients()
        s1, s2 = t1._state(), t2._state()
        for k, v in s1.items():
            if v is None or k.startswith("hyper"):
                continue
            if k.startswith(("table", "wide")):
                # the sparse and wide row updates fold three or more duplicates of an id in arrival order, so two calls on
                # the same gradients may differ in the last bits; the arena and the tied table must not
                assert float((v.double() - s2[k].double()).abs().max()) <= 1e-6 * max(1.0, float(v.abs().max())), k
            else:
                assert torch.equal(v, s2[k]), f"{family}: {k} differs"


def test_single_optimizer_launches_unchanged(device):
    """One plain optimizer: one tick, one dense apply, sparse applies per width; a schedule swaps the tick only."""
    counts = {}
    for name, opt in (("plain", mm.Adagrad(0.05)), ("sched", mm.Adagrad(mm.schedules.ExponentialDecay(0.05, 2, 0.5)))):
        model, batches, _ = _dcn(device)
        model.build(device)
        model.compile(optimizer=opt)
        tr = model.trainer(B)
        tr.capture(*batches[0])
        counts[name] = tr.launches_per_step
    assert counts["plain"] == counts["sched"]


# ---- the reference's examples ---------------------------------------------------------------------------------------
def test_session_example_optimizer_fits_and_replays(device):
    """Model(InputBlockV2, MLPBlock([128, D], no_activation_last_layer=True, dropout=0.2), CategoricalOutput(table,
    logits_temperature=0.05)) with Adam(ExponentialDecay(...)) and label smoothing: fit runs, graph replay equals eager."""
    n_items, D, eps, T = 400, 32, 0.1, 0.05

    def build():
        mm.set_seed(3)
        s = O.schema(n_items, "onehot")
        emb = mm.Embeddings(s.select_by_tag(mm.Tags.CATEGORICAL), dim=D)
        model = mm.Model(mm.InputBlockV2(s, categorical=emb), mm.MLPBlock([128, D], no_activation_last_layer=True, dropout=0.2),
                         mm.CategoricalOutput(to_call=emb.tables["item_id"], logits_temperature=T, target_name="next_item"))
        opt = mm.Adam(learning_rate=mm.schedules.ExponentialDecay(0.005, decay_steps=2, decay_rate=0.96, staircase=True))
        model.compile(optimizer=opt, loss=mm.losses.CategoricalCrossEntropy(from_logits=True, label_smoothing=eps))
        return s, model

    s, model = build()
    data = [(_dev(f, device), torch.from_numpy(((3 * f["last_item"] + 1) % n_items).astype(np.int64)).to(device))
            for f, _ in (O.batch(s, n_items, B, seed=100 + i) for i in range(4))]
    hist = model.fit(data, epochs=3)
    assert len(hist.history["loss"]) == 3 and np.isfinite(hist.history["loss"]).all()
    assert float(model._trainer.hyper[4]) == 12
    runs = []
    for graph in (False, True):
        _, m = build()
        m.build(device)
        tr = m.trainer(B)
        if graph:
            tr.capture(*data[0])
        for x, y in data:
            tr.replay(x, y) if graph else tr.step(x, y)
        runs.append(_state(tr))
    _same(runs[1], runs[0], 1e-5)


def test_lazy_adam_use_case_lowers_the_loss(device):
    """examples/usecases/accelerate-training-of-large-embedding-tables-by-LazyAdam: a TwoTowerModel with LazyAdam on the
    large tables and Adam on the small ones (split_embeddings_on_size), Adam by default."""
    schema, model = TT._ml1m_model(dims=(32, 16))
    model.build(device)
    embeddings = model.embedding_blocks()
    large, small = [], []
    for e in embeddings:
        lg, sm = mm.split_embeddings_on_size(e, threshold=1000)
        large += lg
        small += sm
    assert large and small
    opt = mm.MultiOptimizer(default_optimizer="adam", optimizers_and_blocks=[
        mm.OptimizerBlocks(mm.LazyAdam(), large), mm.OptimizerBlocks("adam", small)])
    model.compile(optimizer=opt)
    data = [_dev(TT._batch(schema, B, 7), device)] * 8
    hist = model.fit(data, batch_size=B, epochs=4)
    loss = hist.history["loss"]
    assert loss[-1] < loss[0], loss
    assert len(model._trainer._groups.groups) == 3
