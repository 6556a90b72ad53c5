"""Torch-tensor front end of the C-ABI (include/mm_b200.h).

PyTorch is used for device memory and streams only: every function here checks its
arguments, takes raw device pointers and calls one entry point of libmm_b200.so on the
current CUDA stream.  There is no CPU path — a CPU tensor is an error.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Sequence

import numpy as np
import torch

from . import _cabi
from ._cabi import ACTIVATIONS, COMBINERS, GatherTable, MM_I32, MM_I64, MM_MAX_TABLES


def _lib():
    return _cabi.load()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _dev(t: torch.Tensor, name: str, dtype=None) -> torch.Tensor:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor, got {type(t).__name__}")
    if not t.is_cuda:
        raise RuntimeError(
            f"{name} is on {t.device}: the models_b200 hot path only runs on CUDA (no CPU fallback)"
        )
    if dtype is not None and t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")
    return t


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _vec(t: Optional[torch.Tensor], n: int, name: str, what: str = "hold {n} contiguous values") -> None:
    """Checks that t is None or an fp32 vector of n contiguous values; the error says f"{name} must {what}"."""
    if t is not None and (_dev(t, name, torch.float32).numel() != n or not t.is_contiguous()):
        raise ValueError(f"{name} must " + what.format(n=n))


def _idx_dtype(t: torch.Tensor, name: str) -> int:
    if t.dtype == torch.int32:
        return MM_I32
    if t.dtype == torch.int64:
        return MM_I64
    raise TypeError(f"{name} must be int32 or int64, got {t.dtype}")


def _row_stride(t: torch.Tensor, name: str) -> int:
    if t.dim() != 2 or t.stride(1) != 1:
        raise ValueError(f"{name} must be 2-D with unit inner stride, got shape {tuple(t.shape)} strides {t.stride()}")
    return t.stride(0)


def launch_count() -> int:
    return int(_lib().mm_launch_count())


def init_uniform_hash(w: torch.Tensor, seed: int, lo: float = -0.05, hi: float = 0.05) -> torch.Tensor:
    _dev(w, "w", torch.float32)
    if not w.is_contiguous():
        raise ValueError("w must be contiguous")
    _cabi.check(_lib().mm_init_uniform_hash(w.data_ptr(), w.numel(), seed & (2**64 - 1), lo, hi, _stream()),
                "mm_init_uniform_hash")
    return w


def _table_array(weights: Sequence[torch.Tensor], indices: Sequence[torch.Tensor], out_cols: Sequence[int], B: int):
    n = len(weights)
    if not (1 <= n <= MM_MAX_TABLES):
        raise ValueError(f"between 1 and {MM_MAX_TABLES} tables per launch, got {n}")
    if not (len(indices) == n and len(out_cols) == n):
        raise ValueError("weights / indices / out_cols length mismatch")
    arr = (GatherTable * n)()
    dt = _idx_dtype(indices[0], "indices[0]")
    for t in range(n):
        w = _dev(weights[t], f"weights[{t}]", torch.float32)
        ix = _dev(indices[t], f"indices[{t}]")
        if w.dim() != 2 or not w.is_contiguous():
            raise ValueError(f"weights[{t}] must be a contiguous (rows, dim) matrix")
        if _idx_dtype(ix, f"indices[{t}]") != dt:
            raise TypeError("all index tensors of one launch must share a dtype")
        if ix.numel() != B or not ix.is_contiguous():
            raise ValueError(f"indices[{t}] must be contiguous with {B} elements, got {tuple(ix.shape)}")
        arr[t].weights = w.data_ptr()
        arr[t].indices = ix.data_ptr()
        arr[t].rows = w.shape[0]
        arr[t].dim = w.shape[1]
        arr[t].out_col = int(out_cols[t])
    return arr, n, dt


def gather_multi(weights, indices, out_cols, out: torch.Tensor, oob: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[b, out_cols[t] : out_cols[t]+dim_t] = weights[t][indices[t][b]]   (mm_gather_multi)."""
    _dev(out, "out", torch.float32)
    B = out.shape[0]
    stride = _row_stride(out, "out")
    if B == 0:
        return out
    for s in range(0, len(weights), MM_MAX_TABLES):
        e = min(len(weights), s + MM_MAX_TABLES)
        arr, n, dt = _table_array(weights[s:e], indices[s:e], out_cols[s:e], B)
        _cabi.check(_lib().mm_gather_multi(arr, n, dt, B, out.data_ptr(), stride, _ptr(oob), _stream()),
                    "mm_gather_multi")
    return out


def gather_bag(weight, values, offsets, combiner: str, out: torch.Tensor, out_col: int = 0,
               oob: Optional[torch.Tensor] = None) -> torch.Tensor:
    _dev(weight, "weight", torch.float32), _dev(values, "values"), _dev(offsets, "offsets"), _dev(out, "out", torch.float32)
    if combiner not in ("mean", "sum", "sqrtn"):
        raise ValueError(f"combiner must be mean, sum or sqrtn, got {combiner!r}")
    B = out.shape[0]
    if offsets.numel() != B + 1:
        raise ValueError(f"offsets must have B+1={B + 1} elements, got {offsets.numel()}")
    _cabi.check(
        _lib().mm_gather_bag(weight.data_ptr(), weight.shape[0], weight.shape[1], values.data_ptr(),
                             _idx_dtype(values, "values"), offsets.data_ptr(), _idx_dtype(offsets, "offsets"),
                             B, COMBINERS[combiner], out.data_ptr(), _row_stride(out, "out"), out_col,
                             _ptr(oob), _stream()),
        "mm_gather_bag")
    return out


def gather_seq(weight, ids, combiner: str, out: torch.Tensor, out_col: int = 0,
               oob: Optional[torch.Tensor] = None) -> torch.Tensor:
    _dev(weight, "weight", torch.float32), _dev(ids, "ids"), _dev(out, "out", torch.float32)
    if combiner not in ("mean", "sum", "max"):
        raise ValueError(f"sequence combiner must be mean, sum or max, got {combiner!r}")
    if ids.dim() != 2 or not ids.is_contiguous():
        raise ValueError("ids must be a contiguous (B, L) matrix")
    B, L = ids.shape
    _cabi.check(
        _lib().mm_gather_seq(weight.data_ptr(), weight.shape[0], weight.shape[1], ids.data_ptr(),
                             _idx_dtype(ids, "ids"), B, L, COMBINERS[combiner], out.data_ptr(),
                             _row_stride(out, "out"), out_col, _ptr(oob), _stream()),
        "mm_gather_seq")
    return out


def _split_out_args(out: torch.Tensor):
    """(fp32 ptr, fp32 stride, split ptr, out_Kp) for an output that is either fp32 (B, W) or the
    split-bf16 operand (B, 2*Kp) of a following tensor-core layer."""
    if out.dtype == torch.bfloat16:
        if out.dim() != 2 or not out.is_contiguous() or out.shape[1] % 128 != 0:
            raise ValueError("a split-bf16 output must be contiguous (B, 2*Kp) with Kp a multiple of 64")
        return None, 0, out.data_ptr(), out.shape[1] // 2
    _dev(out, "out", torch.float32)
    return out.data_ptr(), _row_stride(out, "out"), None, 0


def dot_interaction(x: torch.Tensor, out: torch.Tensor, prefix: Optional[torch.Tensor] = None,
                    self_interaction: bool = False) -> torch.Tensor:
    """x (B,F,D) -> out[:, :P] = prefix, out[:, P:] = upper-triangle pairwise dots.
    `out` fp32 (B, >=P+pairs) or bf16 (B, 2*Kp) = split operand of the next tensor-core layer."""
    _dev(x, "x", torch.float32), _dev(out, "out")
    if x.dim() != 3 or not x.is_contiguous():
        raise ValueError("x must be a contiguous (B, F, D) tensor")
    B, F, D = x.shape
    P = 0 if prefix is None else prefix.shape[1]
    o32, ostride, osplit, okp = _split_out_args(out)
    _cabi.check(
        _lib().mm_dot_interaction(x.data_ptr(), B, F, D, F * D, _ptr(prefix), P,
                                  0 if prefix is None else _row_stride(_dev(prefix, "prefix", torch.float32), "prefix"),
                                  int(self_interaction), o32, ostride, osplit, okp, _stream()),
        "mm_dot_interaction")
    return out


def scale_shift(x: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = x * scale + shift per column (BatchNormalization at inference; mm_scale_shift)."""
    _dev(x, "x", torch.float32), _dev(scale, "scale", torch.float32), _dev(shift, "shift", torch.float32)
    out = torch.empty_like(x) if out is None else _dev(out, "out", torch.float32)
    B, D = x.shape
    if scale.numel() != D or shift.numel() != D:
        raise ValueError(f"scale / shift must have {D} elements")
    _cabi.check(_lib().mm_scale_shift(x.data_ptr(), B, D, _row_stride(x, "x"), scale.data_ptr(), shift.data_ptr(),
                                      out.data_ptr(), _row_stride(out, "out"), _stream()), "mm_scale_shift")
    return out


def cross_combine(x0: torch.Tensor, proj: torch.Tensor, x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out = x0 * proj + x (mm_cross_combine)."""
    for n, t in (("x0", x0), ("proj", proj), ("x", x), ("out", out)):
        _dev(t, n, torch.float32)
    B, D = x.shape
    _cabi.check(_lib().mm_cross_combine(x0.data_ptr(), proj.data_ptr(), x.data_ptr(), B, D, _row_stride(x0, "x0"),
                                        _row_stride(proj, "proj"), _row_stride(x, "x"), out.data_ptr(), _row_stride(out, "out"),
                                        _stream()), "mm_cross_combine")
    return out


def index_bytes_of(t: torch.Tensor) -> int:
    """Width in bytes of the ids a categorical column carries: int32 -> 4, int64 -> 8, and the packed
    host-batch forms uint8 (B,) -> 1, uint16 (B,) -> 2, uint8 (B, 3) -> 3 (little-endian 24-bit)."""
    if t.dtype == torch.int32:
        return 4
    if t.dtype == torch.int64:
        return 8
    if t.dtype == torch.uint16:
        return 2
    if t.dtype == torch.uint8:
        return 3 if (t.dim() == 2 and t.shape[1] == 3) else 1
    raise TypeError(f"ids must be int32, int64, uint16, uint8 or uint8 (B,3), got {t.dtype} {tuple(t.shape)}")


def widen_index(t: torch.Tensor) -> torch.Tensor:
    """Packed ids -> int32 (torch ops; only the paths that do not take packed ids natively use this)."""
    w = index_bytes_of(t)
    if w >= 4:
        return t
    if w == 3:
        b = t.to(torch.int32)
        return b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)
    return t.reshape(-1).to(torch.int32)


def as_index(t: torch.Tensor) -> torch.Tensor:
    """Ids as int32 / int64, the two index dtypes of the gather kernels: the forms of index_bytes_of are widened
    (widen_index), any other dtype is cast to int32 as the reference does (inputs/embedding.py:1127-1129)."""
    try:
        return widen_index(t)
    except TypeError:
        return t.to(torch.int32)


def fused_ids(t: torch.Tensor) -> torch.Tensor:
    """Ids as the fused lookup kernels take them (dlrm_lookup_interact, dlrm_interact_backward, deepfm_head,
    sparse_rows_apply): packed host-batch ids (uint8, uint16, uint8 (B, 3)) at their own width, others as (B,) as_index."""
    return t if t.dtype in (torch.uint8, torch.uint16) else as_index(t).reshape(-1)


def _id_column(ix: torch.Tensor, B: int, name: str, leading: bool = False) -> int:
    """index_bytes_of a column of B contiguous ids (a uint8 (B, 3) column holds B ids).  leading: its first dimension must
    also be B."""
    _dev(ix, name)
    wb = index_bytes_of(ix)
    if ix.numel() != B * (3 if wb == 3 else 1) or not ix.is_contiguous() or (leading and ix.shape[0] != B):
        raise ValueError(f"{name} must be {B} contiguous ids, got {tuple(ix.shape)}")
    return wb


def _lookup_tables(weights, indices, B: int, wdt: torch.dtype, wcols: int, slots=None, rows=None):
    """mm_lookup_table array: table t is weights[t], a contiguous (rows, wcols) wdt matrix, read at the B ids indices[t]
    (any width of index_bytes_of), staged at slots[t] (default t), with rows[t] rows (default weights[t].shape[0])."""
    arr = (_cabi.LookupTable * len(weights))()
    for t in range(len(weights)):
        w = _dev(weights[t], f"weights[{t}]", wdt)
        if w.dim() != 2 or w.shape[1] != wcols or not w.is_contiguous():
            raise ValueError(f"weights[{t}] must be a contiguous (rows, {wcols}) {wdt} matrix")
        arr[t].idx_bytes = _id_column(indices[t], B, f"indices[{t}]")
        arr[t].weights, arr[t].indices = w.data_ptr(), indices[t].data_ptr()
        arr[t].rows = w.shape[0] if rows is None else int(rows[t])
        arr[t].slot = t if slots is None else int(slots[t])
    return arr


def pairs_cols(n_pairs: int) -> int:
    """Columns per half of a pairs-only operand row (dlrm_lookup_interact(pairs_only=True), mlp_tc(a_bottom=...)): the pair
    count rounded up to 8, so that each half is whole 16-byte groups."""
    return (int(n_pairs) + 7) // 8 * 8


def dlrm_lookup_interact(weights, indices, slots, rows, D: int, bottom: Optional[torch.Tensor], bottom_slot: int,
                         out: torch.Tensor, oob: Optional[torch.Tensor] = None, peers=None, rank: int = 0,
                         world: int = 1, operand_rows: bool = False, pairs_only: bool = False) -> torch.Tensor:
    """Fused lookup + interaction with per-table id widths and optional row-sharded tables
    (mm_dlrm_lookup_interact).  weights[t]: the (rows, D) table or this rank's shard; indices[t]: (B,) ids
    (any width, see index_bytes_of); rows[t]: GLOBAL row count; peers[t]: None (replicated) or the `world`
    device pointers of the shards as mapped in this process.  operand_rows=True (D = 64): `weights`, the peers' shards
    and `bottom` are bf16 split rows (rows, 2*D) = [hi | lo] (split_rows / mlp_tc(out_operand=...)); needs a split-bf16
    `out`.  pairs_only=True (with operand_rows and a bottom vector): `out` is (B, 2*pairs_cols(F(F-1)/2)) bf16 and gets the
    pairs only, [hi | lo] (MM_ROWS_OPERAND_PAIRS); the top tower reads the bottom rows from `bottom` (mlp_tc(a_bottom=...))."""
    _dev(out, "out")
    if pairs_only and (not operand_rows or bottom is None):
        raise ValueError("pairs_only needs operand_rows and a bottom vector")
    B = out.shape[0]
    n = len(weights)
    if not (len(indices) == n and len(slots) == n and len(rows) == n):
        raise ValueError("weights / indices / slots / rows length mismatch")
    keep = []
    wdt, wcols = (torch.bfloat16, 2 * D) if operand_rows else (torch.float32, D)
    if operand_rows and bottom is not None and (bottom.dtype != torch.bfloat16 or bottom.shape[1] != 2 * D):
        raise ValueError(f"operand_rows: bottom must be bf16 split rows (B, {2 * D})")
    arr = _lookup_tables(weights, indices, B, wdt, wcols, slots, rows)
    for t in range(n):
        pt = None if peers is None else peers[t]
        if pt is not None:
            if len(pt) != world:
                raise ValueError(f"peers[{t}] must list {world} shard pointers")
            pa = (C.c_void_p * world)(*[int(x) for x in pt])
            keep.append(pa)
            arr[t].peer_weights_host = C.cast(pa, C.POINTER(C.c_void_p))
    if pairs_only:
        F = n + 1
        if out.dtype != torch.bfloat16 or tuple(out.shape) != (B, 2 * pairs_cols(F * (F - 1) // 2)) or not out.is_contiguous():
            raise ValueError(f"pairs_only: out must be a contiguous bf16 ({B}, {2 * pairs_cols(F * (F - 1) // 2)}) matrix")
        o32, ostride, osplit, okp = None, 0, out.data_ptr(), out.shape[1] // 2
    else:
        o32, ostride, osplit, okp = _split_out_args(out)
    _cabi.check(
        _lib().mm_dlrm_lookup_interact(arr, n, B, D, rank, world, _ptr(bottom),
                                       0 if bottom is None else (_row_stride(_dev(bottom, "bottom", wdt), "bottom") // (2 if operand_rows else 1)),
                                       bottom_slot, o32, ostride, osplit, okp, _ptr(oob), 2 if pairs_only else 1 if operand_rows else 0,
                                       _stream()),
        "mm_dlrm_lookup_interact")
    return out


def dense_fp32(x: torch.Tensor, W: torch.Tensor, bias: Optional[torch.Tensor], act: Optional[str],
               out: torch.Tensor, x0: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = act(x @ W + bias)   or, with x0, the DCN-v2 cross  out = x0 * (x @ W + bias) + x."""
    _dev(x, "x", torch.float32), _dev(W, "W", torch.float32), _dev(out, "out", torch.float32)
    if act not in ACTIVATIONS:
        raise ValueError(f"unsupported activation {act!r}; supported: {sorted(k for k in ACTIVATIONS if k)}")
    if W.dim() != 2 or not W.is_contiguous():
        raise ValueError("W must be a contiguous (K, N) matrix")
    K, N = W.shape
    if x.shape[1] != K:
        raise ValueError(f"x has {x.shape[1]} columns but the kernel has {K} rows")
    B = x.shape[0]
    _cabi.check(
        _lib().mm_dense_fp32(x.data_ptr(), B, K, _row_stride(x, "x"), W.data_ptr(), _ptr(bias), N,
                             ACTIVATIONS[act], _ptr(x0), 0 if x0 is None else _row_stride(x0, "x0"),
                             out.data_ptr(), _row_stride(out, "out"), _stream()),
        "mm_dense_fp32")
    return out


def rowwise_dot(q: torch.Tensor, items: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    _dev(q, "q", torch.float32), _dev(items, "items", torch.float32), _dev(out, "out", torch.float32)
    B, D = q.shape
    _cabi.check(_lib().mm_rowwise_dot(q.data_ptr(), items.data_ptr(), B, D, _row_stride(q, "q"),
                                      _row_stride(items, "items"), out.data_ptr(), _stream()),
                "mm_rowwise_dot")
    return out


def _item_ids(pos_ids, neg_ids, downscore: bool):
    """(pos_ids, neg_ids, id dtype code) for the false-negative mask of the in-batch kernels: with downscore, both as
    contiguous (B,) / (N,) vectors of the negative ids' dtype (utils/tf_utils.py:136 casts the positive ids to it);
    without, None (the kernels read no ids)."""
    if not downscore:
        return None, None, MM_I64
    if pos_ids is None or neg_ids is None:
        raise ValueError("downscore_false_negatives requires positive and negative item ids")
    neg_ids = neg_ids.reshape(-1).contiguous()
    pos_ids = pos_ids.reshape(-1).to(neg_ids.dtype).contiguous()
    return pos_ids, neg_ids, _idx_dtype(neg_ids, "neg_ids")


def inbatch_scores(q, pos, neg, out, pos_ids=None, neg_ids=None, downscore=True,
                   false_neg_score: float = -655.04, pos_prob=None, neg_prob=None,
                   temperature: float = 1.0, tensor_cores: bool = True) -> torch.Tensor:
    """out (B, 1+N) = [q.pos | masked(q @ neg^T)] / T  (include/mm_b200.h: mm_inbatch_scores[_tc]).
    tensor_cores=True: wgmma split-bf16 GEMM (fp32-grade); False: exact fp32 CUDA-core kernel."""
    for n_, t_ in (("q", q), ("pos", pos), ("neg", neg)):
        _dev(t_, n_, torch.float32)
        if not t_.is_contiguous():
            raise ValueError(f"{n_} must be contiguous")
    _dev(out, "out", torch.float32)
    if out.dim() != 2 or out.stride(1) != 1 or out.shape[1] != neg.shape[0] + 1:
        raise ValueError("out must be (B, 1+N) with unit inner stride")
    B, D = q.shape
    N = neg.shape[0]
    pos_ids, neg_ids, id_dt = _item_ids(pos_ids, neg_ids, downscore)
    if tensor_cores and N > 0 and B > 0:
        _cabi.check(_lib().mm_positive_scores(q.data_ptr(), pos.data_ptr(), B, D, _ptr(pos_prob), float(temperature),
                                              out.data_ptr(), out.stride(0), _stream()), "mm_positive_scores")
        qs = split_rows(q)
        ns = qs if neg.data_ptr() == q.data_ptr() else split_rows(neg)
        _cabi.check(
            _lib().mm_inbatch_scores_tc(qs.data_ptr(), ns.data_ptr(), B, N, D, _ptr(pos_ids), _ptr(neg_ids), id_dt,
                                        int(bool(downscore)), float(false_neg_score), _ptr(neg_prob),
                                        float(temperature), out.data_ptr(), out.stride(0), _stream()),
            "mm_inbatch_scores_tc")
        return out
    _cabi.check(
        _lib().mm_inbatch_scores(q.data_ptr(), pos.data_ptr(), neg.data_ptr(), B, N, D, _ptr(pos_ids),
                                 _ptr(neg_ids), id_dt, int(bool(downscore)), float(false_neg_score),
                                 _ptr(pos_prob), _ptr(neg_prob), float(temperature), out.data_ptr(),
                                 out.stride(0), _stream()),
        "mm_inbatch_scores")
    return out


def inbatch_softmax_ce(q, pos, neg, pos_ids=None, neg_ids=None, downscore=True, false_neg_score: float = -655.04,
                       pos_prob=None, neg_prob=None, temperature: float = 1.0) -> torch.Tensor:
    """(B,3) = [row max, log-sum-exp, positive logit] of the in-batch contrastive logits [q.pos | masked(q @ neg^T)] / T —
    the inputs of softmax cross-entropy against the one-hot target on column 0 — without materialising the (B, 1+N)
    logits (mm_positive_scores + mm_inbatch_softmax_ce).  loss = stats[:,1] - stats[:,2]."""
    for n_, t_ in (("q", q), ("pos", pos), ("neg", neg)):
        _dev(t_, n_, torch.float32)
        if not t_.is_contiguous():
            raise ValueError(f"{n_} must be contiguous")
    B, D = q.shape
    N = neg.shape[0]
    if N == 0 or B == 0:
        raise ValueError("in-batch softmax needs at least one query and one negative")
    pos_logit = torch.empty((B, 1), dtype=torch.float32, device=q.device)
    stats = torch.empty((B, 3), dtype=torch.float32, device=q.device)
    ws = _catalog_workspace(B, N, 0, q.device)
    positive_scores(q, pos, pos_logit, pos_prob, temperature)
    qs = split_rows(q)
    ns = qs if neg.data_ptr() == q.data_ptr() else split_rows(neg)
    return inbatch_softmax_ce_split(qs, ns, D, pos_logit, stats, ws, pos_ids, neg_ids, downscore, false_neg_score, neg_prob,
                                    temperature)


def positive_scores(q: torch.Tensor, pos: torch.Tensor, out: torch.Tensor, pos_prob=None, temperature: float = 1.0) -> torch.Tensor:
    """out (B,) = (q . pos - log(pos_prob + 1e-16)) / T, row-wise (mm_positive_scores): column 0 of the in-batch logits."""
    for n_, t_ in (("q", q), ("pos", pos), ("out", out)):
        _dev(t_, n_, torch.float32)
    if not (q.is_contiguous() and pos.is_contiguous()) or q.shape != pos.shape or out.numel() != q.shape[0]:
        raise ValueError("q and pos must be contiguous (B, D) and out hold B values")
    _cabi.check(_lib().mm_positive_scores(q.data_ptr(), pos.data_ptr(), q.shape[0], q.shape[1], _ptr(pos_prob), float(temperature),
                                          out.data_ptr(), 1, _stream()), "mm_positive_scores")
    return out


def inbatch_softmax_ce_split(q_split, neg_split, D: int, pos_logit, stats, workspace, pos_ids=None, neg_ids=None, downscore=True,
                             false_neg_score: float = -655.04, neg_prob=None, temperature: float = 1.0) -> torch.Tensor:
    """inbatch_softmax_ce on split operands the caller owns (mm_inbatch_softmax_ce): stats (B, 3) from q_split (B, 2*Kp),
    neg_split (N, 2*Kp) and pos_logit (B,); workspace: uint8 of at least catalog_workspace_bytes(B, N) bytes.  Nothing is
    allocated, so a training step can be captured into a CUDA graph."""
    _dev(q_split, "q_split", torch.bfloat16), _dev(neg_split, "neg_split", torch.bfloat16)
    _dev(pos_logit, "pos_logit", torch.float32), _dev(stats, "stats", torch.float32), _dev(workspace, "workspace", torch.uint8)
    B, N = q_split.shape[0], neg_split.shape[0]
    if stats.numel() != 3 * B or not stats.is_contiguous() or pos_logit.numel() != B:
        raise ValueError(f"stats must be contiguous ({B}, 3) and pos_logit hold {B} values")
    pos_ids, neg_ids, id_dt = _item_ids(pos_ids, neg_ids, downscore)
    _cabi.check(
        _lib().mm_inbatch_softmax_ce(q_split.data_ptr(), neg_split.data_ptr(), B, N, int(D), _ptr(pos_ids), _ptr(neg_ids), id_dt,
                                     int(bool(downscore)), float(false_neg_score), pos_logit.data_ptr(), _ptr(neg_prob),
                                     float(temperature), stats.data_ptr(), workspace.data_ptr(), workspace.numel(), _stream()),
        "mm_inbatch_softmax_ce")
    return stats


def catalog_workspace_bytes(B: int, N: int, k: int = 0) -> int:
    return int(_lib().mm_catalog_workspace_bytes(int(B), int(N), int(k)))


def _catalog_workspace(B: int, N: int, k: int, device) -> torch.Tensor:
    """uint8 workspace of the catalog-scoring kernel for B queries, N items and top-k (at least 16 bytes)."""
    return torch.empty(max(catalog_workspace_bytes(B, N, k), 16), dtype=torch.uint8, device=device)


def inbatch_softmax_ce_backward(q_split, neg_split, D: int, stats, q, pos, row_scale, dq, dpos, dneg, loss=None, pos_ids=None,
                                neg_ids=None, downscore=True, false_neg_score: float = -655.04, neg_prob=None,
                                temperature: float = 1.0) -> None:
    """Backward of inbatch_softmax_ce (mm_inbatch_softmax_ce_backward): from the split operands the forward read
    (q_split (B, 2*Kp), neg_split (N, 2*Kp)) and its stats (B, 3), writes dq, dpos (B, D) and dneg (N, D) of
    sum_b c[b] (lse[b] - s[b,0]) and adds that loss to `loss` (nullable).  row_scale: (B,) or (1,) fp32 c.  dpos may be
    dneg (in-batch negatives, N == B): the sum is written."""
    B, N = _inbatch_buffers(D, q_split, neg_split, stats, 3, (q, pos, dq, dpos, dneg), extra=(("row_scale", row_scale),),
                            joint=False)
    if loss is not None:
        _dev(loss, "loss", torch.float32)
    _vec(neg_prob, N, "neg_prob")
    if loss is not None and loss.numel() < 1:
        raise ValueError("loss must hold at least one value")
    if row_scale.numel() not in (1, B):
        raise ValueError(f"row_scale must hold 1 or {B} values, got {row_scale.numel()}")
    scalar = row_scale.numel() == 1 and B != 1
    pos_ids, neg_ids, id_dt = _item_ids(pos_ids, neg_ids, downscore)
    _cabi.check(
        _lib().mm_inbatch_softmax_ce_backward(q_split.data_ptr(), neg_split.data_ptr(), B, N, int(D), _ptr(pos_ids), _ptr(neg_ids),
                                              id_dt, int(bool(downscore)), float(false_neg_score), _ptr(neg_prob), float(temperature),
                                              stats.data_ptr(), q.data_ptr(), pos.data_ptr(), row_scale.data_ptr(), int(scalar),
                                              dq.data_ptr(), dpos.data_ptr(), dneg.data_ptr(), _ptr(loss), _stream()),
        "mm_inbatch_softmax_ce_backward")


def catalog_softmax_ce_workspace_bytes(B: int, N: int, D: int) -> int:
    """Bytes of the partial-dX workspace catalog_softmax_ce_backward needs for these shapes (0: the catalog is not split)."""
    return int(_lib().mm_catalog_softmax_ce_workspace_bytes(int(B), int(N), int(D)))


def catalog_smoothed_ce_workspace_bytes(B: int, N: int, D: int) -> int:
    """Bytes of the workspace catalog_softmax_ce_backward needs with label_smoothing > 0, and catalog_mean_logit needs."""
    return int(_lib().mm_catalog_smoothed_ce_workspace_bytes(int(B), int(N), int(D)))


def _check_label_smoothing(label_smoothing) -> float:
    eps = float(label_smoothing)
    if not 0.0 <= eps < 1.0:
        raise ValueError(f"label_smoothing must be in [0, 1), got {label_smoothing}")
    return eps


def catalog_softmax_ce_backward(x_split, e_split, D: int, stats, labels, row_scale, dx, de, db=None, bias=None, loss=None,
                                temperature: float = 1.0, workspace=None, oob=None, label_smoothing: float = 0.0) -> None:
    """Backward of the full-catalog soft-max cross-entropy (mm_catalog_softmax_ce_backward) from the operands
    catalog_score read for `stats` (B, 3): x_split = split_rows(x / T) (B, 2*Kp), e_split = split_rows(E) (N, 2*Kp) and
    bias (N,) = b / T (None: no bias).  With G = c (softmax - onehot(labels)) of the logits (x E^T + b) / T, writes dx
    (B, D) = G E / T, the gradient of x itself; de (N, D) = G^T x / T; db (N,) = sum_b G / T (None: not written); and
    adds sum_b c[b] (lse[b] - logit[b, label]) to `loss` (nullable).  labels (B,) int32 / int64 class ids; a label
    outside [0, N) is never used as an address: it takes no one-hot term (its loss term is NaN) and adds one to `oob`
    (nullable int32 counter, the gathers' out-of-range counter).  row_scale: (B,) or (1,) fp32 c.  workspace: uint8 of at
    least catalog_softmax_ce_workspace_bytes(B, N, D) bytes; None allocates one (not during graph capture).

    label_smoothing = eps in [0, 1): the target is (1 - eps) onehot(labels) + eps / N (Keras CategoricalCrossentropy's
    label_smoothing), so G = c (softmax - (1 - eps) onehot - eps / N) and the loss is sum_b c[b] (lse[b] - (1 - eps)
    logit[b, label] - eps mean_j logit[b, j]) (mm_catalog_smoothed_ce_backward; the workspace must then hold
    catalog_smoothed_ce_workspace_bytes(B, N, D) bytes).  eps = 0 is the call above, bit for bit."""
    eps = _check_label_smoothing(label_smoothing)
    B, N = _inbatch_buffers(D, x_split, e_split, stats, 3, extra=(("row_scale", row_scale),), joint=True)
    for n_, t_, shape in (("dx", dx, (B, D)), ("de", de, (N, D))):
        if tuple(_dev(t_, n_, torch.float32).shape) != shape or not t_.is_contiguous():
            raise ValueError(f"{n_} must be contiguous {shape}, got {tuple(t_.shape)}")
    if dx.data_ptr() == de.data_ptr():
        raise ValueError("dx and de must be distinct buffers")
    _vec(db, N, "db")
    _vec(bias, N, "bias")
    if loss is not None and _dev(loss, "loss", torch.float32).numel() < 1:
        raise ValueError("loss must hold at least one value")
    if row_scale.numel() not in (1, B):
        raise ValueError(f"row_scale must hold 1 or {B} values, got {row_scale.numel()}")
    if not float(temperature) > 0.0:
        raise ValueError(f"temperature must be positive, got {temperature}")
    labels = _dev(labels, "labels").reshape(-1)
    if labels.numel() != B or not labels.is_contiguous():
        raise ValueError(f"labels must hold {B} contiguous class ids, got {tuple(labels.shape)}")
    label_dt = _idx_dtype(labels, "labels")
    if oob is not None and (_dev(oob, "oob", torch.int32).numel() < 1):
        raise ValueError("oob must hold at least one int32 counter")
    need = catalog_softmax_ce_workspace_bytes(B, N, D) if eps == 0.0 else catalog_smoothed_ce_workspace_bytes(B, N, D)
    if workspace is None:
        workspace = torch.empty(max(need, 16), dtype=torch.uint8, device=x_split.device)
    elif _dev(workspace, "workspace", torch.uint8).numel() < need:
        raise ValueError(f"workspace must hold at least {need} bytes, got {workspace.numel()}")
    scalar = row_scale.numel() == 1 and B != 1
    if eps > 0.0:
        _cabi.check(
            _lib().mm_catalog_smoothed_ce_backward(x_split.data_ptr(), e_split.data_ptr(), B, N, int(D), _ptr(bias),
                                                   labels.data_ptr(), label_dt, float(temperature), eps, stats.data_ptr(),
                                                   row_scale.data_ptr(), int(scalar), dx.data_ptr(), de.data_ptr(), _ptr(db),
                                                   _ptr(loss), _ptr(oob), workspace.data_ptr(), workspace.numel(), _stream()),
            "mm_catalog_smoothed_ce_backward")
        return
    _cabi.check(
        _lib().mm_catalog_softmax_ce_backward(x_split.data_ptr(), e_split.data_ptr(), B, N, int(D), _ptr(bias), labels.data_ptr(),
                                              label_dt, float(temperature), stats.data_ptr(), row_scale.data_ptr(), int(scalar),
                                              dx.data_ptr(), de.data_ptr(), _ptr(db), _ptr(loss), _ptr(oob), workspace.data_ptr(),
                                              workspace.numel(), _stream()),
        "mm_catalog_softmax_ce_backward")


def catalog_mean_logit(x_split, e_split, D: int, bias=None, out=None, workspace=None) -> torch.Tensor:
    """(B,) mean_j of the logits x_split[b] . e_j + bias_j over the N catalog rows (mm_catalog_mean_logit), from the split
    operands catalog_score reads (x_split (B, 2*Kp) of the tempered queries, e_split (N, 2*Kp), bias (N,) = b / T or
    None): the logit of the label-smoothed target's uniform part.  workspace: uint8 of at least
    mm_catalog_mean_logit_workspace_bytes(N) bytes; None allocates one."""
    _dev(x_split, "x_split", torch.bfloat16), _dev(e_split, "e_split", torch.bfloat16)
    B, N = x_split.shape[0], e_split.shape[0]
    _vec(bias, N, "bias")
    if out is None:
        out = torch.empty(B, dtype=torch.float32, device=x_split.device)
    elif _dev(out, "out", torch.float32).numel() != B or not out.is_contiguous():
        raise ValueError(f"out must be contiguous ({B},)")
    need = int(_lib().mm_catalog_mean_logit_workspace_bytes(int(N)))
    if workspace is None:
        workspace = torch.empty(max(need, 16), dtype=torch.uint8, device=x_split.device)
    elif _dev(workspace, "workspace", torch.uint8).numel() < need:
        raise ValueError(f"workspace must hold at least {need} bytes, got {workspace.numel()}")
    _cabi.check(
        _lib().mm_catalog_mean_logit(x_split.data_ptr(), e_split.data_ptr(), B, N, int(D), _ptr(bias), out.data_ptr(),
                                     workspace.data_ptr(), workspace.numel(), _stream()),
        "mm_catalog_mean_logit")
    return out


def catalog_stats_split(x_split, D: int, e_split, stats, labels, workspace, bias=None) -> torch.Tensor:
    """catalog_score's soft-max statistics on operands the caller owns (mm_catalog_score with k = 0): stats (B, 3) =
    [max, log-sum-exp, logit[label]] of x_split (B, 2*Kp) against e_split (N, 2*Kp) with bias (N,) (nullable); workspace:
    uint8 of at least catalog_workspace_bytes(B, N) bytes.  Nothing is allocated, so a training step can be captured."""
    _dev(x_split, "x_split", torch.bfloat16), _dev(e_split, "e_split", torch.bfloat16)
    _dev(stats, "stats", torch.float32), _dev(workspace, "workspace", torch.uint8)
    B, N = x_split.shape[0], e_split.shape[0]
    if stats.numel() != 3 * B or not stats.is_contiguous():
        raise ValueError(f"stats must be contiguous ({B}, 3)")
    _vec(bias, N, "bias")
    labels = _dev(labels, "labels").reshape(-1)
    if labels.numel() != B or not labels.is_contiguous():
        raise ValueError(f"labels must hold {B} contiguous class ids, got {tuple(labels.shape)}")
    _cabi.check(
        _lib().mm_catalog_score(x_split.data_ptr(), B, int(D), e_split.data_ptr(), N, _ptr(bias), labels.data_ptr(),
                                _idx_dtype(labels, "labels"), stats.data_ptr(), 0, None, None, workspace.data_ptr(),
                                workspace.numel(), _stream()),
        "mm_catalog_score")
    return stats


def slices_add_dense_workspace_bytes(n: int) -> int:
    """Bytes of the workspace slices_add_dense needs for n slices."""
    return int(_lib().mm_slices_add_dense_workspace_bytes(int(n)))


def slices_add_dense(ids, rows, dense, workspace=None) -> None:
    """dense (N, D) += the IndexedSlices (ids (n,) int32 / int64, rows (n, D)) (mm_slices_add_dense): duplicates summed in
    index order, one writer per row, no float atomics (bit-identical repeats); ids outside [0, N) add nothing.
    workspace: uint8 of at least slices_add_dense_workspace_bytes(n) bytes; None allocates one (not during graph capture)."""
    ids = _dev(ids, "ids").reshape(-1)
    _dev(rows, "rows", torch.float32), _dev(dense, "dense", torch.float32)
    n = ids.numel()
    if dense.dim() != 2 or not dense.is_contiguous():
        raise ValueError(f"dense must be a contiguous (N, D) matrix, got {tuple(dense.shape)}")
    N, D = dense.shape
    if tuple(rows.shape) != (n, D) or not rows.is_contiguous() or not ids.is_contiguous():
        raise ValueError(f"rows must be contiguous ({n}, {D}) and ids hold {n} contiguous values, got {tuple(rows.shape)}")
    need = slices_add_dense_workspace_bytes(n)
    if workspace is None:
        workspace = torch.empty(max(need, 16), dtype=torch.uint8, device=dense.device)
    elif _dev(workspace, "workspace", torch.uint8).numel() < need:
        raise ValueError(f"workspace must hold at least {need} bytes, got {workspace.numel()}")
    _cabi.check(
        _lib().mm_slices_add_dense(ids.data_ptr(), _idx_dtype(ids, "ids"), rows.data_ptr(), n, D, dense.data_ptr(), N,
                                   workspace.data_ptr(), workspace.numel(), _stream()),
        "mm_slices_add_dense")


def _inbatch_buffers(D: int, q_split, neg_split, stats, stats_cols: int, grads=None, extra=(), joint=True) -> tuple:
    """The buffers every in-batch kernel reads: the split operands q_split (B, 2*Kp) and neg_split (N, 2*Kp), bf16, and
    the fp32 stats (B, stats_cols); with grads = (q, pos, dq, dpos, dneg), a backward's fp32 q, pos, dq, dpos (B, D) and
    dneg (N, D); extra: more (name, fp32 tensor) pairs of any shape.  All contiguous on the device; returns (B, N).
    joint: one "X must be contiguous (shape), got ..." error per tensor (the pairwise wrappers); otherwise the soft-max
    backward's separate "X must be contiguous", "X must be (shape), got ..." and "q_split and neg_split must be
    contiguous"."""
    _dev(q_split, "q_split", torch.bfloat16), _dev(neg_split, "neg_split", torch.bfloat16)
    B, N = q_split.shape[0], neg_split.shape[0]
    Kp = tc_padded_k(D)
    fp32 = [("stats", stats, (B, stats_cols))]
    if grads is not None:
        fp32 += list(zip(("q", "pos", "dq", "dpos", "dneg"), grads, [(B, D)] * 4 + [(N, D)]))
    for n_, t_ in [(n_, t_) for n_, t_, _ in fp32] + list(extra):
        _dev(t_, n_, torch.float32)
        if not joint and not t_.is_contiguous():
            raise ValueError(f"{n_} must be contiguous")
    for n_, t_, shape in [("q_split", q_split, (B, 2 * Kp)), ("neg_split", neg_split, (N, 2 * Kp))] + fp32:
        if tuple(t_.shape) != shape or (joint and not t_.is_contiguous()):
            raise ValueError(f"{n_} must be {'contiguous ' if joint else ''}{shape}, got {tuple(t_.shape)}")
    if not (q_split.is_contiguous() and neg_split.is_contiguous()):
        raise ValueError("q_split and neg_split must be contiguous")
    return B, N


def _pairwise_args(kind: str, reg_lambda: float, q_split, neg_split, D: int, pos_logit, stats, grads=None) -> tuple:
    """The checks mm_inbatch_pairwise_fwd / _bwd share (grads: as _inbatch_buffers); returns (B, N, kind code)."""
    if kind not in _cabi.PAIRWISE_KINDS:
        raise ValueError(f"pairwise loss kind must be among {sorted(_cabi.PAIRWISE_KINDS)}, got {kind!r}")
    if not math.isfinite(float(reg_lambda)):
        raise ValueError(f"reg_lambda must be finite, got {reg_lambda}")
    _dev(pos_logit, "pos_logit", torch.float32)
    B, N = _inbatch_buffers(D, q_split, neg_split, stats, 4, grads)
    if N == 0:
        raise ValueError("in-batch pairwise losses need at least one negative")
    _vec(pos_logit, B, "pos_logit")
    return B, N, _cabi.PAIRWISE_KINDS[kind]


def inbatch_pairwise(q_split, neg_split, D: int, pos_logit, stats, kind: str, loss=None, pos_ids=None, neg_ids=None,
                     downscore=True, false_neg_score: float = -655.04, temperature: float = 1.0,
                     reg_lambda: float = 1.0) -> torch.Tensor:
    """Forward of an in-batch pairwise ranking loss (mm_inbatch_pairwise_fwd): kind one of _cabi.PAIRWISE_KINDS (the
    reference's names "bpr", "bpr-max", "top1", "top1_v2", "top1-max", "logistic", "hinge"); the positive scores
    pos_logit (B,) (positive_scores, already / T) against the masked scores q_split @ neg_split^T / T.  Writes stats
    (B, 4) = [row loss, dloss/dsp, log-sum-exp, A] for inbatch_pairwise_backward and adds the mean loss over the B N
    elements to `loss` (nullable, one float).  Nothing is allocated, so a training step can be captured into a CUDA graph."""
    B, N, code = _pairwise_args(kind, reg_lambda, q_split, neg_split, D, pos_logit, stats)
    if loss is not None and (_dev(loss, "loss", torch.float32).numel() < 1):
        raise ValueError("loss must hold at least one value")
    pos_ids, neg_ids, id_dt = _item_ids(pos_ids, neg_ids, downscore)
    _cabi.check(
        _lib().mm_inbatch_pairwise_fwd(q_split.data_ptr(), neg_split.data_ptr(), B, N, int(D), _ptr(pos_ids), _ptr(neg_ids), id_dt,
                                       int(bool(downscore)), float(false_neg_score), float(temperature), code, float(reg_lambda),
                                       pos_logit.data_ptr(), stats.data_ptr(), _ptr(loss), _stream()),
        "mm_inbatch_pairwise_fwd")
    return stats


def inbatch_pairwise_backward(q_split, neg_split, D: int, pos_logit, stats, q, pos, dq, dpos, dneg, kind: str, pos_ids=None,
                              neg_ids=None, downscore=True, false_neg_score: float = -655.04, temperature: float = 1.0,
                              reg_lambda: float = 1.0) -> None:
    """Backward of inbatch_pairwise (mm_inbatch_pairwise_bwd) from the operands and stats of the forward: writes dq, dpos
    (B, D) and dneg (N, D) of the mean loss.  dpos may be dneg (in-batch negatives, N == B): the sum is written."""
    B, N, code = _pairwise_args(kind, reg_lambda, q_split, neg_split, D, pos_logit, stats, (q, pos, dq, dpos, dneg))
    if dpos.data_ptr() == dneg.data_ptr() and N != B:
        raise ValueError("dpos may be dneg only when the negatives are the positives (N == B)")
    if dq.data_ptr() in (dpos.data_ptr(), dneg.data_ptr()):
        raise ValueError("dq must not alias dpos / dneg")
    pos_ids, neg_ids, id_dt = _item_ids(pos_ids, neg_ids, downscore)
    _cabi.check(
        _lib().mm_inbatch_pairwise_bwd(q_split.data_ptr(), neg_split.data_ptr(), B, N, int(D), _ptr(pos_ids), _ptr(neg_ids), id_dt,
                                       int(bool(downscore)), float(false_neg_score), float(temperature), code, float(reg_lambda),
                                       pos_logit.data_ptr(), stats.data_ptr(), q.data_ptr(), pos.data_ptr(), dq.data_ptr(),
                                       dpos.data_ptr(), dneg.data_ptr(), _stream()),
        "mm_inbatch_pairwise_bwd")


_CONCAT_DTYPES = {torch.int32: _cabi.MM_I32, torch.int64: _cabi.MM_I64, torch.float32: _cabi.MM_F32,
                  torch.float64: _cabi.MM_F64}


def _concat_pieces(pieces: Sequence[torch.Tensor], B: int, name: str = "pieces", out_cols: Optional[Sequence[int]] = None,
                   max_width: Optional[int] = None):
    """(mm_concat_piece array, pieces in it, row width) of the (B,) / (B, w) input columns `pieces`, read as fp32 into
    columns out_cols[i] (default: one after the other).  max_width: wider pieces are split into pieces of that width."""
    flat, col = [], 0
    for i, t in enumerate(pieces):
        _dev(t, f"{name}[{i}]")
        if t.dtype not in _CONCAT_DTYPES:
            raise TypeError(f"{name}[{i}]: unsupported dtype {t.dtype}")
        if t.dim() == 1:
            t = t.unsqueeze(1)
        if t.dim() != 2 or t.shape[0] != B or (t.shape[1] > 1 and t.stride(1) != 1):
            raise ValueError(f"{name}[{i}] must be (B,) or (B,w) with unit inner stride, got {tuple(t.shape)}")
        w = int(t.shape[1])
        oc = col if out_cols is None else int(out_cols[i])
        for c0 in range(0, w, max_width) if max_width else [0]:
            flat.append((t.data_ptr() + c0 * t.element_size(), t.stride(0), min(max_width, w - c0) if max_width else w,
                         _CONCAT_DTYPES[t.dtype], oc + c0))
        col = oc + w
    arr = (_cabi.ConcatPiece * max(len(flat), 1))()
    for i, (ptr, sstride, w, dt, oc) in enumerate(flat):
        arr[i].src, arr[i].src_stride, arr[i].width, arr[i].dtype, arr[i].out_col = ptr, sstride, w, dt, oc
    return arr, len(flat), col


def _cont_columns(cont, cont_offsets, B: int):
    """(mm_concat_piece array, offsets array, count) of the continuous columns cont, B values each, at cont_offsets."""
    m = len(cont)
    if len(cont_offsets) != m:
        raise ValueError("cont / cont_offsets length mismatch")
    for c, t in enumerate(cont):
        if _dev(t, f"cont[{c}]").numel() != B:
            raise ValueError(f"cont[{c}] must hold {B} values")
    carr, _, _ = _concat_pieces([t.reshape(-1) for t in cont], B, "cont")
    return carr, (C.c_int64 * max(m, 1))(*[int(o) for o in cont_offsets]), m


def concat_columns(pieces: Sequence[torch.Tensor], out: torch.Tensor, out_cols: Optional[Sequence[int]] = None,
                   max_width: int = 256) -> torch.Tensor:
    """out[:, out_cols[i] : out_cols[i]+w_i] = float32(pieces[i])  — (B,) pieces count as (B,1).

    Pieces must already be in the reference's sorted-name order (core/aggregation.py:54-66)."""
    _dev(out, "out", torch.float32)
    B = out.shape[0]
    stride = _row_stride(out, "out")
    # very wide pieces are split so that a launch tile fits in shared memory
    arr, n, _ = _concat_pieces(pieces, B, out_cols=out_cols, max_width=max_width)
    groups, cur, cur_w = [], [], 0
    for f in arr[:n]:
        if cur and (cur_w + f.width > max_width or len(cur) == 64):
            groups.append(cur)
            cur, cur_w = [], 0
        cur.append(f)
        cur_w += f.width
    if cur:
        groups.append(cur)
    for g in groups:
        ga = (_cabi.ConcatPiece * len(g))(*g)
        _cabi.check(_lib().mm_concat_columns(ga, len(g), B, out.data_ptr(), stride, _stream()), "mm_concat_columns")
    return out


def concat_split_supported(pieces: Sequence[torch.Tensor]) -> bool:
    """mm_concat_split handles up to 64 pieces and 320 padded columns in one launch."""
    width = sum(1 if t.dim() == 1 else int(t.shape[1]) for t in pieces)
    return 0 < len(pieces) <= 64 and tc_padded_k(width) <= 320 and all(t.dtype in _CONCAT_DTYPES for t in pieces)


def concat_split(pieces: Sequence[torch.Tensor], out: Optional[torch.Tensor] = None):
    """ConcatFeatures + bf16 split in one launch (mm_concat_split): returns (a_split (B, 2*Kp) bf16, K).
    Pieces in the reference's sorted-name order; (B,) pieces count as (B,1)."""
    B = pieces[0].shape[0]
    arr, n, K = _concat_pieces(pieces, B)
    Kp = tc_padded_k(K)
    if out is None:
        out = torch.empty((B, 2 * Kp), dtype=torch.bfloat16, device=pieces[0].device)
    _dev(out, "out", torch.bfloat16)
    if tuple(out.shape) != (B, 2 * Kp) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous ({B}, {2 * Kp}) bf16 matrix")
    _cabi.check(_lib().mm_concat_split(arr, n, B, out.data_ptr(), Kp, _stream()), "mm_concat_split")
    return out, K


def tower2_small_supported(pieces: Sequence[torch.Tensor], N1: int, N2: int) -> bool:
    """mm_tower2_small applies: <= 16 input columns of concat-able dtypes, N1 in {32,64,128}, N2 in {16,32,64}."""
    if not pieces or any(t.dtype not in _CONCAT_DTYPES for t in pieces):
        return False
    K = sum(1 if t.dim() == 1 else int(t.shape[1]) for t in pieces)
    return bool(_lib().mm_tower2_small_supported(int(K), int(N1), int(N2)))


def tower2_small(pieces: Sequence[torch.Tensor], w1_split: torch.Tensor, N1: int, bias1, act1, w2_split: torch.Tensor, N2: int,
                 bias2, act2, out: Optional[torch.Tensor] = None, out_split: Optional[torch.Tensor] = None):
    """act2(act1(concat(pieces) W1 + b1) W2 + b2) in one launch (mm_tower2_small).  out: (B, N2) fp32 and / or
    out_split: (B, 2*N2) bf16 [hi | lo]."""
    B = pieces[0].shape[0]
    arr, n, col = _concat_pieces(pieces, B)
    _dev(w1_split, "w1_split", torch.bfloat16), _dev(w2_split, "w2_split", torch.bfloat16)
    if tuple(w1_split.shape) != (tc_padded_n(N1), 2 * tc_padded_k(col)) or tuple(w2_split.shape) != (tc_padded_n(N2), 2 * tc_padded_k(N1)):
        raise ValueError("w1_split / w2_split must be the mm_split_weights layouts of the (K, N1) and (N1, N2) kernels")
    if out is not None:
        _dev(out, "out", torch.float32)
        if tuple(out.shape) != (B, N2) or out.stride(1) != 1:
            raise ValueError(f"out must be ({B}, {N2}) fp32")
    if out_split is not None:
        _dev(out_split, "out_split", torch.bfloat16)
        if tuple(out_split.shape) != (B, 2 * N2) or not out_split.is_contiguous():
            raise ValueError(f"out_split must be a contiguous ({B}, {2 * N2}) bf16 matrix")
    _cabi.check(
        _lib().mm_tower2_small(arr, n, B, w1_split.data_ptr(), N1, _ptr(bias1), ACTIVATIONS[act1], w2_split.data_ptr(), N2,
                               _ptr(bias2), ACTIVATIONS[act2], _ptr(out), out.stride(0) if out is not None else 0, _ptr(out_split),
                               _stream()), "mm_tower2_small")
    return out if out is not None else out_split


def l2_normalize(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _dev(x, "x", torch.float32)
    if out is None:
        out = torch.empty_like(x)
    _cabi.check(_lib().mm_l2_normalize(x.data_ptr(), x.shape[0], x.shape[1], _row_stride(x, "x"), out.data_ptr(),
                                       _row_stride(out, "out"), _stream()), "mm_l2_normalize")
    return out


def l2_normalize_backward(x: torch.Tensor, dy: torch.Tensor, dx: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Gradient of l2_normalize at its input x (mm_l2_normalize_backward); dx may be x or dy."""
    _dev(x, "x", torch.float32), _dev(dy, "dy", torch.float32)
    if dx is None:
        dx = torch.empty_like(dy)
    _dev(dx, "dx", torch.float32)
    if x.shape != dy.shape or dx.shape != dy.shape:
        raise ValueError("x, dy and dx must have the same shape")
    _cabi.check(_lib().mm_l2_normalize_backward(x.data_ptr(), dy.data_ptr(), x.shape[0], x.shape[1], _row_stride(x, "x"),
                                                _row_stride(dy, "dy"), dx.data_ptr(), _row_stride(dx, "dx"), _stream()),
                "mm_l2_normalize_backward")
    return dx


# ---------------------------------------------------------------------------------------------
# pretrained embeddings (K24): rows of a device-resident matrix by id, straight into their slot of x0
# ---------------------------------------------------------------------------------------------
def _pretrained_source(P: torch.Tensor, ids: Optional[torch.Tensor], B: int) -> tuple:
    """(rows, Dp, row stride, ids pointer, ids dtype) of a lookup of P (rows, Dp) at ids (B,); ids None: P is a dense
    (B, Dp) input read row by row."""
    _dev(P, "P", torch.float32)
    stride = _row_stride(P, "P")
    if not 1 <= P.shape[1] <= _cabi.PRETRAINED_MAX_DIM:
        raise NotImplementedError(f"pretrained vectors of width {P.shape[1]}: the kernels take 1..{_cabi.PRETRAINED_MAX_DIM}")
    if ids is None:
        if P.shape[0] != B:
            raise ValueError(f"a dense pretrained input must have {B} rows, got {tuple(P.shape)}")
        return P.shape[0], P.shape[1], stride, None, MM_I32
    _dev(ids, "ids")
    if ids.numel() != B or not ids.is_contiguous():
        raise ValueError(f"ids must be {B} contiguous ids, got {tuple(ids.shape)}")
    return P.shape[0], P.shape[1], stride, ids.data_ptr(), _idx_dtype(ids, "ids")


def pretrained_gather(P: torch.Tensor, ids: Optional[torch.Tensor], out: torch.Tensor,
                      oob: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out (B, Dp), a column slice of x0 = P[ids] (ids None: row b of the dense (B, Dp) P)  (mm_pretrained_gather)."""
    _dev(out, "out", torch.float32)
    B = out.shape[0]
    rows, Dp, ps, ip, dt = _pretrained_source(P, ids, B)
    if out.shape[1] != Dp:
        raise ValueError(f"out must be ({B}, {Dp}), got {tuple(out.shape)}")
    _cabi.check(_lib().mm_pretrained_gather(P.data_ptr(), rows, Dp, ps, ip, dt, B, out.data_ptr(), _row_stride(out, "out"),
                                            _ptr(oob), _stream()), "mm_pretrained_gather")
    return out


def pretrained_project(P: torch.Tensor, ids: Optional[torch.Tensor], W: torch.Tensor, bias: Optional[torch.Tensor],
                       out: torch.Tensor, oob: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out (B, N), a column slice of x0 or a (B, N) buffer = P[ids] W + bias, the gathered rows never written
    (mm_pretrained_project)."""
    _dev(out, "out", torch.float32), _dev(W, "W", torch.float32)
    B = out.shape[0]
    rows, Dp, ps, ip, dt = _pretrained_source(P, ids, B)
    if W.dim() != 2 or W.shape[0] != Dp or not W.is_contiguous():
        raise ValueError(f"W must be a contiguous ({Dp}, N) matrix, got {tuple(W.shape)}")
    N = W.shape[1]
    if not 1 <= N <= _cabi.PRETRAINED_MAX_OUT:
        raise NotImplementedError(f"a projection to {N} columns: the kernels take 1..{_cabi.PRETRAINED_MAX_OUT}")
    _vec(bias, N, "bias")
    if out.shape[1] != N:
        raise ValueError(f"out must be ({B}, {N}), got {tuple(out.shape)}")
    _cabi.check(_lib().mm_pretrained_project(P.data_ptr(), rows, Dp, ps, ip, dt, B, W.data_ptr(), _ptr(bias), N, out.data_ptr(),
                                             _row_stride(out, "out"), _ptr(oob), _stream()), "mm_pretrained_project")
    return out


def pretrained_backward_workspace(B: int, Dp: int, N: int, device) -> torch.Tensor:
    """The workspace of pretrained_project_backward at (B, Dp, N)."""
    nbytes = int(_lib().mm_pretrained_backward_workspace_bytes(B, Dp, N))
    return torch.empty(max(1, (nbytes + 15) // 16 * 4), dtype=torch.float32, device=device)


def pretrained_project_backward(P: torch.Tensor, ids: Optional[torch.Tensor], addends: Sequence[torch.Tensor],
                                dW: torch.Tensor, db: Optional[torch.Tensor], ypre: Optional[torch.Tensor] = None,
                                workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dW (Dp, N) = P[ids]^T g, db (N,) = sum_b g, with g the sum of the (B, N) addends (the slot's columns of the input
    gradient), taken through the l2-norm backward at the pre-norm projection ypre (B, N) when given; deterministic
    (mm_pretrained_project_backward)."""
    _dev(dW, "dW", torch.float32)
    if not addends or len(addends) > 4:
        raise ValueError("between 1 and 4 addends")
    B = addends[0].shape[0]
    rows, Dp, ps, ip, dt = _pretrained_source(P, ids, B)
    N = addends[0].shape[1]
    if tuple(dW.shape) != (Dp, N) or not dW.is_contiguous():
        raise ValueError(f"dW must be a contiguous ({Dp}, {N}) matrix")
    _vec(db, N, "db")
    for i, a in enumerate(addends):
        _dev(a, f"addends[{i}]", torch.float32)
        if tuple(a.shape) != (B, N):
            raise ValueError(f"addends[{i}] must be ({B}, {N}), got {tuple(a.shape)}")
    if ypre is not None and (tuple(_dev(ypre, "ypre", torch.float32).shape) != (B, N)):
        raise ValueError(f"ypre must be ({B}, {N})")
    if workspace is None:
        workspace = pretrained_backward_workspace(B, Dp, N, dW.device)
    ptrs = (C.c_void_p * len(addends))(*[a.data_ptr() for a in addends])
    strides = (C.c_int64 * len(addends))(*[_row_stride(a, f"addends[{i}]") for i, a in enumerate(addends)])
    _cabi.check(_lib().mm_pretrained_project_backward(P.data_ptr(), rows, Dp, ps, ip, dt, B, ptrs, strides, len(addends),
                                                      _ptr(ypre), 0 if ypre is None else _row_stride(ypre, "ypre"), N,
                                                      dW.data_ptr(), _ptr(db), workspace.data_ptr(),
                                                      workspace.numel() * 4, _stream()),
                "mm_pretrained_project_backward")
    return dW


# ---------------------------------------------------------------------------------------------
# tensor-core dense path (wgmma split-bf16)
# ---------------------------------------------------------------------------------------------
def tc_padded_k(K: int) -> int:
    return int(_lib().mm_tc_padded_k(int(K)))


def tc_padded_n(N: int) -> int:
    return int(_lib().mm_tc_padded_n(int(N)))


def split_rows(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 (M, K) -> split-bf16 (M, 2*Kp) = [hi | lo], zero padded (mm_split_rows)."""
    _dev(x, "x", torch.float32)
    M, K = x.shape
    Kp = tc_padded_k(K)
    if out is None:
        out = torch.empty((M, 2 * Kp), dtype=torch.bfloat16, device=x.device)
    _cabi.check(_lib().mm_split_rows(x.data_ptr(), M, K, _row_stride(x, "x"), out.data_ptr(), Kp, _stream()), "mm_split_rows")
    return out


def split_weights(W: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Keras kernel (K, N) fp32 -> (Np, 2*Kp) bf16 K-major split (mm_split_weights); one-time (the training step refreshes
    it in place through `out` after every optimizer update)."""
    _dev(W, "W", torch.float32)
    if W.dim() != 2 or not W.is_contiguous():
        raise ValueError("W must be a contiguous (K, N) matrix")
    K, N = W.shape
    Kp, Np = tc_padded_k(K), tc_padded_n(N)
    if out is None:
        out = torch.empty((Np, 2 * Kp), dtype=torch.bfloat16, device=W.device)
    elif tuple(out.shape) != (Np, 2 * Kp) or out.dtype != torch.bfloat16 or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous bf16 ({Np}, {2 * Kp}) matrix")
    _cabi.check(_lib().mm_split_weights(W.data_ptr(), K, N, out.data_ptr(), Kp, Np, _stream()), "mm_split_weights")
    return out


def dense_tc(a_split: torch.Tensor, K: int, w_split: torch.Tensor, N: int, bias: Optional[torch.Tensor],
             act: Optional[str], passes: int = 3, out_f32: Optional[torch.Tensor] = None,
             out_split: Optional[torch.Tensor] = None, x0: Optional[torch.Tensor] = None,
             xres: Optional[torch.Tensor] = None, dropout=None) -> None:
    """One tensor-core dense layer (mm_dense_tc); see include/mm_b200.h.  dropout = (rate, seed, step, layer): Keras
    Dropout(rate) in training after the activation (mm_dense_tc_dropout), step a one-float device counter."""
    _dev(a_split, "a_split", torch.bfloat16), _dev(w_split, "w_split", torch.bfloat16)
    if act not in ACTIVATIONS:
        raise ValueError(f"unsupported activation {act!r}")
    M = a_split.shape[0]
    Kp, Np = tc_padded_k(K), tc_padded_n(N)
    if tuple(a_split.shape) != (M, 2 * Kp) or not a_split.is_contiguous():
        raise ValueError(f"a_split must be contiguous (M, {2 * Kp}), got {tuple(a_split.shape)}")
    if tuple(w_split.shape) != (Np, 2 * Kp) or not w_split.is_contiguous():
        raise ValueError(f"w_split must be contiguous ({Np}, {2 * Kp}), got {tuple(w_split.shape)}")
    out_Kp = 0
    if out_split is not None:
        out_Kp = tc_padded_k(N)
        if tuple(out_split.shape) != (M, 2 * out_Kp) or not out_split.is_contiguous() or out_split.dtype != torch.bfloat16:
            raise ValueError(f"out_split must be contiguous bf16 (M, {2 * out_Kp})")
    xs = 0
    if x0 is not None:
        if xres is None or x0.stride(0) != xres.stride(0):
            raise ValueError("x0 and xres must both be given with equal row strides")
        xs = _row_stride(x0, "x0")
    if dropout is not None:
        rate, seed, step, layer = dropout
        if x0 is not None or not 0.0 <= float(rate) < 1.0:
            raise ValueError(f"dropout: rate in [0, 1) on a plain dense layer, got rate {rate}")
        _dev(step, "step", torch.float32)
        _cabi.check(
            _lib().mm_dense_tc_dropout(a_split.data_ptr(), M, K, Kp, w_split.data_ptr(), N, Np, _ptr(bias), ACTIVATIONS[act],
                                       passes, _ptr(out_f32), 0 if out_f32 is None else _row_stride(out_f32, "out_f32"),
                                       _ptr(out_split), out_Kp, float(rate), int(seed) & (2**64 - 1), step.data_ptr(),
                                       int(layer), _stream()),
            "mm_dense_tc_dropout")
        return
    _cabi.check(
        _lib().mm_dense_tc(a_split.data_ptr(), M, K, Kp, w_split.data_ptr(), N, Np, _ptr(bias), ACTIVATIONS[act],
                           passes, _ptr(x0), _ptr(xres), xs, _ptr(out_f32),
                           0 if out_f32 is None else _row_stride(out_f32, "out_f32"), _ptr(out_split), out_Kp, _stream()),
        "mm_dense_tc")


def catalog_score(q: torch.Tensor, e_split: torch.Tensor, n_items: int, bias: Optional[torch.Tensor] = None,
                  targets: Optional[torch.Tensor] = None, k: int = 0, want_stats: bool = True):
    """Fused query x catalog scoring (mm_catalog_score): returns (stats (B,3) or None, scores (B,k) or
    None, ids (B,k) or None).  q fp32 (B, D); e_split = split_rows(E) with E the (n_items, D) catalog."""
    _dev(q, "q", torch.float32), _dev(e_split, "e_split", torch.bfloat16)
    B, D = q.shape
    Kp = tc_padded_k(D)
    if tuple(e_split.shape) != (n_items, 2 * Kp) or not e_split.is_contiguous():
        raise ValueError(f"e_split must be contiguous ({n_items}, {2 * Kp}) = split_rows(catalog)")
    dev = q.device
    stats = torch.empty((B, 3), dtype=torch.float32, device=dev) if want_stats else None
    scores = torch.empty((B, k), dtype=torch.float32, device=dev) if k else None
    ids = torch.empty((B, k), dtype=torch.int64, device=dev) if k else None
    id_dt = MM_I64
    if targets is not None:
        targets = targets.reshape(-1).contiguous()
        id_dt = _idx_dtype(targets, "targets")
    ws = _catalog_workspace(B, n_items, k, dev)
    _cabi.check(
        _lib().mm_catalog_score(split_rows(q).data_ptr(), B, D, e_split.data_ptr(), n_items, _ptr(bias), _ptr(targets), id_dt,
                                _ptr(stats), k, _ptr(scores), _ptr(ids), ws.data_ptr(), ws.numel(), _stream()),
        "mm_catalog_score")
    return stats, scores, ids


def mlp_tc_supported(K: int, widths: Sequence[int], head: bool = False, heads: bool = False) -> bool:
    """True when mm_mlp_tc can run the tower (mm_mlp_tc_supported): 2..4 layers, every width <= 128, head only
    after <= 32 units, resident weights of layers 2..n + two layer-1 pipeline stages within shared memory.
    heads=True: with mm_mlp_tc_heads's multi-head epilogue."""
    n = len(widths)
    if n < 2 or n > 4:
        return False
    wd = (C.c_int * n)(*[int(w) for w in widths])
    return bool(_lib().mm_mlp_tc_supported(int(K), n, wd, 2 if heads else 1 if head else 0))


def _tower(who: str, a_split: torch.Tensor, K: int, w_splits: Sequence[torch.Tensor], widths: Sequence[int],
           biases: Sequence[Optional[torch.Tensor]], acts: Sequence[Optional[str]], a_bottom: Optional[torch.Tensor] = None):
    """(M, n, weight pointers, widths, bias pointers, activation codes) of a tower over the split-bf16 rows a_split
    (M, 2*Kp): layer l is w_splits[l], the mm_split_weights layout of a (k, widths[l]) kernel, biases[l] None or
    widths[l] fp32 values, acts[l] its activation.  With a_bottom (M, 128), input columns 0..63 come from a_bottom and
    a_split holds columns 64..K-1 as (M, 2*pairs_cols(K - 64)) rows (mm_mlp_tc_pairs)."""
    n = len(widths)
    if not (len(w_splits) == len(biases) == len(acts) == n):
        raise ValueError(f"{who}: w_splits / widths / biases / acts must have one entry per layer")
    _dev(a_split, "a_split", torch.bfloat16)
    cols = 2 * tc_padded_k(K)
    if a_bottom is not None:
        if K <= 64:
            raise ValueError(f"{who}: a_bottom needs K > 64")
        cols = 2 * pairs_cols(K - 64)
        _dev(a_bottom, "a_bottom", torch.bfloat16)
        if tuple(a_bottom.shape) != (a_split.shape[0], 128) or not a_bottom.is_contiguous():
            raise ValueError(f"a_bottom must be a contiguous ({a_split.shape[0]}, 128) bf16 matrix")
    if a_split.dim() != 2 or a_split.shape[1] != cols or not a_split.is_contiguous():
        raise ValueError(f"a_split must be a contiguous (M, {cols}) bf16 matrix")
    k = K
    for l in range(n):
        _dev(w_splits[l], f"w_split[{l}]", torch.bfloat16)
        if tuple(w_splits[l].shape) != (tc_padded_n(int(widths[l])), 2 * tc_padded_k(k)) or not w_splits[l].is_contiguous():
            raise ValueError(f"w_split[{l}] must be the mm_split_weights layout of a ({k}, {widths[l]}) kernel")
        if biases[l] is not None and _dev(biases[l], f"bias[{l}]", torch.float32).numel() != int(widths[l]):
            raise ValueError(f"bias[{l}] must hold {widths[l]} values")
        k = int(widths[l])
    wp = (C.c_void_p * n)(*[w.data_ptr() for w in w_splits])
    wd = (C.c_int * n)(*[int(w) for w in widths])
    bp = (C.c_void_p * n)(*[_ptr(b) for b in biases])
    ac = (C.c_int * n)(*[ACTIVATIONS[a] for a in acts])
    return a_split.shape[0], n, wp, wd, bp, ac


def mlp_tc(a_split: torch.Tensor, K: int, w_splits: Sequence[torch.Tensor], widths: Sequence[int],
           biases: Sequence[Optional[torch.Tensor]], acts: Sequence[Optional[str]], out: Optional[torch.Tensor] = None,
           head_w: Optional[torch.Tensor] = None, head_b: float = 0.0, head_act: Optional[str] = None,
           head_out: Optional[torch.Tensor] = None, out_operand: Optional[torch.Tensor] = None,
           a_bottom: Optional[torch.Tensor] = None):
    """Whole MLP tower in one launch (mm_mlp_tc): layer 1 from the split-bf16 rows `a_split`, layers 2..n on
    chip (activations stay in registers).  out: (M, widths[-1]) fp32 and/or head_out: (M, 1); out_operand:
    (M, 2*widths[-1]) bf16 split rows [hi | lo] for the interaction kernel (mm_mlp_tc_operand_out).  a_bottom: layer 1
    reads input columns 0..63 from these (M, 128) bottom rows and the rest from the pairs rows `a_split`
    (mm_mlp_tc_pairs)."""
    M, n, wp, wd, bp, ac = _tower("mlp_tc", a_split, K, w_splits, widths, biases, acts, a_bottom)
    if out is not None:
        _dev(out, "out", torch.float32)
        if out.dim() != 2 or tuple(out.shape) != (M, int(widths[-1])) or out.stride(1) != 1:
            raise ValueError(f"out must be ({M}, {widths[-1]}) fp32 with unit column stride")
    if (head_w is None) != (head_out is None):
        raise ValueError("head_w and head_out go together")
    if head_w is not None:
        _dev(head_w, "head_w", torch.float32), _dev(head_out, "head_out", torch.float32)
        if head_w.numel() != int(widths[-1]) or not head_w.is_contiguous() or head_out.numel() != M or not head_out.is_contiguous():
            raise ValueError("head_w must hold widths[-1] weights and head_out M contiguous values")
    if a_bottom is not None:
        if out_operand is not None:
            raise ValueError("a_bottom and out_operand exclude each other")
        _cabi.check(
            _lib().mm_mlp_tc_pairs(a_bottom.data_ptr(), a_split.data_ptr(), M, K, n, wp, wd, bp, ac, _ptr(out),
                                   out.stride(0) if out is not None else 0, _ptr(head_w), float(head_b), ACTIVATIONS[head_act],
                                   _ptr(head_out), 0, None, None, _stream()),
            "mm_mlp_tc_pairs")
        return out if out is not None else head_out
    if out_operand is not None:
        if head_w is not None:
            raise ValueError("out_operand and the fused head exclude each other")
        _dev(out_operand, "out_operand", torch.bfloat16)
        if tuple(out_operand.shape) != (M, 2 * int(widths[-1])) or not out_operand.is_contiguous():
            raise ValueError(f"out_operand must be a contiguous ({M}, {2 * int(widths[-1])}) bf16 buffer")
        _cabi.check(
            _lib().mm_mlp_tc_operand_out(a_split.data_ptr(), M, K, n, wp, wd, bp, ac, _ptr(out),
                                         out.stride(0) if out is not None else 0, out_operand.data_ptr(), _stream()),
            "mm_mlp_tc_operand_out")
        return
    _cabi.check(
        _lib().mm_mlp_tc(a_split.data_ptr(), M, K, n, wp, wd, bp, ac, _ptr(out), out.stride(0) if out is not None else 0,
                         _ptr(head_w), float(head_b), ACTIVATIONS[head_act], _ptr(head_out), _stream()),
        "mm_mlp_tc")
    return out if out is not None else head_out


def mlp_tc_heads(a_split: torch.Tensor, K: int, w_splits: Sequence[torch.Tensor], widths: Sequence[int],
                 biases: Sequence[Optional[torch.Tensor]], acts: Sequence[Optional[str]], heads_w: torch.Tensor,
                 heads_b: Optional[torch.Tensor], heads_act: Sequence[Optional[str]], out: torch.Tensor,
                 a_bottom: Optional[torch.Tensor] = None) -> torch.Tensor:
    """mm_mlp_tc_heads: the whole tower with H <= 8 fused output heads; out (H, M) with
    out[h] = heads_act[h](tower(x) @ heads_w[:, h] + heads_b[h]).  heads_w (widths[-1], H) Keras layout, heads_b (H,) on the
    device (read by the kernel, not copied to the host).  a_bottom: as mlp_tc (mm_mlp_tc_pairs)."""
    M, n, wp, wd, bp, ac = _tower("mlp_tc_heads", a_split, K, w_splits, widths, biases, acts, a_bottom)
    _dev(heads_w, "heads_w", torch.float32), _dev(out, "out", torch.float32)
    H = len(heads_act)
    if tuple(heads_w.shape) != (int(widths[-1]), H) or not heads_w.is_contiguous():
        raise ValueError(f"heads_w must be a contiguous ({widths[-1]}, {H}) matrix")
    _vec(heads_b, H, "heads_b")
    if tuple(out.shape) != (H, M) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous ({H}, {M}) matrix")
    ha = (C.c_int * H)(*[ACTIVATIONS[a] for a in heads_act])
    if a_bottom is not None:
        _cabi.check(_lib().mm_mlp_tc_pairs(a_bottom.data_ptr(), a_split.data_ptr(), M, K, n, wp, wd, bp, ac, None, 0,
                                           heads_w.data_ptr(), 0.0, 0, out.data_ptr(), H, _ptr(heads_b), ha, _stream()),
                    "mm_mlp_tc_pairs")
        return out
    _cabi.check(_lib().mm_mlp_tc_heads(a_split.data_ptr(), M, K, n, wp, wd, bp, ac, H, heads_w.data_ptr(), _ptr(heads_b), ha,
                                       out.data_ptr(), _stream()), "mm_mlp_tc_heads")
    return out


def dense_tc_head(a_split: torch.Tensor, K: int, w_split: torch.Tensor, N: int, bias: Optional[torch.Tensor],
                  act: Optional[str], head_w: torch.Tensor, head_b: float, head_act: Optional[str],
                  out: torch.Tensor, passes: int = 3) -> torch.Tensor:
    """Tensor-core dense layer (N <= 32) with the following Dense(N -> 1) fused into its epilogue
    (mm_dense_tc_head): out (M, 1) = head_act(act(x W + b) @ head_w + head_b)."""
    _dev(a_split, "a_split", torch.bfloat16), _dev(w_split, "w_split", torch.bfloat16), _dev(out, "out", torch.float32)
    _dev(head_w, "head_w", torch.float32)
    M = a_split.shape[0]
    if head_w.numel() != N or not head_w.is_contiguous() or out.numel() != M or not out.is_contiguous():
        raise ValueError("head_w must hold N weights and out M contiguous values")
    _cabi.check(
        _lib().mm_dense_tc_head(a_split.data_ptr(), M, K, tc_padded_k(K), w_split.data_ptr(), N, tc_padded_n(N), _ptr(bias),
                                ACTIVATIONS[act], passes, head_w.data_ptr(), float(head_b), ACTIVATIONS[head_act],
                                out.data_ptr(), _stream()),
        "mm_dense_tc_head")
    return out


# ---- training step (include/mm_b200.h K14) -----------------------------------------------------------------------
_TARGET_DTYPES = {torch.int32: MM_I32, torch.int64: MM_I64, torch.float32: _cabi.MM_F32, torch.float64: _cabi.MM_F64}
_SAMPLE_WEIGHT = "be ({n},) contiguous float32"  # _vec's error for a sample-weight column


def _target(t: torch.Tensor, M: int, name: str) -> int:
    """Dtype code of a target column: M contiguous int32 / int64 / float32 / float64 values."""
    _dev(t, name)
    if t.numel() != M or not t.is_contiguous() or t.dtype not in _TARGET_DTYPES:
        raise ValueError(f"{name} must be {M} contiguous int32 / int64 / float32 / float64 values")
    return _TARGET_DTYPES[t.dtype]


def heads_fwd_bwd(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], losses: Sequence[str],
                  targets: Optional[Sequence[torch.Tensor]], out: torch.Tensor, loss: Optional[torch.Tensor] = None,
                  dx: Optional[torch.Tensor] = None, dw: Optional[torch.Tensor] = None, db: Optional[torch.Tensor] = None,
                  loss_weights: Optional[Sequence[float]] = None, mask_relu: bool = True, sample_weight=None) -> torch.Tensor:
    """H <= 8 output heads Dense(K -> 1) on x (M, K), forward and backward in one pass (mm_heads_fwd_bwd).  w (K, H), bias
    (H,); losses[h] in {"binary_crossentropy", "mse"}.  targets None: forward only, out (H, M) = the activated predictions
    (sigmoid / linear).  Otherwise out (H, M) = the logits, loss (1 + H) += [sum_h lambda_h loss_h, loss_0, ...], dw (K, H)
    and db (H,) are ACCUMULATED (each nullable), dx (M, K) is written.  sample_weight: one (M,) fp32 tensor shared by every head, or a list
    of H (entries may be None)."""
    _dev(x, "x", torch.float32), _dev(w, "w", torch.float32), _dev(out, "out", torch.float32)
    M, K = x.shape
    H = len(losses)
    if tuple(w.shape) != (K, H) or not w.is_contiguous():
        raise ValueError(f"w must be a contiguous ({K}, {H}) matrix")
    _vec(bias, H, "bias")
    if tuple(out.shape) != (H, M) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous ({H}, {M}) matrix")
    if any(l not in _cabi.LOSS_KINDS for l in losses):
        raise ValueError(f"losses must be among {sorted(_cabi.LOSS_KINDS)}, got {list(losses)}")
    kinds = (C.c_int * H)(*[_cabi.LOSS_KINDS[l] for l in losses])
    tp = dt = sp = lw = None
    if targets is not None:
        if len(targets) != H:
            raise ValueError(f"one target tensor per head: {H} expected, got {len(targets)}")
        dt = (C.c_int * H)(*[_target(t, M, f"targets[{h}]") for h, t in enumerate(targets)])
        if loss is None:
            raise ValueError("training needs loss")
        _dev(loss, "loss", torch.float32)
        if loss.numel() != 1 + H or not loss.is_contiguous():
            raise ValueError(f"loss must hold 1 + H = {1 + H} contiguous values")
        if dw is not None and (_dev(dw, "dw", torch.float32).shape != (K, H) or not dw.is_contiguous()):
            raise ValueError(f"dw must be a contiguous ({K}, {H}) matrix")
        _vec(db, H, "db")
        sws = list(sample_weight) if isinstance(sample_weight, (list, tuple)) else [sample_weight] * H
        if len(sws) != H:
            raise ValueError(f"one sample-weight tensor per head: {H} expected, got {len(sws)}")
        for h, s in enumerate(sws):
            _vec(s, M, f"sample_weight[{h}]", _SAMPLE_WEIGHT)
        lws = [1.0] * H if loss_weights is None else [float(v) for v in loss_weights]
        if len(lws) != H:
            raise ValueError(f"one loss weight per head: {H} expected, got {len(lws)}")
        tp = (C.c_void_p * H)(*[t.data_ptr() for t in targets])
        sp = (C.c_void_p * H)(*[_ptr(s) for s in sws])
        lw = (C.c_float * H)(*lws)
    _cabi.check(
        _lib().mm_heads_fwd_bwd(x.data_ptr(), M, K, _row_stride(x, "x"), H, w.data_ptr(), _ptr(bias), kinds, lw, tp, dt, sp,
                                out.data_ptr(), _ptr(loss) if targets is not None else None,
                                _ptr(dx) if targets is not None else None,
                                0 if dx is None else _row_stride(_dev(dx, "dx", torch.float32), "dx"), 1 if mask_relu else 0,
                                _ptr(dw) if targets is not None else None, _ptr(db) if targets is not None else None, _stream()),
        "mm_heads_fwd_bwd")
    return out


MMOE_MAX_EXPERTS, MMOE_MAX_UNITS, MMOE_MAX_TASKS = 16, 256, 8  # mm_mmoe_heads_fwd_bwd


def mmoe_heads_fwd_bwd(x: torch.Tensor, E: int, gate_logits: Sequence[torch.Tensor], temperature: float, w: torch.Tensor,
                       bias: Optional[torch.Tensor], losses: Sequence[str], targets: Optional[Sequence[torch.Tensor]],
                       out: torch.Tensor, loss: Optional[torch.Tensor] = None, dx: Optional[torch.Tensor] = None,
                       d_gate_logits: Optional[Sequence[torch.Tensor]] = None, dw: Optional[torch.Tensor] = None,
                       db: Optional[torch.Tensor] = None, loss_weights: Optional[Sequence[float]] = None, mask_relu: bool = True,
                       sample_weight=None) -> torch.Tensor:
    """H <= 8 tasks, each the soft-max gate of its (M, E) logits gate_logits[t] over the E experts' outputs x (M, E U)
    followed by its Dense(U -> 1), forward and backward in one pass (mm_mmoe_heads_fwd_bwd).  w (U, H), bias (H,), losses,
    targets, out, loss, dw, db, loss_weights and sample_weight as heads_fwd_bwd.  Training writes dx (M, E U) and
    d_gate_logits[t] (M, E)."""
    _dev(x, "x", torch.float32), _dev(w, "w", torch.float32), _dev(out, "out", torch.float32)
    M, EU = x.shape
    H = len(losses)
    if not (1 <= E <= MMOE_MAX_EXPERTS) or EU % E:
        raise ValueError(f"x must hold E = {E} experts (1..{MMOE_MAX_EXPERTS}) of equal width, got {EU} columns")
    U = EU // E
    if not (1 <= U <= MMOE_MAX_UNITS) or not (1 <= H <= MMOE_MAX_TASKS):
        raise ValueError(f"expert width {U} must be in 1..{MMOE_MAX_UNITS} and the task count {H} in 1..{MMOE_MAX_TASKS}")
    if not temperature > 0:
        raise ValueError(f"the gate temperature must be > 0, got {temperature}")
    if tuple(w.shape) != (U, H) or not w.is_contiguous():
        raise ValueError(f"w must be a contiguous ({U}, {H}) matrix")
    _vec(bias, H, "bias")
    if tuple(out.shape) != (H, M) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous ({H}, {M}) matrix")
    if any(l not in _cabi.LOSS_KINDS for l in losses):
        raise ValueError(f"losses must be among {sorted(_cabi.LOSS_KINDS)}, got {list(losses)}")

    def gates(ts, name):
        if len(ts) != H:
            raise ValueError(f"{name}: one (M, E) matrix per task: {H} expected, got {len(ts)}")
        for t, g in enumerate(ts):
            if _dev(g, f"{name}[{t}]", torch.float32).shape != (M, E):
                raise ValueError(f"{name}[{t}] must be ({M}, {E}), got {tuple(g.shape)}")
        return ((C.c_void_p * H)(*[g.data_ptr() for g in ts]),
                (C.c_int64 * H)(*[_row_stride(g, f"{name}[{t}]") for t, g in enumerate(ts)]))

    gp, gs = gates(gate_logits, "gate_logits")
    kinds = (C.c_int * H)(*[_cabi.LOSS_KINDS[l] for l in losses])
    tp = dt = sp = lw = dgp = dgs = None
    dxs = 0
    if targets is not None:
        if len(targets) != H:
            raise ValueError(f"one target tensor per task: {H} expected, got {len(targets)}")
        dt = (C.c_int * H)(*[_target(t, M, f"targets[{h}]") for h, t in enumerate(targets)])
        if loss is None or dx is None or d_gate_logits is None:
            raise ValueError("training needs loss, dx and d_gate_logits")
        _vec(loss, 1 + H, "loss")
        if _dev(dx, "dx", torch.float32).shape != (M, EU):
            raise ValueError(f"dx must be ({M}, {EU})")
        dxs = _row_stride(dx, "dx")
        dgp, dgs = gates(d_gate_logits, "d_gate_logits")
        if dw is not None and (_dev(dw, "dw", torch.float32).shape != (U, H) or not dw.is_contiguous()):
            raise ValueError(f"dw must be a contiguous ({U}, {H}) matrix")
        _vec(db, H, "db")
        sws = list(sample_weight) if isinstance(sample_weight, (list, tuple)) else [sample_weight] * H
        if len(sws) != H:
            raise ValueError(f"one sample-weight tensor per task: {H} expected, got {len(sws)}")
        for h, s in enumerate(sws):
            _vec(s, M, f"sample_weight[{h}]", _SAMPLE_WEIGHT)
        lws = [1.0] * H if loss_weights is None else [float(v) for v in loss_weights]
        if len(lws) != H:
            raise ValueError(f"one loss weight per task: {H} expected, got {len(lws)}")
        tp = (C.c_void_p * H)(*[t.data_ptr() for t in targets])
        sp = (C.c_void_p * H)(*[_ptr(s) for s in sws])
        lw = (C.c_float * H)(*lws)
    train = targets is not None
    _cabi.check(
        _lib().mm_mmoe_heads_fwd_bwd(x.data_ptr(), M, E, U, _row_stride(x, "x"), gp, gs, H, float(temperature), w.data_ptr(),
                                     _ptr(bias), kinds, lw, tp, dt, sp, out.data_ptr(), _ptr(loss) if train else None,
                                     _ptr(dx) if train else None, dxs, 1 if mask_relu else 0, dgp, dgs,
                                     _ptr(dw) if train else None, _ptr(db) if train else None, _stream()),
        "mm_mmoe_heads_fwd_bwd")
    return out


def _ptr_array(ts: Sequence[torch.Tensor], name: str, H: int, shape: tuple):
    """(device pointers, row strides) of H fp32 matrices of the given shape, as the ctypes arrays the K19 calls take."""
    if len(ts) != H:
        raise ValueError(f"{name}: one matrix per task: {H} expected, got {len(ts)}")
    for t, g in enumerate(ts):
        if tuple(_dev(g, f"{name}[{t}]", torch.float32).shape) != shape:
            raise ValueError(f"{name}[{t}] must be {shape}, got {tuple(g.shape)}")
    return ((C.c_void_p * H)(*[g.data_ptr() for g in ts]),
            (C.c_int64 * H)(*[_row_stride(g, f"{name}[{t}]") for t, g in enumerate(ts)]))


def _mixture_shape(x: torch.Tensor, E: int, temperature: float):
    _dev(x, "x", torch.float32)
    M, EU = x.shape
    if not (1 <= E <= MMOE_MAX_EXPERTS) or EU % E or not (1 <= EU // E <= MMOE_MAX_UNITS):
        raise ValueError(f"x must hold E = {E} experts (1..{MMOE_MAX_EXPERTS}) of 1..{MMOE_MAX_UNITS} units, got {EU} columns")
    if not temperature > 0:
        raise ValueError(f"the gate temperature must be > 0, got {temperature}")
    return M, EU // E


def mmoe_mix_fwd(x: torch.Tensor, E: int, gate_logits: Sequence[torch.Tensor], temperature: float, p: torch.Tensor,
                 m: torch.Tensor, m_split: Optional[torch.Tensor] = None) -> None:
    """The gates and the mixture alone (mm_mmoe_mix_fwd): p (M, H E) = the gate weights, m (H, M, U) the mixtures, m_split
    (H, M, 2 Kp) their split-bf16 operands (optional)."""
    M, U = _mixture_shape(x, E, temperature)
    H = len(gate_logits)
    if not 1 <= H <= MMOE_MAX_TASKS:
        raise ValueError(f"1..{MMOE_MAX_TASKS} tasks, got {H}")
    gp, gs = _ptr_array(gate_logits, "gate_logits", H, (M, E))
    if tuple(_dev(p, "p", torch.float32).shape) != (M, H * E) or not p.is_contiguous():
        raise ValueError(f"p must be a contiguous ({M}, {H * E}) matrix")
    if tuple(_dev(m, "m", torch.float32).shape) != (H, M, U) or not m.is_contiguous():
        raise ValueError(f"m must be a contiguous ({H}, {M}, {U}) tensor")
    Kp = tc_padded_k(U)
    if m_split is not None and (tuple(_dev(m_split, "m_split", torch.bfloat16).shape) != (H, M, 2 * Kp) or not m_split.is_contiguous()):
        raise ValueError(f"m_split must be a contiguous bf16 ({H}, {M}, {2 * Kp}) tensor")
    _cabi.check(_lib().mm_mmoe_mix_fwd(x.data_ptr(), M, E, U, _row_stride(x, "x"), gp, gs, H, float(temperature), p.data_ptr(),
                                       m.data_ptr(), _ptr(m_split), Kp, _stream()), "mm_mmoe_mix_fwd")


def mmoe_mix_bwd(x: torch.Tensor, E: int, p: torch.Tensor, temperature: float, dm: torch.Tensor, dx: torch.Tensor,
                 d_gate_logits: Sequence[torch.Tensor], mask_relu: bool = True) -> None:
    """Backward of mmoe_mix_fwd (mm_mmoe_mix_bwd): dm (H, M, U) -> dx (M, E U) and d_gate_logits[t] (M, E)."""
    M, U = _mixture_shape(x, E, temperature)
    H = len(d_gate_logits)
    if not 1 <= H <= MMOE_MAX_TASKS:
        raise ValueError(f"1..{MMOE_MAX_TASKS} tasks, got {H}")
    dgp, dgs = _ptr_array(d_gate_logits, "d_gate_logits", H, (M, E))
    if tuple(_dev(p, "p", torch.float32).shape) != (M, H * E) or not p.is_contiguous():
        raise ValueError(f"p must be a contiguous ({M}, {H * E}) matrix")
    if tuple(_dev(dm, "dm", torch.float32).shape) != (H, M, U) or not dm.is_contiguous():
        raise ValueError(f"dm must be a contiguous ({H}, {M}, {U}) tensor")
    if tuple(_dev(dx, "dx", torch.float32).shape) != (M, E * U):
        raise ValueError(f"dx must be ({M}, {E * U})")
    _cabi.check(_lib().mm_mmoe_mix_bwd(x.data_ptr(), M, E, U, _row_stride(x, "x"), p.data_ptr(), H, float(temperature), dm.data_ptr(),
                                       dx.data_ptr(), _row_stride(dx, "dx"), 1 if mask_relu else 0, dgp, dgs, _stream()),
                "mm_mmoe_mix_bwd")


def mmoe_task_heads_fwd_bwd(xs: Sequence[torch.Tensor], w: torch.Tensor, bias: Optional[torch.Tensor], losses: Sequence[str],
                            targets: Optional[Sequence[torch.Tensor]], out: torch.Tensor, loss: Optional[torch.Tensor] = None,
                            dxs: Optional[Sequence[torch.Tensor]] = None, dw: Optional[torch.Tensor] = None,
                            db: Optional[torch.Tensor] = None, loss_weights: Optional[Sequence[float]] = None,
                            mask_relu: bool = True, sample_weight=None) -> torch.Tensor:
    """H output heads where head t reads its own input xs[t] (M, K) (mm_mmoe_task_heads_fwd_bwd); w (K, H), bias, losses,
    targets, out, loss, dw, db, loss_weights and sample_weight as heads_fwd_bwd; training writes dxs[t] (M, K)."""
    H = len(losses)
    if not 1 <= H <= MMOE_MAX_TASKS or not xs:
        raise ValueError(f"1..{MMOE_MAX_TASKS} heads, got {H}")
    M, K = xs[0].shape
    if not 1 <= K <= MMOE_MAX_UNITS:
        raise ValueError(f"the heads read at most {MMOE_MAX_UNITS} inputs, got {K}")
    xp, xst = _ptr_array(xs, "xs", H, (M, K))
    if tuple(_dev(w, "w", torch.float32).shape) != (K, H) or not w.is_contiguous():
        raise ValueError(f"w must be a contiguous ({K}, {H}) matrix")
    _vec(bias, H, "bias")
    if tuple(_dev(out, "out", torch.float32).shape) != (H, M) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous ({H}, {M}) matrix")
    if any(l not in _cabi.LOSS_KINDS for l in losses):
        raise ValueError(f"losses must be among {sorted(_cabi.LOSS_KINDS)}, got {list(losses)}")
    kinds = (C.c_int * H)(*[_cabi.LOSS_KINDS[l] for l in losses])
    tp = dt = sp = lw = dxp = dxst = None
    train = targets is not None
    if train:
        if len(targets) != H:
            raise ValueError(f"one target tensor per head: {H} expected, got {len(targets)}")
        dt = (C.c_int * H)(*[_target(t, M, f"targets[{h}]") for h, t in enumerate(targets)])
        if loss is None or dxs is None:
            raise ValueError("training needs loss and dxs")
        _vec(loss, 1 + H, "loss")
        dxp, dxst = _ptr_array(dxs, "dxs", H, (M, K))
        if dw is not None and (_dev(dw, "dw", torch.float32).shape != (K, H) or not dw.is_contiguous()):
            raise ValueError(f"dw must be a contiguous ({K}, {H}) matrix")
        _vec(db, H, "db")
        sws = list(sample_weight) if isinstance(sample_weight, (list, tuple)) else [sample_weight] * H
        if len(sws) != H:
            raise ValueError(f"one sample-weight tensor per head: {H} expected, got {len(sws)}")
        for h, s_ in enumerate(sws):
            _vec(s_, M, f"sample_weight[{h}]", _SAMPLE_WEIGHT)
        lws = [1.0] * H if loss_weights is None else [float(v) for v in loss_weights]
        if len(lws) != H:
            raise ValueError(f"one loss weight per head: {H} expected, got {len(lws)}")
        tp = (C.c_void_p * H)(*[t.data_ptr() for t in targets])
        sp = (C.c_void_p * H)(*[_ptr(s_) for s_ in sws])
        lw = (C.c_float * H)(*lws)
    _cabi.check(_lib().mm_mmoe_task_heads_fwd_bwd(xp, xst, M, K, H, w.data_ptr(), _ptr(bias), kinds, lw, tp, dt, sp, out.data_ptr(),
                                                  _ptr(loss) if train else None, dxp, dxst, 1 if mask_relu else 0,
                                                  _ptr(dw) if train else None, _ptr(db) if train else None, _stream()),
                "mm_mmoe_task_heads_fwd_bwd")
    return out


NCF_MAX_WIDTH, NCF_MAX_UNITS, NCF_MAX_HEADS = 128, 256, 8  # mm_ncf_head_fwd_bwd


def ncf_head_fwd_bwd(table_u: torch.Tensor, ids_u: torch.Tensor, table_i: torch.Tensor, ids_i: torch.Tensor, h: torch.Tensor,
                     w: torch.Tensor, bias: Optional[torch.Tensor], losses: Sequence[str], targets: Optional[Sequence[torch.Tensor]],
                     out: torch.Tensor, loss: Optional[torch.Tensor] = None, reg: Optional[torch.Tensor] = None, l2: float = 0.0,
                     du: Optional[torch.Tensor] = None, di: Optional[torch.Tensor] = None, dh: Optional[torch.Tensor] = None,
                     dw: Optional[torch.Tensor] = None, db: Optional[torch.Tensor] = None,
                     loss_weights: Optional[Sequence[float]] = None, relu_h: bool = True, sample_weight=None,
                     x_reg: Optional[torch.Tensor] = None, oob: Optional[torch.Tensor] = None) -> torch.Tensor:
    """NCF's GMF branch and output heads in one pass (mm_ncf_head_fwd_bwd): u = table_u[ids_u], i = table_i[ids_i] (D wide,
    ids of any width index_bytes_of accepts), z_t = [u * i | h] . w[:, t] + bias[t] with h (M, U) and w (D + U, H).
    losses, targets, out, loss, dw, db, loss_weights and sample_weight as heads_fwd_bwd.  Training writes du, di (M, D)
    contiguous (the two tables' IndexedSlices values, with 2 l2 u / 2 l2 i added) and dh (M, U) (relu-masked from h when
    relu_h).  reg (1 value, nullable) accumulates l2 (sum |u|^2 + |i|^2 + |x_reg|^2); training adds it to loss[0] too."""
    for n, t in (("table_u", table_u), ("table_i", table_i)):
        if _dev(t, n, torch.float32).dim() != 2 or not t.is_contiguous():
            raise ValueError(f"{n} must be a contiguous (rows, D) matrix")
    D = table_u.shape[1]
    if table_i.shape[1] != D:
        raise ValueError(f"table_u and table_i must have the same width, got {D} and {table_i.shape[1]}")
    _dev(h, "h", torch.float32), _dev(w, "w", torch.float32), _dev(out, "out", torch.float32)
    if h.dim() != 2:
        raise ValueError(f"h must be (M, U), got {tuple(h.shape)}")
    M, U = h.shape
    H = len(losses)
    if not (1 <= D <= NCF_MAX_WIDTH and 1 <= U <= NCF_MAX_UNITS and 1 <= H <= NCF_MAX_HEADS):
        raise ValueError(f"D = {D}, U = {U} and H = {H} must be in 1..{NCF_MAX_WIDTH}, 1..{NCF_MAX_UNITS} and 1..{NCF_MAX_HEADS}")
    wu = _id_column(ids_u, M, "ids_u")
    wi = _id_column(ids_i, M, "ids_i")
    if tuple(w.shape) != (D + U, H) or not w.is_contiguous():
        raise ValueError(f"w must be a contiguous ({D + U}, {H}) matrix")
    _vec(bias, H, "bias")
    if tuple(out.shape) != (H, M) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous ({H}, {M}) matrix")
    if any(l not in _cabi.LOSS_KINDS for l in losses):
        raise ValueError(f"losses must be among {sorted(_cabi.LOSS_KINDS)}, got {list(losses)}")
    if not (0.0 <= float(l2) < float("inf")):
        raise ValueError(f"l2 must be finite and >= 0, got {l2}")
    _vec(reg, 1, "reg")
    if x_reg is not None:
        if reg is None:
            raise ValueError("x_reg needs reg")
        if _dev(x_reg, "x_reg", torch.float32).dim() != 2 or x_reg.shape[0] != M or x_reg.shape[1] < 1:
            raise ValueError(f"x_reg must be ({M}, n) with n >= 1, got {tuple(x_reg.shape)}")
    if oob is not None and (_dev(oob, "oob", torch.int32).numel() < 1 or not oob.is_contiguous()):
        raise ValueError("oob must be an int32 counter")
    kinds = (C.c_int * H)(*[_cabi.LOSS_KINDS[l] for l in losses])
    tp = dt = sp = lw = None
    train = targets is not None
    dhs = 0
    if train:
        if len(targets) != H:
            raise ValueError(f"one target tensor per head: {H} expected, got {len(targets)}")
        dt = (C.c_int * H)(*[_target(t, M, f"targets[{h_}]") for h_, t in enumerate(targets)])
        if loss is None or du is None or di is None or dh is None or dw is None:
            raise ValueError("training needs loss, du, di, dh and dw")
        _vec(loss, 1 + H, "loss")
        for n, g in (("du", du), ("di", di)):
            if tuple(_dev(g, n, torch.float32).shape) != (M, D) or not g.is_contiguous():
                raise ValueError(f"{n} must be a contiguous ({M}, {D}) matrix")
        if tuple(_dev(dh, "dh", torch.float32).shape) != (M, U):
            raise ValueError(f"dh must be ({M}, {U})")
        dhs = _row_stride(dh, "dh")
        if tuple(_dev(dw, "dw", torch.float32).shape) != (D + U, H) or not dw.is_contiguous():
            raise ValueError(f"dw must be a contiguous ({D + U}, {H}) matrix")
        _vec(db, H, "db")
        sws = list(sample_weight) if isinstance(sample_weight, (list, tuple)) else [sample_weight] * H
        if len(sws) != H:
            raise ValueError(f"one sample-weight tensor per head: {H} expected, got {len(sws)}")
        for h_, s_ in enumerate(sws):
            _vec(s_, M, f"sample_weight[{h_}]", _SAMPLE_WEIGHT)
        lws = [1.0] * H if loss_weights is None else [float(v) for v in loss_weights]
        if len(lws) != H:
            raise ValueError(f"one loss weight per head: {H} expected, got {len(lws)}")
        tp = (C.c_void_p * H)(*[t.data_ptr() for t in targets])
        sp = (C.c_void_p * H)(*[_ptr(s_) for s_ in sws])
        lw = (C.c_float * H)(*lws)
    _cabi.check(_lib().mm_ncf_head_fwd_bwd(
        table_u.data_ptr(), table_u.shape[0], ids_u.data_ptr(), wu, table_i.data_ptr(), table_i.shape[0], ids_i.data_ptr(), wi, D,
        h.data_ptr(), _row_stride(h, "h"), U, 1 if relu_h else 0, M, H, w.data_ptr(), _ptr(bias), kinds, lw, tp, dt, sp, float(l2),
        _ptr(x_reg), 0 if x_reg is None else _row_stride(x_reg, "x_reg"), 0 if x_reg is None else x_reg.shape[1], out.data_ptr(),
        _ptr(loss) if train else None, _ptr(reg), _ptr(du) if train else None, _ptr(di) if train else None,
        _ptr(dh) if train else None, dhs, _ptr(dw) if train else None, _ptr(db) if train else None, _ptr(oob), _stream()),
        "mm_ncf_head_fwd_bwd")
    return out


def _wgrad_n(M: int, K: int, dz: torch.Tensor, dw: torch.Tensor, db: Optional[torch.Tensor]) -> int:
    """N of the gradients of a Dense layer with M rows of K inputs: dz (M, N), dw a contiguous (K, N) matrix, db (N,) or None."""
    _dev(dz, "dz", torch.float32), _dev(dw, "dw", torch.float32)
    N = dz.shape[1]
    if dz.shape[0] != M or tuple(dw.shape) != (K, N) or not dw.is_contiguous():
        raise ValueError(f"dz must be ({M}, N) and dw a contiguous ({K}, {N}) matrix")
    _vec(db, N, "db")
    return N


def dense_wgrad(x: torch.Tensor, dz: torch.Tensor, dw: torch.Tensor, db: Optional[torch.Tensor]) -> None:
    """dw (K, N) += x^T dz;  db (N,) += column sums of dz  (mm_dense_wgrad; accumulated)."""
    _dev(x, "x", torch.float32)
    M, K = x.shape
    N = _wgrad_n(M, K, dz, dw, db)
    _cabi.check(_lib().mm_dense_wgrad(x.data_ptr(), M, K, _row_stride(x, "x"), dz.data_ptr(), N, _row_stride(dz, "dz"), dw.data_ptr(),
                                      _ptr(db), _stream()), "mm_dense_wgrad")


def dense_wgrad_split(x_split: torch.Tensor, K: int, dz: torch.Tensor, dw: torch.Tensor, db: Optional[torch.Tensor]) -> None:
    """dense_wgrad with x given as the split-bf16 operand (M, 2*Kp) the forward layer consumed (mm_dense_wgrad_split)."""
    _dev(x_split, "x_split", torch.bfloat16)
    M = x_split.shape[0]
    Kp = tc_padded_k(K)
    if tuple(x_split.shape) != (M, 2 * Kp) or not x_split.is_contiguous():
        raise ValueError(f"x_split must be a contiguous bf16 ({M}, {2 * Kp}) matrix")
    N = _wgrad_n(M, K, dz, dw, db)
    _cabi.check(_lib().mm_dense_wgrad_split(x_split.data_ptr(), M, K, Kp, dz.data_ptr(), N, _row_stride(dz, "dz"), dw.data_ptr(), _ptr(db),
                                            _stream()), "mm_dense_wgrad_split")


def dense_dgrad(dz: torch.Tensor, W: torch.Tensor, dx: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dx (M, K) = dz (M, N) @ W^T, W the Keras kernel (K, N), zeroed where mask <= 0 (mm_dense_dgrad; N <= 128)."""
    _dev(dz, "dz", torch.float32), _dev(W, "W", torch.float32), _dev(dx, "dx", torch.float32)
    M, N = dz.shape
    if W.dim() != 2 or W.shape[1] != N or not W.is_contiguous():
        raise ValueError(f"W must be a contiguous (K, {N}) matrix")
    K = W.shape[0]
    if dx.shape[0] != M or dx.shape[1] != K:
        raise ValueError(f"dx must be ({M}, {K})")
    if mask is not None and (_dev(mask, "mask", torch.float32).shape[0] != M or mask.shape[1] != K):
        raise ValueError(f"mask must be ({M}, {K})")
    _cabi.check(_lib().mm_dense_dgrad(dz.data_ptr(), M, N, _row_stride(dz, "dz"), W.data_ptr(), K, _ptr(mask),
                                      0 if mask is None else _row_stride(mask, "mask"), dx.data_ptr(), _row_stride(dx, "dx"),
                                      _stream()), "mm_dense_dgrad")
    return dx


def relu_mask(x: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """x = mask > 0 ? x : 0, in place (mm_relu_mask)."""
    _dev(x, "x", torch.float32), _dev(mask, "mask", torch.float32)
    if x.shape != mask.shape:
        raise ValueError("x and mask must have the same shape")
    _cabi.check(_lib().mm_relu_mask(x.data_ptr(), x.shape[0], x.shape[1], _row_stride(x, "x"), mask.data_ptr(), _row_stride(mask, "mask"),
                                    _stream()), "mm_relu_mask")
    return x


def dlrm_interact_backward(weights, indices, slots, rows, D: int, bottom: Optional[torch.Tensor], bottom_slot: int,
                           dA: torch.Tensor, grad_rows, d_bottom: Optional[torch.Tensor], mask_bottom: bool = True,
                           operand_rows: bool = False) -> None:
    """Backward of dlrm_lookup_interact (replicated tables): grad_rows[t] (B, D) <- IndexedSlices values of table t,
    d_bottom (B, D) <- gradient of the bottom vector (mm_dlrm_interact_backward).  operand_rows=True (D = 64): `weights`
    and `bottom` are bf16 split rows (rows, 2*D) = [hi | lo], as in dlrm_lookup_interact."""
    _dev(dA, "dA", torch.float32)
    B = dA.shape[0]
    n = len(weights)
    if not (len(indices) == n and len(slots) == n and len(rows) == n and len(grad_rows) == n):
        raise ValueError("weights / indices / slots / rows / grad_rows length mismatch")
    gp = (C.c_void_p * n)()
    gstride = None
    wdt, wcols = (torch.bfloat16, 2 * D) if operand_rows else (torch.float32, D)
    arr = _lookup_tables(weights, indices, B, wdt, wcols, slots, rows)
    for t in range(n):
        g = grad_rows[t]
        if g is not None:
            _dev(g, f"grad_rows[{t}]", torch.float32)
            if g.shape[0] != B or g.shape[1] != D:
                raise ValueError(f"grad_rows[{t}] must be ({B}, {D})")
            st = _row_stride(g, f"grad_rows[{t}]")
            if gstride not in (None, st):
                raise ValueError("all grad_rows must share one row stride")
            gstride = st
            gp[t] = g.data_ptr()
    P = 0
    F = n + (1 if bottom is not None else 0)
    bstride = 0
    if bottom is not None:
        _dev(bottom, "bottom", wdt)
        if bottom.shape[0] != B or bottom.shape[1] != wcols:
            raise ValueError(f"bottom must be ({B}, {wcols}) {wdt}")
        bstride = _row_stride(bottom, "bottom") // (2 if operand_rows else 1)
        P = dA.shape[1] - F * (F - 1) // 2
    _cabi.check(
        _lib().mm_dlrm_interact_backward(arr, n, B, D, _ptr(bottom), bstride, bottom_slot, P, dA.data_ptr(), _row_stride(dA, "dA"), gp,
                                         gstride or D, _ptr(d_bottom),
                                         0 if d_bottom is None else _row_stride(_dev(d_bottom, "d_bottom", torch.float32), "d_bottom"),
                                         1 if mask_bottom else 0, 1 if operand_rows else 0, _stream()),
        "mm_dlrm_interact_backward")


def sparse_rows_apply(opt: str, tables, B: int, D: int, hyper: torch.Tensor) -> None:
    """Optimizer step on IndexedSlices (mm_sparse_rows_apply).  tables: dicts with weights, indices, grad_rows, rep_map and, per
    optimizer, state1 / state2, optionally mirror and dense_grad (a zeroed (rows, D) accumulator: selects the dense path for
    tables with few rows, see include/mm_b200.h)."""
    _dev(hyper, "hyper", torch.float32)
    n = len(tables)
    arr = (_cabi.SparseTable * n)()
    for t, tb in enumerate(tables):
        w = _dev(tb["weights"], f"tables[{t}].weights", torch.float32)
        ix = _dev(tb["indices"], f"tables[{t}].indices")
        g = _dev(tb["grad_rows"], f"tables[{t}].grad_rows", torch.float32)
        rep = _dev(tb["rep_map"], f"tables[{t}].rep_map", torch.int32)
        if w.dim() != 2 or w.shape[1] != D or not w.is_contiguous() or tuple(g.shape) != (B, D) or not g.is_contiguous():
            raise ValueError(f"tables[{t}]: weights must be contiguous (rows, {D}) and grad_rows contiguous ({B}, {D})")
        if rep.numel() != w.shape[0]:
            raise ValueError(f"tables[{t}]: rep_map must hold one int32 per row")
        arr[t].weights, arr[t].rows, arr[t].indices, arr[t].idx_bytes = w.data_ptr(), w.shape[0], ix.data_ptr(), index_bytes_of(ix)
        arr[t].grad_rows, arr[t].rep_map = g.data_ptr(), rep.data_ptr()
        for key in ("state1", "state2"):
            s = tb.get(key)
            if s is not None and (_dev(s, f"tables[{t}].{key}", torch.float32).shape != w.shape or not s.is_contiguous()):
                raise ValueError(f"tables[{t}].{key} must match the weights")
            setattr(arr[t], key, _ptr(s))
        m = tb.get("mirror")
        if m is not None and (_dev(m, f"tables[{t}].mirror", torch.bfloat16).shape != (w.shape[0], 2 * D) or not m.is_contiguous()):
            raise ValueError(f"tables[{t}].mirror must be contiguous bf16 (rows, {2 * D})")
        arr[t].mirror = _ptr(m)
        dg = tb.get("dense_grad")
        if dg is not None and (_dev(dg, f"tables[{t}].dense_grad", torch.float32).shape != w.shape or not dg.is_contiguous()):
            raise ValueError(f"tables[{t}].dense_grad must match the weights")
        arr[t].dense_grad = _ptr(dg)
    _cabi.check(_lib().mm_sparse_rows_apply(arr, n, B, D, _cabi.OPTIMIZERS[opt], hyper.data_ptr(), _stream()), "mm_sparse_rows_apply")


def bag_grad_rows(g: torch.Tensor, ids: torch.Tensor, offsets: Optional[torch.Tensor], rows: int, combiner: str,
                  out: torch.Tensor, out_ids: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Backward of gather_bag (offsets given: ids (nnz,), offsets (B+1,)) or gather_seq (offsets None: ids (B, L)) for
    the pooled-row gradient g (B, D): out (nnz, D) row i = scale(i) * g[bag(i)], zero for ids outside [0, rows)
    (mm_bag_grad_rows).  Every row of `out` is written.  out_ids (nnz,), the ids' dtype: the id of every row that carries
    a gradient, -1 for positions no bag covers and ids outside [0, rows) — the indices for sparse_rows_apply."""
    _dev(g, "g", torch.float32), _dev(ids, "ids"), _dev(out, "out", torch.float32)
    if combiner not in COMBINERS:
        raise ValueError(f"unknown combiner {combiner!r}")
    if g.dim() != 2:
        raise ValueError(f"g must be (B, D), got {tuple(g.shape)}")
    B, D = g.shape
    if not ids.is_contiguous():
        raise ValueError("ids must be contiguous")
    nnz = ids.numel()
    if tuple(out.shape) != (nnz, D) or not out.is_contiguous():
        raise ValueError(f"out must be contiguous ({nnz}, {D}), got {tuple(out.shape)}")
    if offsets is None:
        if ids.dim() != 2 or ids.shape[0] != B:
            raise ValueError(f"fixed-length bags need ids (B={B}, L), got {tuple(ids.shape)}")
        L, off_ptr, off_dt = ids.shape[1], None, MM_I32
    else:
        _dev(offsets, "offsets")
        if offsets.numel() != B + 1 or not offsets.is_contiguous():
            raise ValueError(f"offsets must be contiguous with B+1={B + 1} elements, got {tuple(offsets.shape)}")
        L, off_ptr, off_dt = 0, offsets.data_ptr(), _idx_dtype(offsets, "offsets")
    if out_ids is not None and (_dev(out_ids, "out_ids", ids.dtype).numel() != nnz or not out_ids.is_contiguous()):
        raise ValueError(f"out_ids must be contiguous with {nnz} elements of the ids' dtype")
    _cabi.check(_lib().mm_bag_grad_rows(g.data_ptr(), B, D, _row_stride(g, "g"), ids.data_ptr(), _idx_dtype(ids, "ids"), off_ptr, off_dt,
                                        L, nnz, int(rows), COMBINERS[combiner], out.data_ptr(), _ptr(out_ids), _stream()),
                "mm_bag_grad_rows")
    return out


def cross_backward(x0: torch.Tensor, z: torch.Tensor, g: torch.Tensor, p: Optional[torch.Tensor], acc: torch.Tensor, acc_init: bool,
                   dz: torch.Tensor, dz_split: torch.Tensor) -> None:
    """One DCN-v2 cross layer of the backward (mm_cross_backward): g += p (in place; p None for the top layer),
    dz = g * x0 as fp32 and as the split-bf16 operand dz_split (B, 2*Kp), acc = g * z (acc_init) or acc += g * z.
    All fp32 operands (B, d) with row strides that are multiples of 4."""
    fs = [("x0", x0), ("z", z), ("g", g), ("acc", acc), ("dz", dz)] + ([("p", p)] if p is not None else [])
    for n_, t_ in fs:
        _dev(t_, n_, torch.float32)
    B, d = x0.shape
    for n_, t_ in fs:
        if tuple(t_.shape) != (B, d):
            raise ValueError(f"{n_} must be ({B}, {d}), got {tuple(t_.shape)}")
    _dev(dz_split, "dz_split", torch.bfloat16)
    Kp = tc_padded_k(d)
    if tuple(dz_split.shape) != (B, 2 * Kp) or not dz_split.is_contiguous():
        raise ValueError(f"dz_split must be a contiguous bf16 ({B}, {2 * Kp}) matrix")
    _cabi.check(_lib().mm_cross_backward(x0.data_ptr(), _row_stride(x0, "x0"), z.data_ptr(), _row_stride(z, "z"), g.data_ptr(),
                                         _row_stride(g, "g"), _ptr(p), 0 if p is None else _row_stride(p, "p"), acc.data_ptr(),
                                         _row_stride(acc, "acc"), 1 if acc_init else 0, B, d, dz.data_ptr(), _row_stride(dz, "dz"),
                                         dz_split.data_ptr(), Kp, _stream()), "mm_cross_backward")


def _addends_slices(addends: Sequence[torch.Tensor], slices: Sequence[tuple], B: int, d: int):
    """(pointers, row strides, mm_column_slice array) of a concat backward's (B, d) fp32 addends and its (dst (B, width), col)
    slices."""
    n = len(addends)
    ap, st = (C.c_void_p * max(n, 1))(), (C.c_int64 * max(n, 1))()
    for i, a in enumerate(addends):
        _dev(a, f"addends[{i}]", torch.float32)
        if tuple(a.shape) != (B, d):
            raise ValueError(f"addends[{i}] must be ({B}, {d}), got {tuple(a.shape)}")
        ap[i], st[i] = a.data_ptr(), _row_stride(a, f"addends[{i}]")
    arr = (_cabi.ColumnSlice * max(len(slices), 1))()
    for t, (dst, col) in enumerate(slices):
        _dev(dst, f"slices[{t}].dst", torch.float32)
        if dst.dim() != 2 or dst.shape[0] != B:
            raise ValueError(f"slices[{t}].dst must be ({B}, width), got {tuple(dst.shape)}")
        arr[t].dst, arr[t].dst_stride, arr[t].col, arr[t].width = dst.data_ptr(), _row_stride(dst, f"slices[{t}].dst"), int(col), dst.shape[1]
    return ap, st, arr


def concat_backward(addends: Sequence[torch.Tensor], slices: Sequence[tuple]) -> None:
    """Backward of a concatenated input block (mm_concat_backward): for each (dst (B, w), col) in `slices`,
    dst = sum of the (B, d) addends' columns [col, col + w)."""
    if not addends:
        raise ValueError("concat_backward needs at least one addend")
    B, d = addends[0].shape
    ap, st, arr = _addends_slices(addends, slices, B, d)
    _cabi.check(_lib().mm_concat_backward(ap, st, len(addends), B, d, arr, len(slices), _stream()), "mm_concat_backward")


def concat_l2_workspace(n_slices: int, device) -> torch.Tensor:
    """The per-CTA partials concat_backward_l2 needs for up to n_slices slices."""
    return torch.zeros(n_slices * _cabi.CONCAT_L2_CTAS, dtype=torch.float32, device=device)


def concat_backward_l2(addends: Sequence[torch.Tensor], slices: Sequence[tuple], x0: torch.Tensor, l2: Sequence[float],
                       loss: torch.Tensor, partials: torch.Tensor) -> None:
    """concat_backward plus the embeddings' L2 penalty (mm_concat_backward_l2): for each (dst (B, w), col) in `slices` with
    factor l2[t], dst = sum of the addends' columns [col, col + w) + 2 l2[t] x0[:, col:col + w]; reg = sum_t l2[t] ||x0's
    columns of t||^2 is added to loss[0] (the total) and loss[1] in a fixed order.  partials: concat_l2_workspace."""
    if not addends:
        raise ValueError("concat_backward needs at least one addend")
    B, d = addends[0].shape
    _dev(x0, "x0", torch.float32), _dev(loss, "loss", torch.float32), _dev(partials, "partials", torch.float32)
    if tuple(x0.shape) != (B, d):
        raise ValueError(f"x0 must be ({B}, {d}), got {tuple(x0.shape)}")
    if len(l2) != len(slices):
        raise ValueError(f"one l2 factor per slice expected ({len(slices)}), got {len(l2)}")
    if loss.numel() != 2 or not loss.is_contiguous():
        raise ValueError("loss must hold 2 contiguous values [total, regularization]")
    if not partials.is_contiguous():
        raise ValueError("partials must be contiguous")
    ap, st, arr = _addends_slices(addends, slices, B, d)
    lam = (C.c_float * max(len(l2), 1))(*[float(v) for v in l2])
    _cabi.check(_lib().mm_concat_backward_l2(ap, st, len(addends), B, d, arr, len(slices), x0.data_ptr(), _row_stride(x0, "x0"), lam,
                                             partials.data_ptr(), partials.numel(), loss.data_ptr(), _stream()),
                "mm_concat_backward_l2")


def dense_apply(opt: str, w: torch.Tensor, grad: torch.Tensor, state1: Optional[torch.Tensor], state2: Optional[torch.Tensor],
                hyper: torch.Tensor, grad_scale: float = 1.0) -> None:
    """Optimizer step over a flat fp32 arena; grad is scaled by grad_scale and cleared (mm_dense_apply)."""
    for n_, t_ in (("w", w), ("grad", grad), ("hyper", hyper)):
        _dev(t_, n_, torch.float32)
    if not (w.is_contiguous() and grad.is_contiguous() and w.numel() == grad.numel()):
        raise ValueError("w and grad must be contiguous and equally sized")
    _cabi.check(_lib().mm_dense_apply(_cabi.OPTIMIZERS[opt], w.data_ptr(), grad.data_ptr(), _ptr(state1), _ptr(state2), w.numel(),
                                      hyper.data_ptr(), float(grad_scale), _stream()), "mm_dense_apply")


def opt_tick(hyper: torch.Tensor) -> None:
    _cabi.check(_lib().mm_opt_tick(_dev(hyper, "hyper", torch.float32).data_ptr(), _stream()), "mm_opt_tick")


def schedule_params(kind: str, initial_learning_rate: float = 0.0, decay_steps: float = 1.0, rate: float = 0.0,
                    power: float = 1.0, flag: bool = False, boundaries: Sequence[float] = (),
                    values: Sequence[float] = ()) -> np.ndarray:
    """The K25 device array float[SCHED_COUNT] of a learning-rate schedule `kind` (a key of _cabi.SCHED_KINDS); rate is
    decay_rate, end_learning_rate or alpha, flag staircase or cycle.  PiecewiseConstantDecay takes 1..SCHED_MAX_BOUNDARIES
    increasing boundaries and one value more."""
    if kind not in _cabi.SCHED_KINDS:
        raise ValueError(f"unknown learning-rate schedule {kind!r}; supported: {sorted(_cabi.SCHED_KINDS)}")
    s = np.zeros(_cabi.SCHED_COUNT, dtype=np.float32)
    s[_cabi.SCHED_KIND] = _cabi.SCHED_KINDS[kind]
    if kind == "PiecewiseConstantDecay":
        nb = len(boundaries)
        if not 1 <= nb <= _cabi.SCHED_MAX_BOUNDARIES:
            raise NotImplementedError(f"PiecewiseConstantDecay with {nb} boundaries: the device schedule takes "
                                      f"1..{_cabi.SCHED_MAX_BOUNDARIES}")
        if len(values) != nb + 1:
            raise ValueError(f"{nb} boundaries need {nb + 1} values, got {len(values)}")
        b = np.asarray(boundaries, dtype=np.float32)
        if np.any(np.diff(b) <= 0):
            raise ValueError(f"boundaries must be increasing, got {list(boundaries)}")
        s[_cabi.SCHED_NB] = nb
        s[_cabi.SCHED_BOUNDARIES:_cabi.SCHED_BOUNDARIES + nb] = b
        s[_cabi.SCHED_VALUES:_cabi.SCHED_VALUES + nb + 1] = np.asarray(values, dtype=np.float32)
        return s
    if not decay_steps > 0:
        raise ValueError(f"decay_steps must be > 0, got {decay_steps}")
    s[_cabi.SCHED_INIT], s[_cabi.SCHED_DECAY_STEPS], s[_cabi.SCHED_RATE] = initial_learning_rate, decay_steps, rate
    s[_cabi.SCHED_POWER], s[_cabi.SCHED_FLAG] = power, 1.0 if flag else 0.0
    return s


def opt_tick_schedule(hyper: torch.Tensor, sched: torch.Tensor) -> None:
    """mm_opt_tick with hyper[HYPER_LR] = lr(step) of the schedule `sched` (schedule_params' array on the device) first."""
    _dev(hyper, "hyper", torch.float32), _dev(sched, "sched", torch.float32)
    if hyper.numel() < _cabi.HYPER_COUNT or not hyper.is_contiguous():
        raise ValueError(f"hyper must hold {_cabi.HYPER_COUNT} contiguous values, got {tuple(hyper.shape)}")
    _vec(sched, _cabi.SCHED_COUNT, "sched")
    if sched.device != hyper.device:
        raise ValueError(f"sched is on {sched.device}, hyper on {hyper.device}")
    _cabi.check(_lib().mm_opt_tick_schedule(hyper.data_ptr(), sched.data_ptr(), _stream()), "mm_opt_tick_schedule")


def fill_i32(t: torch.Tensor, value: int) -> torch.Tensor:
    _cabi.check(_lib().mm_fill_i32(_dev(t, "t", torch.int32).data_ptr(), t.numel(), int(value), _stream()), "mm_fill_i32")
    return t


# ---- factorization-machine heads (include/mm_b200.h K15) ---------------------------------------------------------
def fm_pairwise(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """FMPairwiseInteraction: x (B, A, K) -> (B, K) = 0.5 ((sum_a x)^2 - sum_a x^2)  (mm_fm_pairwise)."""
    _dev(x, "x", torch.float32)
    if x.dim() != 3 or not x.is_contiguous():
        raise ValueError("inputs should be a contiguous 3-D tensor")
    B, A, K = x.shape
    if out is None:
        out = torch.empty((B, K), dtype=torch.float32, device=x.device)
    _cabi.check(_lib().mm_fm_pairwise(x.data_ptr(), B, A, K, out.data_ptr(), _stream()), "mm_fm_pairwise")
    return out


def deepfm_head(weights, indices, wide_offsets, cont, cont_offsets, wide_kernel: torch.Tensor, wide_bias: Optional[torch.Tensor],
                addend: Optional[torch.Tensor], out_w: Optional[torch.Tensor], out_b: Optional[torch.Tensor], out_act: Optional[str],
                out: torch.Tensor, oob: Optional[torch.Tensor] = None) -> torch.Tensor:
    """FM pairwise term + wide (one-hot Dense(1) as a row lookup) + deep logit (+ output layer) per sample (mm_deepfm_head)."""
    _dev(out, "out", torch.float32), _dev(wide_kernel, "wide_kernel", torch.float32)
    B = out.numel()
    n = len(weights)
    if not (len(indices) == n and len(wide_offsets) == n):
        raise ValueError("weights / indices / wide_offsets length mismatch")
    D = weights[0].shape[1]
    arr = _lookup_tables(weights, indices, B, torch.float32, D)
    woff = (C.c_int64 * n)(*[int(o) for o in wide_offsets])
    carr, coff, m = _cont_columns(cont, cont_offsets, B)
    if addend is not None and (_dev(addend, "addend", torch.float32).numel() != B):
        raise ValueError(f"addend must hold {B} values")
    a_stride = 0 if addend is None else (addend.stride(0) if addend.dim() >= 1 else 1)
    _cabi.check(
        _lib().mm_deepfm_head(arr, woff, n, B, D, carr, coff, m, wide_kernel.data_ptr(), _ptr(wide_bias), _ptr(addend), a_stride,
                              _ptr(out_w), _ptr(out_b), ACTIVATIONS[out_act], out.data_ptr(), _ptr(oob), _stream()),
        "mm_deepfm_head")
    return out


# ---- DeepFM training (include/mm_b200.h, added with DeepFM training) ------------------------------------------------
def _wide_blocks(indices, rows, offsets, B: int):
    n = len(indices)
    if not (len(rows) == n and len(offsets) == n):
        raise ValueError("indices / rows / offsets length mismatch")
    arr = (_cabi.WideBlock * max(n, 1))()
    for t in range(n):
        ix = indices[t]
        w = _id_column(ix, B, f"indices[{t}]", leading=True)
        arr[t].indices, arr[t].rows, arr[t].offset, arr[t].idx_bytes = ix.data_ptr(), int(rows[t]), int(offsets[t]), w
    return arr, n


def deepfm_head_fwd_bwd(x0: torch.Tensor, emb_cols, D: int, indices, rows, wide_offsets, cont, cont_offsets,
                        wide_kernel: torch.Tensor, wide_bias: Optional[torch.Tensor], h: torch.Tensor, mask_h: bool,
                        w_dl: torch.Tensor, b_dl: Optional[torch.Tensor], act_dl: str, out_w: torch.Tensor,
                        out_b: Optional[torch.Tensor], loss: str, targets: torch.Tensor, sample_weight: Optional[torch.Tensor],
                        logits: torch.Tensor, loss_buf: torch.Tensor, ds: torch.Tensor, dh: torch.Tensor,
                        dw_out: Optional[torch.Tensor] = None, db_out: Optional[torch.Tensor] = None,
                        dw_dl: Optional[torch.Tensor] = None, db_dl: Optional[torch.Tensor] = None,
                        d_wide_bias: Optional[torch.Tensor] = None, d_cont: Optional[torch.Tensor] = None,
                        oob: Optional[torch.Tensor] = None) -> None:
    """The DeepFM head's forward, loss and backward in one pass (mm_deepfm_head_fwd_bwd).  x0 (B, d) holds the gathered
    rows at emb_cols; indices[f] (B,) ids of any width of index_bytes_of, rows[f] its table's rows, wide_offsets[f] its
    block in the wide kernel; cont (B,) columns at cont_offsets.  Writes logits, ds (B,) and dh (B, U); ACCUMULATES
    loss_buf (2,) and the gradients (each nullable)."""
    for n_, t_ in (("x0", x0), ("wide_kernel", wide_kernel), ("h", h), ("w_dl", w_dl), ("out_w", out_w), ("logits", logits),
                   ("loss_buf", loss_buf), ("ds", ds), ("dh", dh)):
        _dev(t_, n_, torch.float32)
    B = x0.shape[0]
    U = h.shape[1]
    if h.shape[0] != B or tuple(dh.shape) != (B, U):
        raise ValueError(f"h and dh must be ({B}, units)")
    if not wide_kernel.is_contiguous() or w_dl.numel() != U or not w_dl.is_contiguous():
        raise ValueError(f"wide_kernel must be contiguous and w_dl hold {U} contiguous values")
    for n_, t_, k in (("out_w", out_w, 1), ("out_b", out_b, 1), ("b_dl", b_dl, 1), ("wide_bias", wide_bias, 1),
                      ("dw_out", dw_out, 1), ("db_out", db_out, 1), ("db_dl", db_dl, 1), ("d_wide_bias", d_wide_bias, 1),
                      ("dw_dl", dw_dl, U), ("d_cont", d_cont, len(cont))):
        _vec(t_, k, n_, "hold {n} contiguous float32 values")
    if logits.numel() != B or ds.numel() != B or not logits.is_contiguous() or not ds.is_contiguous():
        raise ValueError(f"logits and ds must hold {B} contiguous values")
    if loss_buf.numel() != 2 or not loss_buf.is_contiguous():
        raise ValueError("loss_buf must hold 2 contiguous values")
    if loss not in _cabi.LOSS_KINDS:
        raise ValueError(f"loss must be among {sorted(_cabi.LOSS_KINDS)}, got {loss!r}")
    if act_dl not in ("linear", "relu"):
        raise ValueError(f"the deep logit's activation must be linear or relu, got {act_dl!r}")
    target_dtype = _target(targets, B, "targets")
    _vec(sample_weight, B, "sample_weight", _SAMPLE_WEIGHT)
    n = len(indices)
    if len(emb_cols) != n:
        raise ValueError("emb_cols / indices length mismatch")
    arr, _ = _wide_blocks(indices, rows, wide_offsets, B)
    cols = (C.c_int64 * max(n, 1))(*[int(c) for c in emb_cols])
    carr, coff, m = _cont_columns(cont, cont_offsets, B)
    _cabi.check(
        _lib().mm_deepfm_head_fwd_bwd(x0.data_ptr(), _row_stride(x0, "x0"), cols, int(D), arr, n, carr, coff, m, wide_kernel.data_ptr(),
                                      _ptr(wide_bias), h.data_ptr(), _row_stride(h, "h"), U, 1 if mask_h else 0, w_dl.data_ptr(),
                                      _ptr(b_dl), ACTIVATIONS[act_dl], out_w.data_ptr(), _ptr(out_b), _cabi.LOSS_KINDS[loss],
                                      targets.data_ptr(), target_dtype, _ptr(sample_weight), B, logits.data_ptr(),
                                      loss_buf.data_ptr(), ds.data_ptr(), dh.data_ptr(), _row_stride(dh, "dh"), _ptr(dw_out),
                                      _ptr(db_out), _ptr(dw_dl), _ptr(db_dl), _ptr(d_wide_bias), _ptr(d_cont), _ptr(oob), _stream()),
        "mm_deepfm_head_fwd_bwd")


def fm_concat_backward(addends: Sequence[torch.Tensor], x0: torch.Tensor, ds: torch.Tensor, slices: Sequence[tuple]) -> None:
    """concat_backward plus the FM term (mm_fm_concat_backward): for each (dst (B, D), col) in `slices`,
    dst = sum of the addends' columns [col, col + D) + ds[:, None] * (S - x0[:, col:col + D]), S the row sum of that slice."""
    _dev(x0, "x0", torch.float32), _dev(ds, "ds", torch.float32)
    B, d = x0.shape
    if ds.numel() != B or not ds.is_contiguous():
        raise ValueError(f"ds must hold {B} contiguous values")
    ap, st, arr = _addends_slices(addends, slices, B, d)
    _cabi.check(_lib().mm_fm_concat_backward(ap, st, len(addends), B, d, x0.data_ptr(), _row_stride(x0, "x0"), ds.data_ptr(), arr,
                                             len(slices), _stream()), "mm_fm_concat_backward")


def wide_rows_apply(opt: str, wide: torch.Tensor, state1: Optional[torch.Tensor], state2: Optional[torch.Tensor], indices, rows,
                    offsets, grad: torch.Tensor, acc: torch.Tensor, rep_map: torch.Tensor, dense_offsets, dense_grad: Optional[torch.Tensor],
                    bias: Optional[torch.Tensor], bias_state1: Optional[torch.Tensor], bias_state2: Optional[torch.Tensor],
                    hyper: torch.Tensor) -> None:
    """Optimizer step of a wide kernel (mm_wide_rows_apply): block f = rows [offsets[f], offsets[f] + rows[f]) addressed by
    indices[f], gradient values grad (B,) for every block; the rows at dense_offsets and the bias take the dense rule with
    dense_grad (len(dense_offsets) [+ 1],), which is cleared."""
    W = wide.numel()
    for n_, t_ in (("wide", wide), ("grad", grad), ("acc", acc), ("hyper", hyper)):
        _dev(t_, n_, torch.float32)
    _dev(rep_map, "rep_map", torch.int32)
    for n_, t_ in (("wide", wide), ("acc", acc), ("rep_map", rep_map), ("state1", state1), ("state2", state2)):
        if t_ is not None and (t_.numel() != W or not t_.is_contiguous()):
            raise ValueError(f"{n_} must hold {W} contiguous values (one per row of the wide kernel)")
    for n_, t_ in (("state1", state1), ("state2", state2), ("bias", bias), ("bias_state1", bias_state1), ("bias_state2", bias_state2)):
        if t_ is not None:
            _dev(t_, n_, torch.float32)
    B = grad.numel()
    if not grad.is_contiguous():
        raise ValueError("grad must be contiguous")
    arr, n = _wide_blocks(indices, rows, offsets, B)
    m = len(dense_offsets)
    k = m + (1 if bias is not None else 0)
    if k and (dense_grad is None or _dev(dense_grad, "dense_grad", torch.float32).numel() != k or not dense_grad.is_contiguous()):
        raise ValueError(f"dense_grad must hold {k} contiguous values")
    doff = (C.c_int64 * max(m, 1))(*[int(o) for o in dense_offsets])
    _cabi.check(_lib().mm_wide_rows_apply(wide.data_ptr(), _ptr(state1), _ptr(state2), W, arr, n, B, grad.data_ptr(), acc.data_ptr(),
                                          rep_map.data_ptr(), doff, m, _ptr(dense_grad), _ptr(bias), _ptr(bias_state1), _ptr(bias_state2),
                                          _cabi.OPTIMIZERS[opt], hyper.data_ptr(), _stream()), "mm_wide_rows_apply")


def metrics_workspace_bytes(M: int, H: int) -> int:
    return int(_lib().mm_metrics_workspace_bytes(int(M), int(H)))


def metrics_update(z: torch.Tensor, losses: Sequence[str], targets: Sequence[torch.Tensor], state: torch.Tensor,
                   workspace: torch.Tensor, num_buckets: int, pred_forms: Sequence[int],
                   thresholds: Sequence[Sequence[float]], sample_weight: Optional[Sequence[Optional[torch.Tensor]]] = None,
                   metric_weights: Optional[Sequence[Sequence[Optional[torch.Tensor]]]] = None) -> torch.Tensor:
    """Add one batch of H <= 8 heads' logits z (H, M) into the fp64 metric state (mm_metrics_update): loss sums, AUC
    histograms of num_buckets, confusion counts at each head's thresholds (<= 4) and squared-error sums, per metric set.
    losses[h] in {"binary_crossentropy", "mse"}; targets[h] (M,) int32 / int64 / float32 / float64; pred_forms[h]
    _cabi.PRED_ACT / PRED_HEAD; sample_weight[h] the loss weights (or None); metric_weights[s][h] the weights of metric set s
    (1 or 2 sets; entries None: unweighted; default one unweighted set).  state (H, METRICS_SCALARS + 4 num_buckets)
    float64, accumulated."""
    _dev(z, "z", torch.float32)
    H = len(losses)
    if not 1 <= H <= _cabi.METRICS_MAX_HEADS:
        raise ValueError(f"1..{_cabi.METRICS_MAX_HEADS} heads, got {H}")
    if z.dim() != 2 or z.shape[0] != H or not z.is_contiguous():
        raise ValueError(f"z must be a contiguous ({H}, M) matrix, got {tuple(z.shape)}")
    M = z.shape[1]
    T = int(num_buckets)
    if not 2 <= T <= _cabi.METRICS_MAX_BUCKETS:
        raise ValueError(f"num_buckets must lie in [2, {_cabi.METRICS_MAX_BUCKETS}], got {T}")
    _dev(state, "state", torch.float64)
    if tuple(state.shape) != (H, _cabi.METRICS_SCALARS + 4 * T) or not state.is_contiguous():
        raise ValueError(f"state must be a contiguous ({H}, {_cabi.METRICS_SCALARS + 4 * T}) float64 matrix")
    sets = [[None] * H] if metric_weights is None else [list(s) for s in metric_weights]
    if len(sets) not in (1, 2) or any(len(s) != H for s in sets):
        raise ValueError(f"one or two metric sets of {H} weight entries each")
    sws = list(sample_weight) if sample_weight is not None else [None] * H
    for name, seq in (("targets", targets), ("pred_forms", pred_forms), ("thresholds", thresholds), ("sample_weight", sws)):
        if len(seq) != H:
            raise ValueError(f"{name}: one entry per head ({H}), got {len(seq)}")
    arr = (_cabi.MetricsHead * H)()
    for h in range(H):
        if losses[h] not in _cabi.LOSS_KINDS:
            raise ValueError(f"losses must be among {sorted(_cabi.LOSS_KINDS)}, got {losses[h]!r}")
        arr[h].target_dtype = _target(targets[h], M, f"targets[{h}]")
        ws = [sws[h]] + [s[h] for s in sets]
        for i, w in enumerate(ws):
            if w is not None and (_dev(w, "weights", torch.float32).numel() != M or not w.is_contiguous()):
                raise ValueError(f"head {h}: sample / metric weights must be ({M},) contiguous float32")
        thr = [float(v) for v in thresholds[h]]
        if len(thr) > _cabi.METRICS_MAX_THRESHOLDS:
            raise ValueError(f"head {h}: at most {_cabi.METRICS_MAX_THRESHOLDS} thresholds, got {len(thr)}")
        arr[h].targets = targets[h].data_ptr()
        arr[h].sample_weight = _ptr(sws[h])
        for s in range(len(sets)):
            arr[h].metric_weights[s] = _ptr(sets[s][h])
        arr[h].loss_kind = _cabi.LOSS_KINDS[losses[h]]
        arr[h].pred_form = int(pred_forms[h])
        arr[h].n_thresholds = len(thr)
        for i, v in enumerate(thr):
            arr[h].thresholds[i] = v
    _dev(workspace, "workspace")
    need = metrics_workspace_bytes(M, H)
    if workspace.numel() * workspace.element_size() < need or not workspace.is_contiguous():
        raise ValueError(f"workspace must hold {need} contiguous bytes")
    _cabi.check(_lib().mm_metrics_update(z.data_ptr(), M, H, arr, T, len(sets), state.data_ptr(), workspace.data_ptr(),
                                         workspace.numel() * workspace.element_size(), _stream()), "mm_metrics_update")
    return state


# ---- Wide&Deep head (include/mm_b200.h K18) -------------------------------------------------------------------------
_BAG_ID_BYTES = {torch.uint8: 1, torch.uint16: 2, torch.int32: 4, torch.int64: 8}


def _wide_bags(bags, B: int):
    """mm_wide_bag array of bag blocks (values, offsets, rows, offset, mode): values (nnz,) ids with offsets (B + 1,)
    int32 / int64, or a (B, L) id matrix with offsets None; ids uint8 / uint16 / int32 / int64; mode "multi_hot" or
    "count"."""
    arr = (_cabi.WideBag * max(len(bags), 1))()
    for i, (values, offsets, rows, offset, mode) in enumerate(bags):
        v = _dev(values, f"bags[{i}].values")
        if v.dtype not in _BAG_ID_BYTES or not v.is_contiguous():
            raise ValueError(f"bags[{i}].values must be contiguous uint8 / uint16 / int32 / int64 ids, got {v.dtype}")
        if mode not in _cabi.WIDE_MODES:
            raise ValueError(f"bags[{i}]: mode must be one of {sorted(_cabi.WIDE_MODES)}, got {mode!r}")
        if offsets is None:
            if v.dim() != 2 or v.shape[0] != B:
                raise ValueError(f"bags[{i}]: fixed-length ids must be a (B={B}, L) matrix, got {tuple(v.shape)}")
            arr[i].length, arr[i].offsets, arr[i].off_dtype = v.shape[1], None, MM_I32
        else:
            o = _dev(offsets, f"bags[{i}].offsets")
            if o.numel() != B + 1 or not o.is_contiguous():
                raise ValueError(f"bags[{i}].offsets must be contiguous with B+1={B + 1} elements, got {tuple(o.shape)}")
            arr[i].length, arr[i].offsets, arr[i].off_dtype = 0, o.data_ptr(), _idx_dtype(o, f"bags[{i}].offsets")
        arr[i].values, arr[i].nnz, arr[i].idx_bytes = v.data_ptr(), v.numel(), _BAG_ID_BYTES[v.dtype]
        arr[i].rows, arr[i].offset, arr[i].mode = int(rows), int(offset), _cabi.WIDE_MODES[mode]
    return arr, len(bags)


def wide_deep_head_fwd_bwd(onehot, bags, wide_kernel: Optional[torch.Tensor], wide_bias: Optional[torch.Tensor],
                           h: Optional[torch.Tensor], mask_h: bool, w_dl: Optional[torch.Tensor], b_dl: Optional[torch.Tensor],
                           act_dl: str, out_w: torch.Tensor, out_b: Optional[torch.Tensor], out: torch.Tensor,
                           out_act: Optional[str] = "linear", loss: Optional[str] = None, targets: Optional[torch.Tensor] = None,
                           sample_weight: Optional[torch.Tensor] = None, loss_buf: Optional[torch.Tensor] = None,
                           ds: Optional[torch.Tensor] = None, dh: Optional[torch.Tensor] = None,
                           dw_out: Optional[torch.Tensor] = None, db_out: Optional[torch.Tensor] = None,
                           dw_dl: Optional[torch.Tensor] = None, db_dl: Optional[torch.Tensor] = None,
                           d_wide_bias: Optional[torch.Tensor] = None, oob: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The Wide&Deep head in one pass (mm_wide_deep_head_fwd_bwd).  onehot: (ids (B,) of any width of index_bytes_of, rows,
    offset) per one-hot wide feature; bags: see _wide_bags; h (B, U) the deep tower's last hidden layer and w_dl (U,) /
    b_dl the deep logit's Dense(1), or h None for a model without a deep part.  targets None: out (B,) = out_act(z).
    Otherwise out = z, ds (B,) and dh (B, U) are written and loss_buf (2,) and the gradients (each nullable) ACCUMULATED."""
    _dev(out, "out", torch.float32), _dev(out_w, "out_w", torch.float32)
    B = out.numel()
    if not out.is_contiguous():
        raise ValueError("out must be contiguous")
    if wide_kernel is not None and (not _dev(wide_kernel, "wide_kernel", torch.float32).is_contiguous()):
        raise ValueError("wide_kernel must be contiguous")
    for n_, t_ in (("out_w", out_w), ("out_b", out_b), ("b_dl", b_dl), ("wide_bias", wide_bias), ("dw_out", dw_out),
                   ("db_out", db_out), ("db_dl", db_dl), ("d_wide_bias", d_wide_bias)):
        _vec(t_, 1, n_, "hold {n} contiguous float32 values")
    U, hs, dhs = 0, 0, 0
    if h is not None:
        _dev(h, "h", torch.float32)
        U = h.shape[1]
        hs = _row_stride(h, "h")
        if h.shape[0] != B or w_dl is None:
            raise ValueError(f"h must be ({B}, units) with the deep logit's kernel w_dl")
        _vec(w_dl, U, "w_dl", "hold {n} contiguous float32 values")
        _vec(dw_dl, U, "dw_dl", "hold {n} contiguous float32 values")
        if act_dl not in ("linear", "relu"):
            raise ValueError(f"the deep logit's activation must be linear or relu, got {act_dl!r}")
    target_dtype = 0
    if targets is not None:
        if loss not in _cabi.LOSS_KINDS:
            raise ValueError(f"loss must be among {sorted(_cabi.LOSS_KINDS)}, got {loss!r}")
        target_dtype = _target(targets, B, "targets")
        _vec(sample_weight, B, "sample_weight", _SAMPLE_WEIGHT)
        _vec(ds, B, "ds", "hold {n} contiguous float32 values")
        if ds is None:
            raise ValueError("training needs ds")
        if loss_buf is not None and (_dev(loss_buf, "loss_buf", torch.float32).numel() != 2 or not loss_buf.is_contiguous()):
            raise ValueError("loss_buf must hold 2 contiguous values")
        if h is not None:
            if dh is None or tuple(_dev(dh, "dh", torch.float32).shape) != (B, U):
                raise ValueError(f"training with a deep part needs dh ({B}, {U})")
            dhs = _row_stride(dh, "dh")
    n_oh = len(onehot)
    oh = (_cabi.WideBlock * max(n_oh, 1))()
    for i, (ix, rows, off) in enumerate(onehot):
        oh[i].idx_bytes = _id_column(ix, B, f"onehot[{i}]", leading=True)
        oh[i].indices, oh[i].rows, oh[i].offset = ix.data_ptr(), int(rows), int(off)
    barr, n_bag = _wide_bags(bags, B)
    train = targets is not None
    _cabi.check(
        _lib().mm_wide_deep_head_fwd_bwd(oh, n_oh, barr, n_bag, _ptr(wide_kernel), _ptr(wide_bias), _ptr(h), hs, U, 1 if mask_h else 0,
                                         _ptr(w_dl), _ptr(b_dl), ACTIVATIONS[act_dl], out_w.data_ptr(), _ptr(out_b),
                                         ACTIVATIONS[out_act], _cabi.LOSS_KINDS[loss] if train else 0, _ptr(targets), target_dtype,
                                         _ptr(sample_weight) if train else None, B, out.data_ptr(), _ptr(loss_buf) if train else None,
                                         _ptr(ds) if train else None, _ptr(dh) if train else None, dhs,
                                         *[_ptr(t) if train else None for t in (dw_out, db_out, dw_dl, db_dl, d_wide_bias)], _ptr(oob),
                                         _stream()),
        "mm_wide_deep_head_fwd_bwd")
    return out


def wide_bag_grad(bag, B: int, ds: torch.Tensor, out_ids: torch.Tensor, out_values: torch.Tensor) -> None:
    """One bag block's gradient as nnz (id, value) pairs for wide_rows_apply (mm_wide_bag_grad): out_ids (nnz,) int64, -1
    where no term of the forward sits; out_values (nnz,) fp32."""
    _dev(ds, "ds", torch.float32)
    if ds.numel() < B or not ds.is_contiguous():
        raise ValueError(f"ds must hold {B} contiguous values")
    arr, _ = _wide_bags([bag], B)
    nnz = arr[0].nnz
    if _dev(out_ids, "out_ids", torch.int64).numel() != nnz or not out_ids.is_contiguous():
        raise ValueError(f"out_ids must hold {nnz} contiguous int64 values")
    _vec(out_values, nnz, "out_values", "hold {n} contiguous float32 values")
    _cabi.check(_lib().mm_wide_bag_grad(arr, B, ds.data_ptr(), out_ids.data_ptr(), out_values.data_ptr(), _stream()), "mm_wide_bag_grad")
