"""Torch-tensor front end of the C-ABI (include/mm_b200.h).

PyTorch is used for device memory and streams only: every function here checks its
arguments, takes raw device pointers and calls one entry point of libmm_b200.so on the
current CUDA stream.  There is no CPU path — a CPU tensor is an error.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

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


def dlrm_gather_interact(weights, indices, slots, D: int, bottom: Optional[torch.Tensor], bottom_slot: int,
                         out: torch.Tensor, oob: Optional[torch.Tensor] = None) -> torch.Tensor:
    _dev(out, "out")
    B = out.shape[0]
    arr, n, dt = _table_array(weights, indices, [s * D for s in slots], B)
    o32, ostride, osplit, okp = _split_out_args(out)
    _cabi.check(
        _lib().mm_dlrm_gather_interact(arr, n, dt, B, D, _ptr(bottom),
                                       0 if bottom is None else _row_stride(_dev(bottom, "bottom", torch.float32), "bottom"),
                                       bottom_slot, o32, ostride, osplit, okp, _ptr(oob), _stream()),
        "mm_dlrm_gather_interact")
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


def dlrm_lookup_interact(weights, indices, slots, rows, D: int, bottom: Optional[torch.Tensor], bottom_slot: int,
                         out: torch.Tensor, oob: Optional[torch.Tensor] = None, peers=None, rank: int = 0,
                         world: int = 1, operand_rows: bool = False) -> torch.Tensor:
    """Fused lookup + interaction with per-table id widths and optional row-sharded tables
    (mm_dlrm_lookup_interact).  weights[t]: the (rows, D) table or this rank's shard; indices[t]: (B,) ids
    (any width, see index_bytes_of); rows[t]: GLOBAL row count; peers[t]: None (replicated) or the `world`
    device pointers of the shards as mapped in this process.  operand_rows=True (D = 64): `weights`, the peers' shards
    and `bottom` are bf16 split rows (rows, 2*D) = [hi | lo] (split_rows / mlp_tc(out_operand=...)); needs a split-bf16
    `out`."""
    _dev(out, "out")
    B = out.shape[0]
    n = len(weights)
    if not (len(indices) == n and len(slots) == n and len(rows) == n):
        raise ValueError("weights / indices / slots / rows length mismatch")
    arr = (_cabi.LookupTable * n)()
    keep = []
    wdt, wcols = (torch.bfloat16, 2 * D) if operand_rows else (torch.float32, D)
    if operand_rows and bottom is not None and (bottom.dtype != torch.bfloat16 or bottom.shape[1] != 2 * D):
        raise ValueError(f"operand_rows: bottom must be bf16 split rows (B, {2 * D})")
    for t in range(n):
        w = _dev(weights[t], f"weights[{t}]", wdt)
        ix = _dev(indices[t], f"indices[{t}]")
        if w.dim() != 2 or w.shape[1] != wcols or not w.is_contiguous():
            raise ValueError(f"weights[{t}] must be a contiguous (rows, {wcols}) {wdt} matrix")
        wb = index_bytes_of(ix)
        if ix.numel() != B * (3 if wb == 3 else 1) or not ix.is_contiguous():
            raise ValueError(f"indices[{t}] must be contiguous with {B} ids, got {tuple(ix.shape)}")
        arr[t].weights = w.data_ptr()
        arr[t].indices = ix.data_ptr()
        arr[t].rows = int(rows[t])
        arr[t].slot = int(slots[t])
        arr[t].idx_bytes = wb
        pt = None if peers is None else peers[t]
        if pt is not None:
            if len(pt) != world:
                raise ValueError(f"peers[{t}] must list {world} shard pointers")
            pa = (C.c_void_p * world)(*[int(x) for x in pt])
            keep.append(pa)
            arr[t].peer_weights_host = C.cast(pa, C.POINTER(C.c_void_p))
    o32, ostride, osplit, okp = _split_out_args(out)
    _cabi.check(
        _lib().mm_dlrm_lookup_interact(arr, n, B, D, rank, world, _ptr(bottom),
                                       0 if bottom is None else (_row_stride(_dev(bottom, "bottom", wdt), "bottom") // (2 if operand_rows else 1)),
                                       bottom_slot, o32, ostride, osplit, okp, _ptr(oob), 1 if operand_rows else 0, _stream()),
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
    id_dt = MM_I64
    if downscore:
        if pos_ids is None or neg_ids is None:
            raise ValueError("downscore_false_negatives requires positive and negative item ids")
        neg_ids = neg_ids.reshape(-1).contiguous()
        # reference: positive ids are cast to the negative ids' dtype (utils/tf_utils.py:136)
        pos_ids = pos_ids.reshape(-1).to(neg_ids.dtype).contiguous()
        id_dt = _idx_dtype(neg_ids, "neg_ids")
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
    id_dt = MM_I64
    if downscore:
        if pos_ids is None or neg_ids is None:
            raise ValueError("downscore_false_negatives requires positive and negative item ids")
        neg_ids = neg_ids.reshape(-1).contiguous()
        pos_ids = pos_ids.reshape(-1).to(neg_ids.dtype).contiguous()  # utils/tf_utils.py:136
        id_dt = _idx_dtype(neg_ids, "neg_ids")
    dev = q.device
    pos_logit = torch.empty((B, 1), dtype=torch.float32, device=dev)
    _cabi.check(_lib().mm_positive_scores(q.data_ptr(), pos.data_ptr(), B, D, _ptr(pos_prob), float(temperature),
                                          pos_logit.data_ptr(), 1, _stream()), "mm_positive_scores")
    qs = split_rows(q)
    ns = qs if neg.data_ptr() == q.data_ptr() else split_rows(neg)
    stats = torch.empty((B, 3), dtype=torch.float32, device=dev)
    nbytes = int(_lib().mm_catalog_workspace_bytes(B, N, 0))
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
    _cabi.check(
        _lib().mm_inbatch_softmax_ce(qs.data_ptr(), ns.data_ptr(), B, N, D, _ptr(pos_ids) if downscore else None,
                                     _ptr(neg_ids) if downscore else None, id_dt, int(bool(downscore)), float(false_neg_score),
                                     pos_logit.data_ptr(), _ptr(neg_prob), float(temperature), stats.data_ptr(), ws.data_ptr(),
                                     nbytes, _stream()),
        "mm_inbatch_softmax_ce")
    return stats


_CONCAT_DTYPES = {torch.int32: _cabi.MM_I32, torch.int64: _cabi.MM_I64, torch.float32: _cabi.MM_F32,
                  torch.float64: _cabi.MM_F64}


def concat_columns(pieces: Sequence[torch.Tensor], out: torch.Tensor, out_cols: Optional[Sequence[int]] = None,
                   max_width: int = 256) -> torch.Tensor:
    """out[:, out_cols[i] : out_cols[i]+w_i] = float32(pieces[i])  — (B,) pieces count as (B,1).

    Pieces must already be in the reference's sorted-name order (core/aggregation.py:54-66)."""
    _dev(out, "out", torch.float32)
    B = out.shape[0]
    stride = _row_stride(out, "out")
    flat = []
    col = 0
    for i, t in enumerate(pieces):
        _dev(t, f"pieces[{i}]")
        if t.dtype not in _CONCAT_DTYPES:
            raise TypeError(f"pieces[{i}]: unsupported dtype {t.dtype}")
        if t.dim() == 1:
            t = t.unsqueeze(1)
        if t.dim() != 2 or t.shape[0] != B or (t.shape[1] > 1 and t.stride(1) != 1):
            raise ValueError(f"pieces[{i}] must be (B,) or (B,w) with unit inner stride, got {tuple(t.shape)}")
        w = t.shape[1]
        oc = col if out_cols is None else int(out_cols[i])
        for c0 in range(0, w, max_width):  # split very wide pieces so a launch tile fits in smem
            flat.append((t.data_ptr() + c0 * t.element_size(), t.stride(0), min(max_width, w - c0),
                         _CONCAT_DTYPES[t.dtype], oc + c0))
        col = oc + w
    groups, cur, cur_w = [], [], 0
    for f in flat:
        if cur and (cur_w + f[2] > max_width or len(cur) == 64):
            groups.append(cur)
            cur, cur_w = [], 0
        cur.append(f)
        cur_w += f[2]
    if cur:
        groups.append(cur)
    for g in groups:
        arr = (_cabi.ConcatPiece * len(g))()
        for i, (ptr, sstride, w, dt, oc) in enumerate(g):
            arr[i].src, arr[i].src_stride, arr[i].width, arr[i].dtype, arr[i].out_col = ptr, sstride, w, dt, oc
        _cabi.check(_lib().mm_concat_columns(arr, len(g), B, out.data_ptr(), stride, _stream()), "mm_concat_columns")
    return out


def concat_split_supported(pieces: Sequence[torch.Tensor]) -> bool:
    """mm_concat_split handles up to 64 pieces and 320 padded columns in one launch."""
    width = sum(1 if t.dim() == 1 else int(t.shape[1]) for t in pieces)
    return 0 < len(pieces) <= 64 and tc_padded_k(width) <= 320 and all(t.dtype in _CONCAT_DTYPES for t in pieces)


def concat_split(pieces: Sequence[torch.Tensor], out: Optional[torch.Tensor] = None):
    """ConcatFeatures + bf16 split in one launch (mm_concat_split): returns (a_split (B, 2*Kp) bf16, K).
    Pieces in the reference's sorted-name order; (B,) pieces count as (B,1)."""
    flat, col = [], 0
    B = pieces[0].shape[0]
    for i, t in enumerate(pieces):
        _dev(t, f"pieces[{i}]")
        if t.dtype not in _CONCAT_DTYPES:
            raise TypeError(f"pieces[{i}]: unsupported dtype {t.dtype}")
        if t.dim() == 1:
            t = t.unsqueeze(1)
        if t.dim() != 2 or t.shape[0] != B or (t.shape[1] > 1 and t.stride(1) != 1):
            raise ValueError(f"pieces[{i}] must be (B,) or (B,w) with unit inner stride, got {tuple(t.shape)}")
        flat.append((t.data_ptr(), t.stride(0), int(t.shape[1]), _CONCAT_DTYPES[t.dtype], col))
        col += int(t.shape[1])
    K, Kp = col, tc_padded_k(col)
    if out is None:
        out = torch.empty((B, 2 * Kp), dtype=torch.bfloat16, device=pieces[0].device)
    _dev(out, "out", torch.bfloat16)
    if tuple(out.shape) != (B, 2 * Kp) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous ({B}, {2 * Kp}) bf16 matrix")
    arr = (_cabi.ConcatPiece * len(flat))()
    for i, (ptr, sstride, w, dt, oc) in enumerate(flat):
        arr[i].src, arr[i].src_stride, arr[i].width, arr[i].dtype, arr[i].out_col = ptr, sstride, w, dt, oc
    _cabi.check(_lib().mm_concat_split(arr, len(flat), B, out.data_ptr(), Kp, _stream()), "mm_concat_split")
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
    flat, col = [], 0
    B = pieces[0].shape[0]
    for i, t in enumerate(pieces):
        _dev(t, f"pieces[{i}]")
        if t.dim() == 1:
            t = t.unsqueeze(1)
        if t.dim() != 2 or t.shape[0] != B or (t.shape[1] > 1 and t.stride(1) != 1):
            raise ValueError(f"pieces[{i}] must be (B,) or (B,w) with unit inner stride, got {tuple(t.shape)}")
        flat.append((t.data_ptr(), t.stride(0), int(t.shape[1]), _CONCAT_DTYPES[t.dtype], col))
        col += int(t.shape[1])
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
    arr = (_cabi.ConcatPiece * len(flat))()
    for i, (ptr, sstride, w, dt, oc) in enumerate(flat):
        arr[i].src, arr[i].src_stride, arr[i].width, arr[i].dtype, arr[i].out_col = ptr, sstride, w, dt, oc
    _cabi.check(
        _lib().mm_tower2_small(arr, len(flat), B, w1_split.data_ptr(), N1, _ptr(bias1), ACTIVATIONS[act1], w2_split.data_ptr(), N2,
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
             xres: Optional[torch.Tensor] = None) -> None:
    """One tensor-core dense layer (mm_dense_tc); see include/mm_b200.h."""
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
    nbytes = int(_lib().mm_catalog_workspace_bytes(B, n_items, k))
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
    _cabi.check(
        _lib().mm_catalog_score(split_rows(q).data_ptr(), B, D, e_split.data_ptr(), n_items, _ptr(bias), _ptr(targets), id_dt,
                                _ptr(stats), k, _ptr(scores), _ptr(ids), ws.data_ptr(), nbytes, _stream()),
        "mm_catalog_score")
    return stats, scores, ids


def mlp_forward(x: torch.Tensor, kernels: Sequence[torch.Tensor], biases: Sequence[Optional[torch.Tensor]],
                acts: Sequence[Optional[str]], out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """MLPBlock in ONE C call over fp32 Keras-layout kernels (mm_mlp_forward): the bf16 splits of the input,
    the weights and the intermediate activations live in a workspace allocated here."""
    _dev(x, "x", torch.float32)
    M, K = x.shape
    n = len(kernels)
    widths = [int(k.shape[1]) for k in kernels]
    kk = K
    for l, kern in enumerate(kernels):
        _dev(kern, f"kernels[{l}]", torch.float32)
        if kern.dim() != 2 or kern.shape[0] != kk or not kern.is_contiguous():
            raise ValueError(f"kernels[{l}] must be a contiguous ({kk}, units) matrix, got {tuple(kern.shape)}")
        if biases[l] is not None:
            _dev(biases[l], f"biases[{l}]", torch.float32)
        kk = widths[l]
    if out is None:
        out = torch.empty((M, widths[-1]), dtype=torch.float32, device=x.device)
    wd = (C.c_int * n)(*widths)
    need = int(_lib().mm_mlp_workspace_bytes(M, K, n, wd))
    if need < 0:
        raise ValueError("mm_mlp_workspace_bytes rejected the tower (1..8 layers, positive widths)")
    ws = torch.empty(max(need, 256), dtype=torch.uint8, device=x.device)
    kp = (C.c_void_p * n)(*[k.data_ptr() for k in kernels])
    bp = (C.c_void_p * n)(*[_ptr(b) for b in biases])
    ac = (C.c_int * n)(*[ACTIVATIONS[a] for a in acts])
    _cabi.check(_lib().mm_mlp_forward(x.data_ptr(), M, K, _row_stride(x, "x"), n, kp, bp, wd, ac, out.data_ptr(),
                                      _row_stride(out, "out"), ws.data_ptr(), need, _stream()), "mm_mlp_forward")
    return out


def cross_forward(x0: torch.Tensor, kernels: Sequence[torch.Tensor], biases: Sequence[Optional[torch.Tensor]],
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """CrossBlock stack in ONE C call (mm_cross_forward): x_{l+1} = x0 * (x_l W_l + b_l) + x_l."""
    _dev(x0, "x0", torch.float32)
    M, d = x0.shape
    depth = len(kernels)
    for l, kern in enumerate(kernels):
        _dev(kern, f"kernels[{l}]", torch.float32)
        if tuple(kern.shape) != (d, d) or not kern.is_contiguous():
            raise ValueError(f"kernels[{l}] must be a contiguous ({d}, {d}) matrix")
    if out is None:
        out = torch.empty((M, d), dtype=torch.float32, device=x0.device)
    need = int(_lib().mm_cross_workspace_bytes(M, d, depth))
    if need < 0:
        raise ValueError(f"Number of cross layers (depth) should be positive but is {depth}.")
    ws = torch.empty(max(need, 256), dtype=torch.uint8, device=x0.device)
    kp = (C.c_void_p * depth)(*[k.data_ptr() for k in kernels])
    bp = (C.c_void_p * depth)(*[_ptr(b) for b in biases])
    _cabi.check(_lib().mm_cross_forward(x0.data_ptr(), M, d, _row_stride(x0, "x0"), depth, kp, bp, out.data_ptr(),
                                        _row_stride(out, "out"), ws.data_ptr(), need, _stream()), "mm_cross_forward")
    return out


def mlp_tc_supported(K: int, widths: Sequence[int], head: bool = False) -> bool:
    """True when mm_mlp_tc can run the tower (mm_mlp_tc_supported): 2..4 layers, every width <= 128, head only
    after <= 32 units, resident weights of layers 2..n + two layer-1 pipeline stages within shared memory."""
    n = len(widths)
    if n < 2 or n > 4:
        return False
    wd = (C.c_int * n)(*[int(w) for w in widths])
    return bool(_lib().mm_mlp_tc_supported(int(K), n, wd, 1 if head else 0))


def mlp_tc(a_split: torch.Tensor, K: int, w_splits: Sequence[torch.Tensor], widths: Sequence[int],
           biases: Sequence[Optional[torch.Tensor]], acts: Sequence[Optional[str]], out: Optional[torch.Tensor] = None,
           head_w: Optional[torch.Tensor] = None, head_b: float = 0.0, head_act: Optional[str] = None,
           head_out: Optional[torch.Tensor] = None, out_operand: Optional[torch.Tensor] = None):
    """Whole MLP tower in one launch (mm_mlp_tc): layer 1 from the split-bf16 rows `a_split`, layers 2..n on
    chip (activations stay in registers).  out: (M, widths[-1]) fp32 and/or head_out: (M, 1); out_operand:
    (M, 2*widths[-1]) bf16 split rows [hi | lo] for the interaction kernel (mm_mlp_tc_operand_out)."""
    n = len(widths)
    if not (len(w_splits) == len(biases) == len(acts) == n):
        raise ValueError("mlp_tc: w_splits / widths / biases / acts must have one entry per layer")
    _dev(a_split, "a_split", torch.bfloat16)
    M = a_split.shape[0]
    if a_split.dim() != 2 or a_split.shape[1] != 2 * tc_padded_k(K) or not a_split.is_contiguous():
        raise ValueError(f"a_split must be a contiguous (M, {2 * tc_padded_k(K)}) bf16 matrix")
    k = K
    for l in range(n):
        _dev(w_splits[l], f"w_split[{l}]", torch.bfloat16)
        if tuple(w_splits[l].shape) != (tc_padded_n(int(widths[l])), 2 * tc_padded_k(k)) or not w_splits[l].is_contiguous():
            raise ValueError(f"w_split[{l}] must be the mm_split_weights layout of a ({k}, {widths[l]}) kernel")
        if biases[l] is not None:
            _dev(biases[l], f"bias[{l}]", torch.float32)
            if biases[l].numel() != int(widths[l]):
                raise ValueError(f"bias[{l}] must hold {widths[l]} values")
        k = int(widths[l])
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
    wp = (C.c_void_p * n)(*[w.data_ptr() for w in w_splits])
    bp = (C.c_void_p * n)(*[_ptr(b) for b in biases])
    wd = (C.c_int * n)(*[int(w) for w in widths])
    ac = (C.c_int * n)(*[ACTIVATIONS[a] for a in acts])
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


def bce_head_fwd_bwd(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], targets: torch.Tensor,
                     loss_sum: torch.Tensor, dx: Optional[torch.Tensor], dw: torch.Tensor, db: Optional[torch.Tensor],
                     mask_relu: bool = True, sample_weight: Optional[torch.Tensor] = None,
                     logits: Optional[torch.Tensor] = None) -> None:
    """Dense(K -> 1) + sigmoid + binary cross-entropy, forward and backward (mm_bce_head_fwd_bwd).  loss_sum (1,), dw (K,),
    db (1,) are ACCUMULATED; dx (M, K) is written (zeroed where x <= 0 when mask_relu)."""
    _dev(x, "x", torch.float32), _dev(w, "w", torch.float32), _dev(targets, "targets"), _dev(loss_sum, "loss_sum", torch.float32)
    _dev(dw, "dw", torch.float32)
    M, K = x.shape
    if w.numel() != K or dw.numel() != K or not w.is_contiguous() or not dw.is_contiguous():
        raise ValueError(f"w and dw must hold {K} contiguous values")
    if targets.numel() != M or not targets.is_contiguous() or targets.dtype not in _TARGET_DTYPES:
        raise ValueError(f"targets must be {M} contiguous int32 / int64 / float32 / float64 values")
    if sample_weight is not None and (sample_weight.numel() != M or sample_weight.dtype != torch.float32 or not sample_weight.is_contiguous()):
        raise ValueError("sample_weight must be (M,) contiguous float32")
    if logits is not None and (logits.numel() != M or logits.dtype != torch.float32 or not logits.is_contiguous()):
        raise ValueError("logits must be (M,) contiguous float32")
    _cabi.check(
        _lib().mm_bce_head_fwd_bwd(x.data_ptr(), M, K, _row_stride(x, "x"), w.data_ptr(), _ptr(bias), targets.data_ptr(),
                                   _TARGET_DTYPES[targets.dtype], _ptr(sample_weight), _ptr(logits), loss_sum.data_ptr(), _ptr(dx),
                                   0 if dx is None else _row_stride(_dev(dx, "dx", torch.float32), "dx"), 1 if mask_relu else 0,
                                   dw.data_ptr(), _ptr(db), _stream()),
        "mm_bce_head_fwd_bwd")


def dense_wgrad(x: torch.Tensor, dz: torch.Tensor, dw: torch.Tensor, db: Optional[torch.Tensor]) -> None:
    """dw (K, N) += x^T dz;  db (N,) += column sums of dz  (mm_dense_wgrad; accumulated)."""
    _dev(x, "x", torch.float32), _dev(dz, "dz", torch.float32), _dev(dw, "dw", torch.float32)
    M, K = x.shape
    N = dz.shape[1]
    if dz.shape[0] != M or tuple(dw.shape) != (K, N) or not dw.is_contiguous():
        raise ValueError(f"dz must be ({M}, N) and dw a contiguous ({K}, {N}) matrix")
    if db is not None and (_dev(db, "db", torch.float32).numel() != N or not db.is_contiguous()):
        raise ValueError(f"db must hold {N} contiguous values")
    _cabi.check(_lib().mm_dense_wgrad(x.data_ptr(), M, K, _row_stride(x, "x"), dz.data_ptr(), N, _row_stride(dz, "dz"), dw.data_ptr(),
                                      _ptr(db), _stream()), "mm_dense_wgrad")


def dense_wgrad_split(x_split: torch.Tensor, K: int, dz: torch.Tensor, dw: torch.Tensor, db: Optional[torch.Tensor]) -> None:
    """dense_wgrad with x given as the split-bf16 operand (M, 2*Kp) the forward layer consumed (mm_dense_wgrad_split)."""
    _dev(x_split, "x_split", torch.bfloat16), _dev(dz, "dz", torch.float32), _dev(dw, "dw", torch.float32)
    M = x_split.shape[0]
    Kp = tc_padded_k(K)
    N = dz.shape[1]
    if tuple(x_split.shape) != (M, 2 * Kp) or not x_split.is_contiguous():
        raise ValueError(f"x_split must be a contiguous bf16 ({M}, {2 * Kp}) matrix")
    if dz.shape[0] != M or tuple(dw.shape) != (K, N) or not dw.is_contiguous():
        raise ValueError(f"dz must be ({M}, N) and dw a contiguous ({K}, {N}) matrix")
    if db is not None and (_dev(db, "db", torch.float32).numel() != N or not db.is_contiguous()):
        raise ValueError(f"db must hold {N} contiguous values")
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
    arr = (_cabi.LookupTable * n)()
    gp = (C.c_void_p * n)()
    gstride = None
    wdt, wcols = (torch.bfloat16, 2 * D) if operand_rows else (torch.float32, D)
    for t in range(n):
        w = _dev(weights[t], f"weights[{t}]", wdt)
        ix = _dev(indices[t], f"indices[{t}]")
        if w.dim() != 2 or w.shape[1] != wcols or not w.is_contiguous():
            raise ValueError(f"weights[{t}] must be a contiguous (rows, {wcols}) {wdt} matrix")
        wb = index_bytes_of(ix)
        if ix.numel() != B * (3 if wb == 3 else 1) or not ix.is_contiguous():
            raise ValueError(f"indices[{t}] must be contiguous with {B} ids")
        arr[t].weights, arr[t].indices, arr[t].rows, arr[t].slot, arr[t].idx_bytes = w.data_ptr(), ix.data_ptr(), int(rows[t]), int(slots[t]), wb
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
    arr = (_cabi.LookupTable * n)()
    for t in range(n):
        w = _dev(weights[t], f"weights[{t}]", torch.float32)
        ix = _dev(indices[t], f"indices[{t}]")
        if w.dim() != 2 or w.shape[1] != D or not w.is_contiguous():
            raise ValueError(f"weights[{t}] must be a contiguous (rows, {D}) float32 matrix")
        wb = index_bytes_of(ix)
        if ix.numel() != B * (3 if wb == 3 else 1) or not ix.is_contiguous():
            raise ValueError(f"indices[{t}] must be contiguous with {B} ids")
        arr[t].weights, arr[t].indices, arr[t].rows, arr[t].slot, arr[t].idx_bytes = w.data_ptr(), ix.data_ptr(), w.shape[0], t, wb
    woff = (C.c_int64 * n)(*[int(o) for o in wide_offsets])
    m = len(cont)
    if len(cont_offsets) != m:
        raise ValueError("cont / cont_offsets length mismatch")
    carr = (_cabi.ConcatPiece * max(m, 1))()
    for c, t in enumerate(cont):
        _dev(t, f"cont[{c}]")
        if t.dtype not in _CONCAT_DTYPES or t.numel() != B:
            raise ValueError(f"cont[{c}] must hold {B} int32 / int64 / float32 / float64 values")
        v = t.reshape(-1)
        carr[c].src, carr[c].src_stride, carr[c].width, carr[c].dtype, carr[c].out_col = v.data_ptr(), v.stride(0), 1, _CONCAT_DTYPES[t.dtype], c
    coff = (C.c_int64 * max(m, 1))(*[int(o) for o in cont_offsets])
    if addend is not None and (_dev(addend, "addend", torch.float32).numel() != B):
        raise ValueError(f"addend must hold {B} values")
    a_stride = 0 if addend is None else (addend.stride(0) if addend.dim() >= 1 else 1)
    _cabi.check(
        _lib().mm_deepfm_head(arr, woff, n, B, D, carr, coff, m, wide_kernel.data_ptr(), _ptr(wide_bias), _ptr(addend), a_stride,
                              _ptr(out_w), _ptr(out_b), ACTIVATIONS[out_act], out.data_ptr(), _ptr(oob), _stream()),
        "mm_deepfm_head")
    return out
