"""Every C entry point that reads packed id columns rejects a malformed one before launching anything
(include/mm_b200.h, mm_lookup_table): a width outside {1, 2, 3, 4, 8} or too narrow for the table's rows is
MM_ERR_ARG, a 4- or 8-byte id array off its alignment is MM_ERR_ALIGN.

The calls pass made-up device addresses that the host never dereferences.  They run only where no kernel can be
launched, so a library that failed to reject the input would return a CUDA error instead of touching memory."""
import ctypes as C

import pytest
import torch

from models_b200 import _cabi

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="passes fake device pointers: CPU-only check")

MM_ERR_ARG, MM_ERR_ALIGN = -1, -3
BASE = 0x7F0000000000  # 256-byte aligned fake device address


def _ptr(k: int, misalign: int = 0) -> int:
    return BASE + 0x10000 * k + misalign


def _lookup_table(slot: int, rows: int, idx_bytes: int, misalign: int = 0) -> _cabi.LookupTable:
    t = _cabi.LookupTable()
    t.weights, t.indices, t.rows, t.slot, t.idx_bytes = _ptr(1 + 2 * slot), _ptr(2 + 2 * slot, misalign), rows, slot, idx_bytes
    return t


def _sparse_rows_apply(idx_bytes: int, misalign: int = 0) -> int:
    s = _cabi.SparseTable()
    s.weights, s.rows, s.indices, s.idx_bytes = _ptr(1), 100, _ptr(2, misalign), idx_bytes
    s.grad_rows, s.rep_map = _ptr(3), _ptr(4)
    arr = (_cabi.SparseTable * 1)(s)
    return _cabi.load().mm_sparse_rows_apply(arr, 1, 8, 16, _cabi.OPTIMIZERS["sgd"], _ptr(5), None)


def test_deepfm_head_rejects_misaligned_int32_ids():
    arr = (_cabi.LookupTable * 1)(_lookup_table(0, 100, 4, misalign=2))
    woff = (C.c_int64 * 1)(0)
    rc = _cabi.load().mm_deepfm_head(arr, woff, 1, 4, 16, None, None, 0, _ptr(9), None, None, 0, None, None, 0, _ptr(10),
                                     None, None)
    assert rc == MM_ERR_ALIGN and "misaligned ids" in _cabi.last_error()


def test_sparse_rows_apply_rejects_unknown_id_width():
    assert _sparse_rows_apply(5) == MM_ERR_ARG and "idx_bytes" in _cabi.last_error()


def test_sparse_rows_apply_rejects_misaligned_int64_ids():
    assert _sparse_rows_apply(8, misalign=4) == MM_ERR_ALIGN and "misaligned ids" in _cabi.last_error()


def test_interact_backward_rejects_ids_too_narrow_for_the_table():
    arr = (_cabi.LookupTable * 2)(_lookup_table(0, 300, 1), _lookup_table(1, 300, 4))
    grads = (C.c_void_p * 2)()
    rc = _cabi.load().mm_dlrm_interact_backward(arr, 2, 8, 64, None, 0, -1, 0, _ptr(9), 4, grads, 64, None, 0, 0, 0, None)
    assert rc == MM_ERR_ARG and "do not fit" in _cabi.last_error()
