"""Row-sparse optimizer steps for per-row parameter tables, such as the user encoders' long-term user vectors (DESIGN 4.18).

A table with one row per user (or per item) is touched a few thousand rows at a time; dae_optimizer_step would stream all of it and
its slots on every batch.  rows_step updates only the listed rows, lazily: rows not listed keep their slots as they are.
"""
from . import _cabi
from ._cabi import call


def rows_step(table, slot1, slot2, counts, rows, n, grad, opt, lr, momentum, stream):
    """One dae_rows_optimizer_step: rows rows[i] (int32 device tensor, -1: skip; distinct) of table [R, H] fp32 and of its slots
    (laid out as the table; None where opt has none) take one step of opt's rule from grad row i ([n, H] fp32).  counts (int32 [R],
    required for 'adam') counts each row's updates, and Adam's bias correction uses the row's own count."""
    call('dae_rows_optimizer_step', table.data_ptr(), table.stride(0), table.shape[1], rows.data_ptr(), n, grad.data_ptr(),
         grad.stride(0), _cabi.ptr(slot1), _cabi.ptr(slot2), _cabi.ptr(counts), _cabi.OPT[opt], lr, momentum, stream)
