"""Reference results of column-vs-column TableScans (ColumnVsColumnTableScanImpl). TEST INFRASTRUCTURE ONLY.

Numeric pairs: the segments are decoded by the CPU oracle (oracle_lib.decode_segment) and compared row by row by
tests/cpp/column_scan_oracle.cpp, which uses the real std::less<void> and friends, so C++ applies its own conversion
rules. String pairs: the row values as Python bytes, compared with Python's bytes ordering (unsigned bytes, a proper
prefix first: std::string::compare). Neither path uses a dictionary translation.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as orc
from hyrise_b200 import capi
from hyrise_b200.device import ROW_ID_DTYPE, ColumnComparison
from hyrise_b200.storage import NUMPY_TYPES, Table

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBRARY_PATH = os.path.join(REPO, "build", "libcolumn_scan_oracle.so")

_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIBRARY_PATH):
            subprocess.check_call(["make", "-C", REPO, "build/libcolumn_scan_oracle.so"])
        lib = C.CDLL(LIBRARY_PATH)
        lib.csc_scan_decoded.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_uint64,
                                         C.c_int32, C.c_void_p]
        _lib = lib
    return _lib


def numeric_matches(left_type: int, left_values, left_nulls, right_type: int, right_values, right_nulls,
                    condition: int) -> np.ndarray:
    """Per row: neither side NULL and `left <condition> right` under C++'s comparators."""
    # a string side arrives as value-IDs: the restatement rejects it ("Trying to compare strings and non-strings")
    left = np.ascontiguousarray(left_values, dtype=NUMPY_TYPES.get(left_type, np.uint32))
    right = np.ascontiguousarray(right_values, dtype=NUMPY_TYPES.get(right_type, np.uint32))
    left_nulls = np.ascontiguousarray(left_nulls, dtype=np.uint8)
    right_nulls = np.ascontiguousarray(right_nulls, dtype=np.uint8)
    rows = len(left)
    assert len(right) == rows and len(left_nulls) == rows and len(right_nulls) == rows
    out = np.zeros(max(rows, 1), dtype=np.uint8)
    status = load().csc_scan_decoded(left_type, left.ctypes.data, left_nulls.ctypes.data, right_type, right.ctypes.data,
                                     right_nulls.ctypes.data, rows, condition, out.ctypes.data)
    if status != 0:
        raise capi.HyriseB200Error(status, "column-vs-column oracle rejected the pair")
    return out[:rows].astype(bool)


_STRING_COMPARATORS = {
    capi.PRED_EQUALS: lambda a, b: a == b,
    capi.PRED_NOT_EQUALS: lambda a, b: a != b,
    capi.PRED_LESS_THAN: lambda a, b: a < b,
    capi.PRED_LESS_THAN_EQUALS: lambda a, b: a <= b,
    capi.PRED_GREATER_THAN: lambda a, b: a > b,
    capi.PRED_GREATER_THAN_EQUALS: lambda a, b: a >= b,
}


def string_matches(left: list, right: list, condition: int) -> np.ndarray:
    """Per row: both values are bytes (None = NULL) and `left <condition> right` as std::string::compare orders them."""
    compare = _STRING_COMPARATORS[condition]
    return np.array([a is not None and b is not None and compare(bytes(a), bytes(b)) for a, b in zip(left, right)],
                    dtype=bool)


def chunk_matches(table: Table, comparison: ColumnComparison, strings: dict | None = None) -> list[np.ndarray]:
    """Match flags of every row, per chunk. `strings`: column id -> the column's row values (bytes or None), in row order,
    for string pairs."""
    left_type = table.column_definitions[comparison.left_column_id].data_type
    right_type = table.column_definitions[comparison.right_column_id].data_type
    per_chunk = []
    begin = 0
    for chunk in table.chunks:
        rows = chunk.size
        if left_type == capi.TYPE_STRING and right_type == capi.TYPE_STRING:
            left = strings[comparison.left_column_id][begin: begin + rows]
            right = strings[comparison.right_column_id][begin: begin + rows]
            per_chunk.append(string_matches(left, right, comparison.condition))
        else:
            left_values, left_nulls = orc.decode_segment(chunk.segments[comparison.left_column_id])
            right_values, right_nulls = orc.decode_segment(chunk.segments[comparison.right_column_id])
            per_chunk.append(numeric_matches(left_type, left_values, left_nulls, right_type, right_values, right_nulls,
                                             comparison.condition))
        begin += rows
    return per_chunk


def table_scan_columns(table: Table, comparison: ColumnComparison, input_filter: orc.HostPosList | None = None,
                       ascending: bool = True, strings: dict | None = None) -> orc.HostPosList:
    """The scan's PosList: per chunk the matching RowIDs in row order; with `input_filter`, the matching entries of the
    filter in its order (per chunk when `ascending`, else one list; a NULL_ROW_ID never matches)."""
    matches = chunk_matches(table, comparison, strings)
    if input_filter is None:
        lists = []
        for chunk_id, flags in enumerate(matches):
            part = np.zeros(int(flags.sum()), dtype=ROW_ID_DTYPE)
            part["chunk_id"] = chunk_id
            part["chunk_offset"] = np.flatnonzero(flags)
            lists.append(part)
        rows = np.concatenate(lists) if lists else np.zeros(0, dtype=ROW_ID_DTYPE)
        offsets = np.concatenate([[0], np.cumsum([len(part) for part in lists])]).astype(np.uint64)
        return orc.HostPosList(rows, offsets)
    flat = np.concatenate(matches) if matches else np.zeros(0, dtype=bool)
    starts = np.concatenate([[0], np.cumsum([len(flags) for flags in matches])]).astype(np.int64)
    chunk_ids = input_filter.row_ids["chunk_id"].astype(np.int64)
    valid = chunk_ids != capi.INVALID_VALUE_ID  # NULL_ROW_ID (outer join): never matches
    keep = np.zeros(len(chunk_ids), dtype=bool)
    keep[valid] = flat[starts[chunk_ids[valid]] + input_filter.row_ids["chunk_offset"][valid].astype(np.int64)]
    rows = input_filter.row_ids[keep].copy()
    if not ascending:
        return orc.HostPosList(rows, np.array([0, len(rows)], dtype=np.uint64))
    counts = np.bincount(rows["chunk_id"].astype(np.int64), minlength=table.chunk_count) if len(rows) else \
        np.zeros(table.chunk_count, dtype=np.int64)
    return orc.HostPosList(rows, np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64))
