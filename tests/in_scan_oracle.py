"""Reference results of `<column> [NOT] IN (<literal>, ...)` TableScans. TEST INFRASTRUCTURE ONLY.

The rows are decoded by the CPU oracle (oracle_lib.decode_segment; string rows from the host dictionaries) and evaluated
by tests/cpp/in_scan_oracle.cpp, a row-by-row restatement of ExpressionEvaluator::_evaluate_in_expression with the real
std::equal_to in C++'s common type. It uses neither the normalised intervals nor dictionary bitmaps.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as orc
from hyrise_b200 import capi
from hyrise_b200.device import ROW_ID_DTYPE, InList, literal_type
from hyrise_b200.storage import NUMPY_TYPES, Table

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBRARY_PATH = os.path.join(REPO, "build", "libin_scan_oracle.so")
NULL_ELEMENT = -1

_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIBRARY_PATH):
            subprocess.check_call(["make", "-C", REPO, "build/libin_scan_oracle.so"])
        lib = C.CDLL(LIBRARY_PATH)
        lib.ino_scan.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int32,
                                 C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = lib
    return _lib


def _strings(values) -> tuple[bytes | None, np.ndarray]:
    values = [bytes(value) for value in values]
    offsets = np.zeros(len(values) + 1, dtype=np.uint64)
    if values:
        offsets[1:] = np.cumsum([len(value) for value in values])
    return b"".join(values) or None, offsets


def selected(column_type: int, values, nulls, elements, negated: bool) -> np.ndarray:
    """Per row: is `value [NOT] IN (elements)` non-zero and not NULL. `values`: an array of the column type, or bytes per
    row for a string column; `elements`: Python / numpy literals, typed as device.literal_type types them."""
    rows = len(values)
    nulls = np.ascontiguousarray(np.asarray(nulls, dtype=bool).astype(np.uint8)) if rows else np.zeros(1, np.uint8)
    typed = [literal_type(element) for element in elements]
    types = np.array([NULL_ELEMENT if t is None else t for t, _ in typed] or [0], dtype=np.int32)
    literals = capi.literal_array([(t, v) for t, v in typed if t not in (None, capi.TYPE_STRING)])
    numeric_index = iter(range(len(typed)))
    element_values = (capi.Value * max(len(typed), 1))()
    for index, (data_type, _) in enumerate(typed):
        if data_type not in (None, capi.TYPE_STRING):
            element_values[index] = literals[next(numeric_index)].value
    element_chars, element_offsets = _strings([v if t == capi.TYPE_STRING else b"" for t, v in typed])
    out = np.zeros(max(rows, 1), dtype=np.uint8)
    keep = []
    if column_type == capi.TYPE_STRING:
        chars, offsets = _strings(values)
        arguments = (None, chars, offsets.ctypes.data)
    else:
        array = np.ascontiguousarray(values, dtype=NUMPY_TYPES[column_type])
        keep.append(array)
        arguments = (array.ctypes.data, None, None)
    status = load().ino_scan(column_type, *arguments, nulls.ctypes.data, rows, int(negated), len(typed),
                             types.ctypes.data, element_values, element_chars, element_offsets.ctypes.data,
                             out.ctypes.data)
    if status != 0:
        raise capi.HyriseB200Error(status, "IN oracle rejected the column")
    return out[:rows].astype(bool)


def null_row_selected(column_type: int, elements, negated: bool) -> bool:
    """Whether a NULL value (a NULL row, or a NULL_ROW_ID of an outer join) is selected."""
    values = [b""] if column_type == capi.TYPE_STRING else np.zeros(1, dtype=NUMPY_TYPES[column_type])
    return bool(selected(column_type, values, [True], elements, negated)[0])


def segment_rows(segment) -> tuple[object, np.ndarray]:
    """Decoded values (bytes per row for strings) and the null mask of one segment."""
    if segment.data_type == capi.TYPE_STRING:
        return [bytes(value) for value in segment.decode()], segment.null_mask()
    values, nulls = orc.decode_segment(segment)
    return values, nulls.astype(bool)


def chunk_matches(table: Table, in_list: InList) -> list[np.ndarray]:
    column_type = table.column_definitions[in_list.column_id].data_type
    negated = in_list.condition == capi.PRED_NOT_IN
    out = []
    for chunk in table.chunks:
        values, nulls = segment_rows(chunk.segments[in_list.column_id])
        out.append(selected(column_type, values, nulls, in_list.elements, negated))
    return out


def table_scan_in(table: Table, in_list: InList, input_filter: orc.HostPosList | None = None,
                  ascending: bool = True) -> orc.HostPosList:
    """The scan's PosList: per chunk the selected RowIDs in row order; with `input_filter`, the selected entries of the
    filter in its order (per chunk when `ascending`, else one list; a NULL_ROW_ID reads as NULL)."""
    matches = chunk_matches(table, in_list)
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
    valid = chunk_ids != capi.INVALID_VALUE_ID
    keep = np.zeros(len(chunk_ids), dtype=bool)
    keep[valid] = flat[starts[chunk_ids[valid]] + input_filter.row_ids["chunk_offset"][valid].astype(np.int64)]
    column_type = table.column_definitions[in_list.column_id].data_type
    keep[~valid] = null_row_selected(column_type, in_list.elements, in_list.condition == capi.PRED_NOT_IN)
    rows = input_filter.row_ids[keep].copy()
    if not ascending:
        return orc.HostPosList(rows, np.array([0, len(rows)], dtype=np.uint64))
    counts = np.bincount(rows["chunk_id"].astype(np.int64), minlength=table.chunk_count) if len(rows) else \
        np.zeros(table.chunk_count, dtype=np.int64)
    return orc.HostPosList(rows, np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64))
