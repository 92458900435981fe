"""Reference results of JoinHash with secondary predicates (hyb_join_hash_predicates). TEST INFRASTRUCTURE ONLY.

A predicate `(build column, probe column, condition)` reads `build value <condition> probe value`, the direction of
MultiPredicateJoinEvaluator(build_table, probe_table, ...). FieldComparator::compare (multi_predicate_join_evaluator.cpp)
fails on a NULL on either side and otherwise compares in the two types' std::common_type: int x int in int64, int x float
in float, anything with a double in double. numpy's casts and comparisons are C's, so NaN fails all but !=, -0.0 == +0.0,
and an int64 rounds once to the nearest float or double.

- `nested_loop` restates JoinVerification (join_verification.cpp:50-213) with the predicates, in numpy: an unordered
  multiset.
- `ordered` is orc_join_hash_predicates (tests/cpp/join_predicates_oracle.cpp): JoinHashImpl with a
  MultiPredicateJoinEvaluator restated in C++ on the CPU oracle's join steps, comparing with the std functors on the
  columns' own types. It gives the exact output: pairs, order and partition offsets.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as orc
from helpers import NULL_ROW
from hyrise_b200 import capi
from hyrise_b200.device import ROW_ID_DTYPE
from hyrise_b200.storage import Table

INVALID_CHUNK_ID = 0xFFFFFFFF
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBRARY_PATH = os.path.join(REPO, "build", "libjoin_predicates_oracle.so")
_lib = None
SEMI_OR_ANTI = (capi.JOIN_SEMI, capi.JOIN_ANTI_NULL_AS_TRUE, capi.JOIN_ANTI_NULL_AS_FALSE)

_COMPARATORS = {
    capi.PRED_EQUALS: np.equal,
    capi.PRED_NOT_EQUALS: np.not_equal,
    capi.PRED_LESS_THAN: np.less,
    capi.PRED_LESS_THAN_EQUALS: np.less_equal,
    capi.PRED_GREATER_THAN: np.greater,
    capi.PRED_GREATER_THAN_EQUALS: np.greater_equal,
}
FLIPPED = {capi.PRED_EQUALS: capi.PRED_EQUALS, capi.PRED_NOT_EQUALS: capi.PRED_NOT_EQUALS,
           capi.PRED_LESS_THAN: capi.PRED_GREATER_THAN, capi.PRED_LESS_THAN_EQUALS: capi.PRED_GREATER_THAN_EQUALS,
           capi.PRED_GREATER_THAN: capi.PRED_LESS_THAN, capi.PRED_GREATER_THAN_EQUALS: capi.PRED_LESS_THAN_EQUALS}


def flip(predicates):
    """The predicates of the swapped join (join_hash.cpp:158-165)."""
    return [(probe_column, build_column, FLIPPED[condition]) for build_column, probe_column, condition in predicates]


def common_dtype(a: int, b: int):
    if capi.TYPE_FLOAT64 in (a, b):
        return np.float64
    if capi.TYPE_FLOAT32 in (a, b):
        return np.float32
    return np.int64


def _values_at(table: Table, column: int, row_ids: np.ndarray, dtype):
    """Values (cast to `dtype`) and NULL flags of a column at RowIDs; NULL_ROW_ID reads as NULL."""
    values, nulls = table.column_values(column)
    starts = np.zeros(table.chunk_count + 1, dtype=np.int64)
    starts[1:] = np.cumsum([chunk.size for chunk in table.chunks])
    chunk_ids = row_ids["chunk_id"].astype(np.int64)
    invalid = row_ids["chunk_id"] == INVALID_CHUNK_ID
    flat = np.where(invalid, 0, starts[np.where(invalid, 0, chunk_ids)] + row_ids["chunk_offset"].astype(np.int64))
    if len(values) == 0:
        return np.zeros(len(row_ids), dtype=dtype), np.ones(len(row_ids), dtype=bool)
    return values[flat].astype(dtype), nulls[flat] | invalid


def side_rows(table: Table, column: int, filter_list=None) -> list:
    """[(RowID tuple, key or None)] of a join side in position order; a NULL_ROW_ID of the filter has a NULL key."""
    if filter_list is not None:
        row_ids = filter_list.row_ids
    else:
        row_ids = np.zeros(table.row_count, dtype=ROW_ID_DTYPE)
        row_ids["chunk_id"] = np.repeat(np.arange(table.chunk_count), [chunk.size for chunk in table.chunks])
        row_ids["chunk_offset"] = np.concatenate([np.arange(chunk.size) for chunk in table.chunks]) if table.chunks else []
    keys, nulls = _values_at(table, column, row_ids, np.int64)
    return [((int(r["chunk_id"]), int(r["chunk_offset"])), None if null else int(key))
            for r, key, null in zip(row_ids, keys, nulls)]


def passes(build: Table, probe: Table, predicates, build_rows: np.ndarray, probe_rows: np.ndarray) -> np.ndarray:
    """Per (build RowID, probe RowID) pair: every predicate holds."""
    ok = np.ones(len(build_rows), dtype=bool)
    for build_column, probe_column, condition in predicates:
        dtype = common_dtype(build.column_definitions[build_column].data_type,
                             probe.column_definitions[probe_column].data_type)
        a, a_null = _values_at(build, build_column, build_rows, dtype)
        b, b_null = _values_at(probe, probe_column, probe_rows, dtype)
        with np.errstate(invalid="ignore"):
            ok &= _COMPARATORS[condition](a, b) & ~a_null & ~b_null
    return ok


def _row_array(rows) -> np.ndarray:
    out = np.zeros(len(rows), dtype=ROW_ID_DTYPE)
    if rows:
        out["chunk_id"], out["chunk_offset"] = zip(*rows)
    return out


def nested_loop(build: Table, build_column: int, probe: Table, probe_column: int, mode: int, predicates,
                build_filter=None, probe_filter=None):
    """JoinVerification with secondary predicates: multiset of (build RowID, probe RowID) pairs, or probe RowIDs for
    Semi / Anti."""
    build_rows = side_rows(build, build_column, build_filter)
    probe_rows = side_rows(probe, probe_column, probe_filter)
    build_keys = {}
    for row_id, key in build_rows:
        if key is not None:
            build_keys.setdefault(key, []).append(row_id)
    candidates = [build_keys.get(key, []) if key is not None else [] for _, key in probe_rows]
    pairs = [(b, probe_id) for (probe_id, _), rows in zip(probe_rows, candidates) for b in rows]
    ok = iter(passes(build, probe, predicates, _row_array([b for b, _ in pairs]), _row_array([p for _, p in pairs])))
    out = []
    for (probe_id, _), rows in zip(probe_rows, candidates):
        matches = [b for b in rows if next(ok)]
        if mode == capi.JOIN_INNER:
            out.extend((b, probe_id) for b in matches)
        elif mode in (capi.JOIN_LEFT, capi.JOIN_RIGHT):
            out.extend((b, probe_id) for b in matches) if matches else out.append((NULL_ROW, probe_id))
        elif mode == capi.JOIN_SEMI:
            if matches:
                out.append(probe_id)
        elif mode == capi.JOIN_ANTI_NULL_AS_FALSE:
            if not matches:
                out.append(probe_id)
        else:
            raise ValueError(f"mode {mode} takes no secondary predicates")
    return out


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIBRARY_PATH):
            subprocess.check_call(["make", "-C", REPO, "build/libjoin_predicates_oracle.so"])
        lib = C.CDLL(LIBRARY_PATH)
        lib.orc_join_hash_predicates.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                                 C.c_int32, C.c_int32, C.c_void_p, C.c_uint32, C.c_void_p]
        lib.orc_join_hash_predicates.restype = C.c_int
        lib.orc_join_result_free.argtypes = [C.c_void_p]
        lib.orc_join_result_free.restype = None
        _lib = lib
    return _lib


def ordered(build: Table, build_column: int, probe: Table, probe_column: int, mode: int, radix_bits: int, predicates,
            build_filter=None, probe_filter=None) -> orc.HostJoinResult:
    """The exact output of JoinHash with secondary predicates — pairs (or probe RowIDs), order, partition offsets — from
    orc_join_hash_predicates (tests/cpp/join_predicates_oracle.cpp); without predicates orc_join_hash's."""
    if not predicates:
        return orc.join_hash(build, build_column, probe, probe_column, mode, radix_bits, build_filter=build_filter,
                             probe_filter=probe_filter)
    lib = load()
    build_holder, probe_holder = build.view(), probe.view()
    build_struct = build_filter.struct() if build_filter is not None else None
    probe_struct = probe_filter.struct() if probe_filter is not None else None
    structs = (capi.JoinPredicate * len(predicates))(*[capi.JoinPredicate(b, p, c, 0) for b, p, c in predicates])
    raw = orc.OrcJoinResult()
    status = lib.orc_join_hash_predicates(build_holder.pointer(), build_column,
                                          C.byref(build_struct) if build_struct else None, probe_holder.pointer(),
                                          probe_column, C.byref(probe_struct) if probe_struct else None, mode,
                                          radix_bits, structs, len(predicates), C.byref(raw))
    if status != capi.HYB_OK:
        raise capi.HyriseB200Error(status, "orc_join_hash_predicates rejected the join")
    result = orc.HostJoinResult(raw)
    lib.orc_join_result_free(C.byref(raw))
    return result


def result_rows(result) -> list:
    """Output rows as hashable tuples (the form nested_loop returns)."""
    probe = [(int(r["chunk_id"]), int(r["chunk_offset"])) for r in result.probe]
    if result.build is None:
        return probe
    return list(zip([(int(r["chunk_id"]), int(r["chunk_offset"])) for r in result.build], probe))
