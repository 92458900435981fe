"""ctypes bindings of the C-ABI declared in include/hyrise_b200.h.

The library is the product: importing this module without a built ``hyrise_b200/lib/libhyrise_b200.so`` raises — there
is no CPU fallback (run ``python -c "import __graft_entry__ as g; g.build()"`` or ``make`` first).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libhyrise_b200.so")

# --- enums (include/hyrise_b200.h) -----------------------------------------------------------------------------------
HYB_OK, HYB_ERR_INVALID, HYB_ERR_UNSUPPORTED, HYB_ERR_CUDA, HYB_ERR_OOM, HYB_ERR_NOT_FOUND = range(6)

TYPE_INT32, TYPE_INT64, TYPE_FLOAT32, TYPE_FLOAT64, TYPE_STRING = range(5)
ENC_UNENCODED, ENC_DICTIONARY, ENC_FRAME_OF_REFERENCE = range(3)
VEC_NONE, VEC_FIXED_1B, VEC_FIXED_2B, VEC_FIXED_4B, VEC_BITPACKED = range(5)

(PRED_EQUALS, PRED_NOT_EQUALS, PRED_LESS_THAN, PRED_LESS_THAN_EQUALS, PRED_GREATER_THAN, PRED_GREATER_THAN_EQUALS,
 PRED_BETWEEN_INCLUSIVE, PRED_BETWEEN_LOWER_EXCLUSIVE, PRED_BETWEEN_UPPER_EXCLUSIVE, PRED_BETWEEN_EXCLUSIVE,
 PRED_IN, PRED_NOT_IN, PRED_LIKE, PRED_NOT_LIKE, PRED_LIKE_INSENSITIVE, PRED_NOT_LIKE_INSENSITIVE,
 PRED_IS_NULL, PRED_IS_NOT_NULL) = range(18)

(JOIN_INNER, JOIN_LEFT, JOIN_RIGHT, JOIN_FULL_OUTER, JOIN_CROSS, JOIN_SEMI, JOIN_ANTI_NULL_AS_TRUE,
 JOIN_ANTI_NULL_AS_FALSE) = range(8)

(AGG_MIN, AGG_MAX, AGG_SUM, AGG_AVG, AGG_COUNT, AGG_COUNT_STAR, AGG_COUNT_DISTINCT, AGG_STDDEV_SAMP,
 AGG_ANY) = range(9)

EXPR_COLUMN, EXPR_LITERAL, EXPR_ADD, EXPR_SUB, EXPR_MUL, EXPR_DIV, EXPR_MOD, EXPR_NULL = range(8)

TERM_LEAF, TERM_AND, TERM_OR, TERM_SCAN, TERM_IN = range(5)  # hyb_expression_term_kind

(AGG_PATH_NONE, AGG_PATH_STREAM_STATIC, AGG_PATH_STREAM_GENERIC, AGG_PATH_TILE_G4, AGG_PATH_TILE_G8, AGG_PATH_GENERAL,
 AGG_PATH_GENERAL_REGROWN) = range(7)

# hyb_join_path: one JOIN_PATH_TABLE_* | one JOIN_PATH_PROBE_* | JOIN_PATH_RERUN (include/hyrise_b200.h)
(JOIN_PATH_TABLE_RANK, JOIN_PATH_TABLE_DIRECT, JOIN_PATH_TABLE_DIRECT_SHIFTED, JOIN_PATH_TABLE_HASH,
 JOIN_PATH_TABLE_HASH_WIDE) = range(1, 6)
JOIN_PATH_TABLE_MASK = 0xF
JOIN_PATH_PROBE_NONE, JOIN_PATH_PROBE_SPAN, JOIN_PATH_PROBE_TILE_LEAN, JOIN_PATH_PROBE_TILE = 0x00, 0x10, 0x20, 0x30
JOIN_PATH_PROBE_MASK = 0xF0
JOIN_PATH_RERUN = 0x100
JOIN_PATH_SECONDARY = 0x200

MAX_EXPR_NODES = 16
MAX_GROUPBY_COLUMNS = 8
MAX_AGGREGATES = 16
MAX_FUSED_PREDICATES = 8
MAX_EXPRESSION_LEAVES = 8
MAX_EXPRESSION_COLUMNS = 8
MAX_EXPRESSION_TESTS = 16
MAX_EXPRESSION_DEPTH = 8
MAX_SORT_COLUMNS = 8
MAX_JOIN_PREDICATES = 4
SORT_KEY_AGGREGATE, SORT_KEY_COLUMN = range(2)  # hyb_aggregate_sort_key::kind
INVALID_VALUE_ID = 0xFFFFFFFF
DEFAULT_CHUNK_SIZE = 65535
FOR_BLOCK_SIZE = 2048


# --- structs ---------------------------------------------------------------------------------------------------------
class RowID(C.Structure):
    _fields_ = [("chunk_id", C.c_uint32), ("chunk_offset", C.c_uint32)]


class Value(C.Union):
    _fields_ = [("i32", C.c_int32), ("i64", C.c_int64), ("f32", C.c_float), ("f64", C.c_double)]


class SegmentDesc(C.Structure):
    _fields_ = [
        ("encoding", C.c_int32),
        ("data_type", C.c_int32),
        ("vector_type", C.c_int32),
        ("bit_width", C.c_int32),
        ("row_count", C.c_uint32),
        ("dictionary_size", C.c_uint32),
        ("values", C.c_void_p),
        ("nulls", C.c_void_p),
        ("attribute_vector", C.c_void_p),
        ("dictionary_codes", C.c_void_p),
    ]


class TableView(C.Structure):
    _fields_ = [("chunk_count", C.c_uint32), ("column_count", C.c_uint32), ("segments", C.POINTER(SegmentDesc))]


class HostBlock(C.Structure):
    _fields_ = [("base", C.c_void_p), ("bytes", C.c_uint64)]


class ScanPredicate(C.Structure):
    _fields_ = [
        ("column_id", C.c_uint32),
        ("condition", C.c_int32),
        ("lower", Value),
        ("upper", Value),
        ("value_id_bounds", C.c_void_p),
    ]


class ColumnScanPredicate(C.Structure):
    _fields_ = [
        ("left_column_id", C.c_uint32),
        ("condition", C.c_int32),
        ("right_column_id", C.c_uint32),
        ("reserved", C.c_uint32),
        ("right_in_left", C.c_void_p),
    ]


class Literal(C.Structure):
    _fields_ = [("data_type", C.c_int32), ("value", Value)]


class InPredicate(C.Structure):
    _fields_ = [
        ("column_id", C.c_uint32),
        ("condition", C.c_int32),
        ("element_count", C.c_uint32),
        ("has_null_element", C.c_uint32),
        ("elements", C.POINTER(Literal)),
        ("dictionary_matches", C.c_void_p),
    ]


class JoinSide(C.Structure):
    _fields_ = [("table", C.c_uint64), ("column_id", C.c_uint32), ("filter", C.c_uint64)]


class JoinPredicate(C.Structure):
    _fields_ = [("build_column_id", C.c_uint32), ("probe_column_id", C.c_uint32), ("condition", C.c_int32),
                ("reserved", C.c_uint32)]


class ExprNode(C.Structure):
    _fields_ = [("op", C.c_int32), ("column_id", C.c_uint32), ("literal_type", C.c_int32), ("literal", Value)]


class ExpressionTerm(C.Structure):
    _fields_ = [("kind", C.c_int32), ("condition", C.c_int32), ("node_counts", C.c_uint32 * 3), ("reserved", C.c_uint32),
                ("operands", (ExprNode * MAX_EXPR_NODES) * 3)]


class ExpressionScanPredicate(C.Structure):
    _fields_ = [("term_count", C.c_uint32), ("reserved", C.c_uint32), ("terms", C.POINTER(ExpressionTerm))]


class ExpressionLeafTests(C.Structure):
    _fields_ = [("scan_count", C.c_uint32), ("in_count", C.c_uint32), ("scans", C.POINTER(ScanPredicate)),
                ("ins", C.POINTER(InPredicate))]


class AggregateDef(C.Structure):
    _fields_ = [("function", C.c_int32), ("node_count", C.c_uint32), ("nodes", ExprNode * MAX_EXPR_NODES)]


class AggregateQuery(C.Structure):
    _fields_ = [
        ("table", C.c_uint64),
        ("filter", C.c_uint64),
        ("predicate_count", C.c_uint32),
        ("predicates", C.POINTER(ScanPredicate)),
        ("groupby_count", C.c_uint32),
        ("groupby_column_ids", C.POINTER(C.c_uint32)),
        ("aggregate_count", C.c_uint32),
        ("aggregates", C.POINTER(AggregateDef)),
    ]


class SortColumn(C.Structure):
    _fields_ = [("column_id", C.c_uint32), ("descending", C.c_int32)]


class AggregateSortKey(C.Structure):
    _fields_ = [("kind", C.c_int32), ("index", C.c_uint32), ("descending", C.c_int32)]


class AggregateOutputColumn(C.Structure):
    """hyb_aggregate_output_column: kind SORT_KEY_AGGREGATE | SORT_KEY_COLUMN, and the aggregate or column index."""
    _fields_ = [("kind", C.c_int32), ("index", C.c_uint32)]


class DistributedStats(C.Structure):
    _fields_ = [("split_count_ms", C.c_float), ("count_wait_ms", C.c_float), ("push_ms", C.c_float),
                ("done_wait_ms", C.c_float), ("local_ms", C.c_float), ("finish_ms", C.c_float),
                ("tuples_sent", C.c_uint64), ("tuples_received", C.c_uint64), ("nvlink_bytes", C.c_uint64),
                ("colocated", C.c_uint32), ("aggregate_partitioned", C.c_uint32)]


class OperatorStats(C.Structure):
    _fields_ = [
        ("device_ms", C.c_float),
        ("dominant_kernel_ms", C.c_float),
        ("kernel_launches", C.c_uint32),
        # AGG_PATH_* of an AggregateHash call, JOIN_PATH_* bits of a JoinHash call, 1 / 2 after
        # hyb_table_scan_expression_tests (column-test leaves only / mixed with operand leaves), 0 after any other scan,
        # the number of scatter passes after hyb_sort / hyb_aggregate_result_sort
        ("path", C.c_uint32),
        ("algorithmic_bytes", C.c_uint64),
        ("input_rows", C.c_uint64),
        ("output_rows", C.c_uint64),
    ]


# Every symbol include/hyrise_b200.h declares: (name, argtypes). All return int except the two noted.
_P = C.c_void_p
_CTX = C.c_void_p
_U64 = C.c_uint64
_U32 = C.c_uint32
_I32 = C.c_int32
SYMBOLS = {
    "hyb_abi_version": [],
    "hyb_last_error": [],
    "hyb_context_create": [C.c_int, C.POINTER(_CTX)],
    "hyb_context_destroy": [_CTX],
    "hyb_device_count": [C.POINTER(C.c_int)],
    "hyb_context_synchronize": [_CTX],
    "hyb_context_set_option": [_CTX, C.c_char_p, C.c_char_p],
    "hyb_host_alloc": [C.c_size_t, C.POINTER(_P)],
    "hyb_host_free": [_P],
    "hyb_table_upload": [_CTX, C.POINTER(TableView), C.POINTER(_U64)],
    "hyb_table_create": [_CTX, _U32, C.POINTER(_U64)],
    "hyb_table_append_chunk": [_CTX, _U64, C.POINTER(SegmentDesc)],
    "hyb_table_append_chunk_device": [_CTX, _U64, C.POINTER(SegmentDesc)],
    "hyb_table_drop": [_CTX, _U64],
    "hyb_blocks_upload": [_CTX, C.POINTER(HostBlock), _U32, C.POINTER(_U64)],
    "hyb_table_upload_from_blocks": [_CTX, C.POINTER(TableView), _U64, C.POINTER(_U64)],
    "hyb_blocks_free": [_CTX, _U64],
    "hyb_binary_table_open": [C.c_char_p, _I32, C.POINTER(C.c_void_p)],
    "hyb_binary_table_close": [C.c_void_p],
    "hyb_binary_table_info": [C.c_void_p, C.POINTER(_U32), C.POINTER(_U32), C.POINTER(_U32)],
    "hyb_binary_table_column": [C.c_void_p, _U32, C.POINTER(C.c_char_p), C.POINTER(_I32), C.POINTER(_I32)],
    "hyb_binary_table_view": [C.c_void_p, C.POINTER(TableView)],
    "hyb_binary_table_sorted_columns": [C.c_void_p, _U32, C.POINTER(C.c_uint16), C.POINTER(C.c_uint8), C.POINTER(_U32)],
    "hyb_binary_table_string_dictionary": [C.c_void_p, _U32, _U32, C.POINTER(C.c_void_p), C.POINTER(C.POINTER(C.c_uint64)),
                                           C.POINTER(_U32)],
    "hyb_binary_table_value_id_bounds": [C.c_void_p, _U32, C.c_char_p, _U64, C.c_char_p, _U64, C.POINTER(_U32)],
    "hyb_binary_table_like_bitmaps": [C.c_void_p, _U32, C.c_char_p, _U64, _I32, C.POINTER(_U32), C.POINTER(_U32)],
    "hyb_binary_table_column_translation": [C.c_void_p, _U32, _U32, C.POINTER(_U32), C.POINTER(_U32)],
    "hyb_binary_table_blocks": [C.c_void_p, C.POINTER(HostBlock), C.POINTER(_U32)],
    "hyb_table_upload_binary": [_CTX, C.c_void_p, C.POINTER(_U64)],
    "hyb_table_info": [_CTX, _U64, C.POINTER(_U32), C.POINTER(_U32), C.POINTER(_U64), C.POINTER(_U64)],
    "hyb_flip_predicate_condition": [_I32, C.POINTER(_I32)],
    "hyb_next_float_towards": [C.c_double, C.c_double, C.POINTER(C.c_float), C.POINTER(_I32)],
    "hyb_lossless_predicate_cast": [_I32, C.POINTER(Literal), _I32, _I32, C.POINTER(_I32), C.POINTER(Value)],
    "hyb_lossless_between_cast": [_I32, C.POINTER(Literal), C.POINTER(Literal), _I32, C.POINTER(_I32), C.POINTER(Value),
                                  C.POINTER(Value)],
    "hyb_like_dictionary_matches": [C.c_char_p, _U64, _I32, C.c_void_p, C.POINTER(_U64), _U32, C.POINTER(_U32),
                                    C.POINTER(_U32)],
    "hyb_dictionary_translate": [C.c_void_p, C.POINTER(_U64), _U32, C.c_void_p, C.POINTER(_U64), _U32, C.POINTER(_U32)],
    "hyb_dictionary_order_ranks": [_U32, C.POINTER(C.c_void_p), C.POINTER(C.POINTER(_U64)), C.POINTER(_U32), C.POINTER(_U32),
                                   C.POINTER(_U32)],
    "hyb_binary_table_string_order_ranks": [C.c_void_p, _U32, C.POINTER(_U32), C.POINTER(_U32)],
    "hyb_table_set_string_order": [_CTX, _U64, _U32, C.POINTER(_U32), _U64],
    "hyb_table_scan": [_CTX, _U64, C.POINTER(ScanPredicate), _U64, C.POINTER(_U64)],
    "hyb_table_scan_columns": [_CTX, _U64, C.POINTER(ColumnScanPredicate), _U64, C.POINTER(_U64)],
    "hyb_table_scan_in": [_CTX, _U64, C.POINTER(InPredicate), _U64, C.POINTER(_U64)],
    "hyb_table_scan_expression": [_CTX, _U64, C.POINTER(ExpressionScanPredicate), _U64, C.POINTER(_U64)],
    "hyb_table_scan_expression_tests": [_CTX, _U64, C.POINTER(ExpressionScanPredicate), C.POINTER(ExpressionLeafTests),
                                        _U64, C.POINTER(_U64)],
    "hyb_in_dictionary_matches": [_I32, C.c_void_p, C.POINTER(_U64), _U32, C.c_void_p, C.POINTER(_U64), _U32,
                                  C.POINTER(_U32), C.POINTER(_U32)],
    "hyb_binary_table_in_bitmaps": [C.c_void_p, _U32, _I32, C.c_void_p, C.POINTER(_U64), _U32, C.POINTER(_U32),
                                    C.POINTER(_U32)],
    "hyb_in_list_normalize": [_I32, C.POINTER(Literal), _U32, C.POINTER(Value), C.POINTER(_U32)],
    "hyb_pos_list_info": [_CTX, _U64, C.POINTER(_U64), C.POINTER(_U32)],
    "hyb_pos_list_chunk_offsets": [_CTX, _U64, _P],
    "hyb_pos_list_copy": [_CTX, _U64, _U64, _U64, _P],
    "hyb_pos_list_free": [_CTX, _U64],
    "hyb_join_hash": [_CTX, C.POINTER(JoinSide), C.POINTER(JoinSide), _I32, _I32, C.POINTER(_U64)],
    "hyb_join_hash_predicates": [_CTX, C.POINTER(JoinSide), C.POINTER(JoinSide), _I32, _I32, C.POINTER(JoinPredicate), _U32,
                                 C.POINTER(_U64)],
    "hyb_join_result_info": [_CTX, _U64, C.POINTER(_U64), C.POINTER(_U32), C.POINTER(_I32)],
    "hyb_join_result_partition_offsets": [_CTX, _U64, _P],
    "hyb_join_result_copy": [_CTX, _U64, _U64, _U64, _P, _P],
    "hyb_join_result_free": [_CTX, _U64],
    "hyb_join_result_pos_list": [_CTX, _U64, _I32, C.POINTER(_U64)],
    "hyb_join_result_output_chunks": [_CTX, _U64, _P, C.POINTER(_U32)],
    "hyb_join_side_positions": [_CTX, C.POINTER(JoinSide), C.POINTER(_U64)],
    "hyb_join_materialize": [_CTX, C.POINTER(JoinSide), _U32, _P, _P],
    "hyb_join_partition": [_CTX, C.POINTER(JoinSide), _U32, _U32, _P, _P, C.POINTER(_U64)],
    "hyb_join_partition_push": [_CTX, C.POINTER(JoinSide), _U32, _U32, _P, _P],
    "hyb_exchange_arena_create": [_CTX, _U64, C.POINTER(_P), _P],
    "hyb_exchange_arena_open": [_CTX, _P, C.POINTER(_P)],
    "hyb_exchange_arena_close": [_CTX, _P],
    "hyb_exchange_arena_destroy": [_CTX, _P],
    "hyb_peer_group_create": [_CTX, _U32, _U32, _U64, _P, C.POINTER(_U64)],
    "hyb_peer_group_connect": [_CTX, _U64, _P],
    "hyb_peer_group_destroy": [_CTX, _U64],
    "hyb_join_hash_distributed": [_CTX, _U64, C.POINTER(JoinSide), C.POINTER(JoinSide), _U32, _U32, _I32, C.POINTER(_U64)],
    "hyb_aggregate_hash_distributed": [_CTX, _U64, C.POINTER(AggregateQuery), _U32, _U64, C.POINTER(_U64)],
    "hyb_peer_group_stats": [_CTX, _U64, C.POINTER(DistributedStats)],
    "hyb_aggregate_hash": [_CTX, C.POINTER(AggregateQuery), C.POINTER(_U64)],
    "hyb_aggregate_hash_expression": [_CTX, C.POINTER(AggregateQuery), C.POINTER(ExpressionScanPredicate),
                                      C.POINTER(ExpressionLeafTests), C.POINTER(_U64)],
    "hyb_aggregate_result_info": [_CTX, _U64, C.POINTER(_U64), C.POINTER(_I32)],
    "hyb_aggregate_result_row_ids": [_CTX, _U64, _P],
    "hyb_aggregate_result_values": [_CTX, _U64, _U32, _P, _P, C.POINTER(_I32)],
    "hyb_aggregate_result_free": [_CTX, _U64],
    "hyb_aggregate_result_top_k": [_CTX, _U64, _U32, _U32, _I32, _P, C.POINTER(_U32)],
    "hyb_sort": [_CTX, _U64, _U64, C.POINTER(SortColumn), _U32, C.POINTER(_U64)],
    "hyb_aggregate_result_sort": [_CTX, _U64, C.POINTER(AggregateSortKey), _U32, _P],
    "hyb_aggregate_result_table": [_CTX, _U64, C.POINTER(AggregateOutputColumn), _U32, _U32, C.POINTER(_U64)],
    "hyb_last_operator_stats": [_CTX, C.POINTER(OperatorStats)],
    "hyb_pos_list_device_ptr": [_CTX, _U64, C.POINTER(_P)],
    "hyb_join_result_device_ptrs": [_CTX, _U64, C.POINTER(_P), C.POINTER(_P)],
    "hyb_context_stream": [_CTX, C.POINTER(_P)],
}


LIKE_CONDITIONS = (PRED_LIKE, PRED_NOT_LIKE, PRED_LIKE_INSENSITIVE, PRED_NOT_LIKE_INSENSITIVE)


def like_dictionary_matches(pattern: bytes, condition: int, entries) -> "np.ndarray":
    """hyb_like_dictionary_matches: the LikeMatcher result of every entry of one string dictionary (a sequence of bytes)
    as ceil(len / 32) uint32 words, entry i = bit i & 31 of word i >> 5; NOT variants are already inverted. Host only."""
    import numpy as np

    entries = [bytes(entry) for entry in entries]
    offsets = np.zeros(len(entries) + 1, dtype=np.uint64)
    if entries:
        offsets[1:] = np.cumsum([len(entry) for entry in entries])
    chars = b"".join(entries) or None  # NULL: every entry is empty
    words = np.zeros(max((len(entries) + 31) // 32, 1), dtype=np.uint32)
    check(load_library().hyb_like_dictionary_matches(pattern, len(pattern), condition, chars,
                                                     offsets.ctypes.data_as(C.POINTER(C.c_uint64)), len(entries),
                                                     words.ctypes.data_as(C.POINTER(C.c_uint32)), None))
    return words[: (len(entries) + 31) // 32]


def _string_dictionary_arguments(entries) -> tuple:
    """(chars or None, uint64 offsets) of a sequence of bytes in the layout of the dictionary entry points."""
    import numpy as np

    entries = [bytes(entry) for entry in entries]
    offsets = np.zeros(len(entries) + 1, dtype=np.uint64)
    if entries:
        offsets[1:] = np.cumsum([len(entry) for entry in entries])
    return b"".join(entries) or None, offsets  # NULL characters: every entry is empty


def dictionary_translate(left_entries, right_entries) -> "np.ndarray":
    """hyb_dictionary_translate: right_in_left of one chunk, for two sorted unique string dictionaries (sequences of
    bytes): word j = 2 * lower_bound(left, right[j]) + (right[j] in left). Host only."""
    import numpy as np

    left_chars, left_offsets = _string_dictionary_arguments(left_entries)
    right_chars, right_offsets = _string_dictionary_arguments(right_entries)
    count = len(right_offsets) - 1
    words = np.zeros(max(count, 1), dtype=np.uint32)
    check(load_library().hyb_dictionary_translate(left_chars, left_offsets.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                  len(left_offsets) - 1, right_chars,
                                                  right_offsets.ctypes.data_as(C.POINTER(C.c_uint64)), count,
                                                  words.ctypes.data_as(C.POINTER(C.c_uint32))))
    return words[:count]


def dictionary_order_ranks(dictionaries) -> tuple["np.ndarray", int]:
    """hyb_dictionary_order_ranks: (ranks, distinct count) for sorted unique string dictionaries (sequences of bytes):
    every entry's dense rank among the distinct strings of all of them, dictionary after dictionary. Host only."""
    import numpy as np

    arguments = [_string_dictionary_arguments(dictionary) for dictionary in dictionaries]
    count = len(arguments)
    chars = (C.c_void_p * max(count, 1))(*[C.cast(C.c_char_p(chars), C.c_void_p) if chars else None
                                           for chars, _ in arguments])
    offsets = (C.POINTER(C.c_uint64) * max(count, 1))(*[offsets.ctypes.data_as(C.POINTER(C.c_uint64))
                                                         for _, offsets in arguments])
    counts = (C.c_uint32 * max(count, 1))(*[len(offsets) - 1 for _, offsets in arguments])
    total = sum(len(offsets) - 1 for _, offsets in arguments)
    ranks = np.zeros(max(total, 1), dtype=np.uint32)
    distinct = C.c_uint32()
    check(load_library().hyb_dictionary_order_ranks(count, chars, offsets, counts, ranks.ctypes.data_as(C.POINTER(C.c_uint32)),
                                                    C.byref(distinct)))
    return ranks[:total], distinct.value


def in_dictionary_matches(condition: int, elements, entries) -> "np.ndarray":
    """hyb_in_dictionary_matches: membership of every entry of one string dictionary (a sequence of bytes) in the list
    `elements` (bytes, any order, repeats allowed) as ceil(len / 32) uint32 words, entry i = bit i & 31 of word i >> 5;
    NOT IN is already inverted. Host only."""
    import numpy as np

    element_chars, element_offsets = _string_dictionary_arguments(elements)
    chars, offsets = _string_dictionary_arguments(entries)
    count = len(offsets) - 1
    words = np.zeros(max((count + 31) // 32, 1), dtype=np.uint32)
    check(load_library().hyb_in_dictionary_matches(condition, element_chars,
                                                   element_offsets.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                   len(element_offsets) - 1, chars,
                                                   offsets.ctypes.data_as(C.POINTER(C.c_uint64)), count,
                                                   words.ctypes.data_as(C.POINTER(C.c_uint32)), None))
    return words[: (count + 31) // 32]


def literal_array(literals) -> "C.Array":
    """A ctypes array of hyb_literal from (data_type, value) pairs of numeric types (at least one slot)."""
    array = (Literal * max(len(literals), 1))()
    for index, (data_type, value) in enumerate(literals):
        array[index].data_type = data_type
        if data_type == TYPE_INT32:
            array[index].value.i32 = int(value)
        elif data_type == TYPE_INT64:
            array[index].value.i64 = int(value)
        elif data_type == TYPE_FLOAT32:
            array[index].value.f32 = float(value)
        elif data_type == TYPE_FLOAT64:
            array[index].value.f64 = float(value)
    return array


def in_list_normalize(column_type: int, literals) -> list:
    """hyb_in_list_normalize: the numeric list `literals` ((data_type, value) pairs) as the sorted, disjoint closed
    intervals [(lo, hi), ...] of `column_type` values it matches; Python ints for integer columns, floats otherwise
    (float32 bounds exactly representable). Host only."""
    elements = literal_array(literals)
    count = C.c_uint32(0)
    lib = load_library()
    check(lib.hyb_in_list_normalize(column_type, elements, len(literals), None, C.byref(count)))
    bounds = (Value * max(2 * count.value, 1))()
    check(lib.hyb_in_list_normalize(column_type, elements, len(literals), bounds, C.byref(count)))
    member = {TYPE_INT32: "i32", TYPE_INT64: "i64", TYPE_FLOAT32: "f32", TYPE_FLOAT64: "f64"}[column_type]
    return [(getattr(bounds[2 * i], member), getattr(bounds[2 * i + 1], member)) for i in range(count.value)]


IPC_HANDLE_BYTES = 64
EXCHANGE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p))


class HyriseB200Error(RuntimeError):
    """Raised for any non-zero hyb_status (the shim's Fail(), utils/assert.hpp:48-82)."""

    def __init__(self, status: int, message: str):
        super().__init__(f"hyb_status {status}: {message}")
        self.status = status


class UnsupportedOnDevice(HyriseB200Error):
    """HYB_ERR_UNSUPPORTED: the caller must run the CPU operator."""


_lib = None


def load_library(path: str | None = None) -> C.CDLL:
    """dlopen the C-ABI library and bind every declared symbol. Fails loudly when the library is missing."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise ImportError(
            f"{path} is missing: the CUDA extension is the product path and has no CPU fallback. "
            "Build it with `python -c 'import __graft_entry__ as g; g.build()'`."
        )
    lib = C.CDLL(path)
    for name, argtypes in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.argtypes = argtypes
        fn.restype = C.c_char_p if name == "hyb_last_error" else None if name == "hyb_binary_table_close" else C.c_int
    _lib = lib
    return lib


def check(status: int) -> None:
    if status == HYB_OK:
        return
    message = load_library().hyb_last_error().decode("utf-8", "replace")
    if status == HYB_ERR_UNSUPPORTED:
        raise UnsupportedOnDevice(status, message)
    raise HyriseB200Error(status, message)
