"""Thin object wrapper over the C-ABI (capi.py): context, device tables, device-resident results.

Everything here is plumbing: it marshals numpy buffers into the structs of include/hyrise_b200.h and back. All compute
happens in libhyrise_b200.so.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Sequence

import numpy as np

from . import capi
from .capi import check
from .storage import NUMPY_TYPES, Chunk, ColumnDefinition, Segment, Table, TableViewHolder

ROW_ID_DTYPE = np.dtype([("chunk_id", np.uint32), ("chunk_offset", np.uint32)])
# hyb_dictionary_position: a string MIN / MAX result, entry value_id of chunk chunk_id's dictionary
POSITION_DTYPE = np.dtype([("chunk_id", np.uint32), ("value_id", np.uint32)])


@dataclass
class Predicate:
    """column <condition> value | column BETWEEN lower AND upper | column IS [NOT] NULL | column [NOT] LIKE pattern — the
    arguments of ColumnVsValueTableScanImpl / ColumnBetweenTableScanImpl / ColumnIsNullTableScanImpl after
    lossless_predicate_variant_cast (table_scan.cpp:340-366), or of ColumnLikeTableScanImpl with the pattern (bytes or
    str) in `lower`."""

    column_id: int
    condition: int
    lower: object = None
    upper: object = None


@dataclass
class ColumnComparison:
    """left column <condition> right column — the arguments of ColumnVsColumnTableScanImpl; condition is one of
    PRED_EQUALS .. PRED_GREATER_THAN_EQUALS."""

    left_column_id: int
    condition: int
    right_column_id: int


def build_column_scan_predicate(table: Table, comparison: ColumnComparison, right_in_left: np.ndarray | None = None,
                                ) -> tuple[capi.ColumnScanPredicate, object]:
    """The C struct plus an object that must stay alive while it is in use. String pairs get the translation of the
    right dictionaries into the left ones (Table.string_column_translation) unless `right_in_left` is given."""
    struct = capi.ColumnScanPredicate()
    struct.left_column_id = comparison.left_column_id
    struct.condition = comparison.condition
    struct.right_column_id = comparison.right_column_id
    keepalive = None
    definitions = table.column_definitions
    strings = all(column < len(definitions) and definitions[column].data_type == capi.TYPE_STRING
                  for column in (comparison.left_column_id, comparison.right_column_id))
    if right_in_left is None and strings:
        right_in_left = table.string_column_translation(comparison.left_column_id, comparison.right_column_id)
    if right_in_left is not None:
        keepalive = np.zeros(max(len(right_in_left), 1), dtype=np.uint32)  # never NULL, even without dictionary entries
        keepalive[: len(right_in_left)] = right_in_left
        struct.right_in_left = keepalive.ctypes.data
    return struct, keepalive


@dataclass
class InList:
    """column [NOT] IN (elements) — the literal list of an InExpression (condition PRED_IN or PRED_NOT_IN). Elements are
    typed the way Hyrise types SQL literals (literal_type): int -> int32 if it fits, else int64; float -> double;
    np.float32 -> float; str / bytes -> string; None -> NULL."""

    column_id: int
    condition: int
    elements: Sequence = ()


def literal_type(element) -> tuple[int | None, object]:
    """(hyb data type, value) of one IN list element; (None, None) for NULL. Strings come back as bytes (str: UTF-8)."""
    if element is None:
        return None, None
    if isinstance(element, (bool, np.bool_)):
        raise TypeError("a boolean is not a SQL literal of Hyrise")
    if isinstance(element, (str, bytes, np.bytes_)):
        return capi.TYPE_STRING, element.encode() if isinstance(element, str) else bytes(element)
    if isinstance(element, np.float32):
        return capi.TYPE_FLOAT32, float(element)
    if isinstance(element, np.int32):
        return capi.TYPE_INT32, int(element)
    if isinstance(element, np.int64):
        return capi.TYPE_INT64, int(element)
    if isinstance(element, (int, np.integer)):
        value = int(element)
        if -2**31 <= value < 2**31:
            return capi.TYPE_INT32, value
        if -2**63 <= value < 2**63:
            return capi.TYPE_INT64, value
        raise OverflowError(f"{value} exceeds int64")
    if isinstance(element, (float, np.floating)):
        return capi.TYPE_FLOAT64, float(element)
    raise TypeError(f"unsupported IN list element {element!r}")


def build_in_predicate(table: Table, in_list: InList, dictionary_matches: np.ndarray | None = None,
                       ) -> tuple[capi.InPredicate, object]:
    """The C struct plus an object that must stay alive while it is in use. A string column gets the dictionary bitmaps
    of its string elements (Table.string_in_bitmaps) unless `dictionary_matches` is given, and none when the list has no
    string element; a numeric column gets its numeric elements and whether the list holds a NULL (its string elements
    are dropped, as the reference drops them)."""
    struct = capi.InPredicate()
    struct.column_id = in_list.column_id
    struct.condition = in_list.condition
    typed = [literal_type(element) for element in in_list.elements]
    definitions = table.column_definitions
    strings = in_list.column_id < len(definitions) and definitions[in_list.column_id].data_type == capi.TYPE_STRING
    if strings:
        string_elements = [value for data_type, value in typed if data_type == capi.TYPE_STRING]
        if dictionary_matches is None and string_elements:
            dictionary_matches = table.string_in_bitmaps(in_list.column_id, in_list.condition, string_elements)
        keepalive = None
        if dictionary_matches is not None:
            keepalive = np.zeros(max(len(dictionary_matches), 1), dtype=np.uint32)  # never NULL, even without entries
            keepalive[: len(dictionary_matches)] = dictionary_matches
            struct.dictionary_matches = keepalive.ctypes.data
        return struct, keepalive
    numeric = [(data_type, value) for data_type, value in typed if data_type not in (None, capi.TYPE_STRING)]
    elements = capi.literal_array(numeric)
    struct.element_count = len(numeric)
    struct.has_null_element = int(any(data_type is None for data_type, _ in typed))
    struct.elements = C.cast(elements, C.POINTER(capi.Literal))
    if dictionary_matches is not None:  # bitmaps on a numeric column: the library rejects them
        words = np.ascontiguousarray(dictionary_matches, dtype=np.uint32)
        struct.dictionary_matches = words.ctypes.data
        return struct, (elements, words)
    return struct, elements


def _set_value(target: capi.Value, data_type: int, value) -> None:
    if value is None:
        return
    if data_type == capi.TYPE_INT32:
        target.i32 = int(value)
    elif data_type == capi.TYPE_INT64:
        target.i64 = int(value)
    elif data_type == capi.TYPE_FLOAT32:
        target.f32 = float(np.float32(value))
    elif data_type == capi.TYPE_FLOAT64:
        target.f64 = float(value)


def build_scan_predicate(table: Table, predicate: Predicate) -> tuple[capi.ScanPredicate, object]:
    """Returns the C struct plus an object that must stay alive while the struct is in use."""
    data_type = table.column_definitions[predicate.column_id].data_type
    struct = capi.ScanPredicate()
    struct.column_id = predicate.column_id
    struct.condition = predicate.condition
    keepalive = None
    needs_value = predicate.condition not in (capi.PRED_IS_NULL, capi.PRED_IS_NOT_NULL)
    if predicate.condition in capi.LIKE_CONDITIONS and data_type != capi.TYPE_STRING:
        # ScanLikeNonStringColumn (table_scan_string_test.cpp): LIKE on a non-string column is an error, not a CPU job
        raise capi.HyriseB200Error(capi.HYB_ERR_INVALID, "LIKE needs a string column")
    if data_type == capi.TYPE_STRING:
        if predicate.condition in capi.LIKE_CONDITIONS:
            bitmaps = table.string_like_bitmaps(predicate)
            keepalive = np.zeros(max(bitmaps.size, 1), dtype=np.uint32)  # never NULL, even without dictionary entries
            keepalive[: bitmaps.size] = bitmaps
            struct.value_id_bounds = keepalive.ctypes.data
        elif needs_value:
            keepalive = np.ascontiguousarray(table.string_value_id_bounds(predicate), dtype=np.uint32)
            struct.value_id_bounds = keepalive.ctypes.data
    else:
        _set_value(struct.lower, data_type, predicate.lower)
        _set_value(struct.upper, data_type, predicate.upper)
    return struct, keepalive


@dataclass
class Expression:
    """Reverse-Polish arithmetic over columns/literals: nodes are ("col", id) | ("lit", type, value) | "+" "-" "*" "/"."""

    nodes: Sequence

    @staticmethod
    def column(column_id: int) -> "Expression":
        return Expression([("col", column_id)])


@dataclass
class Aggregate:
    function: int
    expression: Expression | None = None  # None for COUNT(*)


_OPS = {"+": capi.EXPR_ADD, "-": capi.EXPR_SUB, "*": capi.EXPR_MUL, "/": capi.EXPR_DIV, "%": capi.EXPR_MOD}


def _fill_nodes(targets, nodes: Sequence) -> None:
    """Writes RPN nodes ("col", id) | ("lit", type, value) | ("null",) | "+" "-" "*" "/" "%" into hyb_expr_node slots."""
    for position, node in enumerate(nodes):
        target = targets[position]
        if isinstance(node, str):
            target.op = _OPS[node]
        elif node[0] == "col":
            target.op = capi.EXPR_COLUMN
            target.column_id = node[1]
        elif node[0] == "null":
            target.op = capi.EXPR_NULL
        else:
            target.op = capi.EXPR_LITERAL
            target.literal_type = node[1]
            _set_value(target.literal, node[1], node[2])


def build_aggregate_defs(aggregates: Sequence[Aggregate]):
    defs = (capi.AggregateDef * max(len(aggregates), 1))()
    for index, aggregate in enumerate(aggregates):
        defs[index].function = aggregate.function
        nodes = [] if aggregate.expression is None else list(aggregate.expression.nodes)
        if len(nodes) > capi.MAX_EXPR_NODES:
            raise capi.UnsupportedOnDevice(capi.HYB_ERR_UNSUPPORTED, "expression too long")
        defs[index].node_count = len(nodes)
        _fill_nodes(defs[index].nodes, nodes)
    return defs


@dataclass
class ScanExpression:
    """The predicate of hyb_table_scan_expression as a postfix term list: ("leaf", condition, operands) | "and" | "or".
    An operand is an RPN node list as in Expression, plus ("null",) for a NULL literal and "%" for modulo. Operands per
    condition: = .. >=: (left, right); BETWEEN: (value, lower, upper); IS [NOT] NULL: (operand,). Combine with & and |.
    Column-test leaves ("scan", Predicate) | ("in", InList) are what hyb_table_scan / hyb_table_scan_in take; a tree
    holding one runs through hyb_table_scan_expression_tests."""

    terms: list

    @staticmethod
    def leaf(condition: int, *operands: Sequence) -> "ScanExpression":
        return ScanExpression([("leaf", condition, [list(operand) for operand in operands])])

    @staticmethod
    def scan(predicate: Predicate) -> "ScanExpression":
        """A HYB_TERM_SCAN leaf: the rows hyb_table_scan selects for `predicate` (a numeric literal has the column's
        type already, see hyb_lossless_predicate_cast)."""
        return ScanExpression([("scan", predicate)])

    @staticmethod
    def in_list(in_list: InList) -> "ScanExpression":
        """A HYB_TERM_IN leaf: the rows hyb_table_scan_in selects for `in_list`."""
        return ScanExpression([("in", in_list)])

    def has_tests(self) -> bool:
        return any(not isinstance(term, str) and term[0] in ("scan", "in") for term in self.terms)

    def __and__(self, other: "ScanExpression") -> "ScanExpression":
        return ScanExpression(self.terms + other.terms + ["and"])

    def __or__(self, other: "ScanExpression") -> "ScanExpression":
        return ScanExpression(self.terms + other.terms + ["or"])

    def leaves(self) -> list:
        return [term for term in self.terms if not isinstance(term, str)]


def build_expression_scan_predicate(expression: ScanExpression) -> tuple[capi.ExpressionScanPredicate, object]:
    """The C struct plus the term array it points to (keep it alive while the struct is in use). An operand longer than
    MAX_EXPR_NODES does not fit the struct: UnsupportedOnDevice, as the library answers."""
    terms = (capi.ExpressionTerm * max(len(expression.terms), 1))()
    for index, term in enumerate(expression.terms):
        if isinstance(term, str):
            terms[index].kind = {"and": capi.TERM_AND, "or": capi.TERM_OR}[term]
            continue
        if term[0] in ("scan", "in"):
            terms[index].kind = capi.TERM_SCAN if term[0] == "scan" else capi.TERM_IN
            continue
        _, condition, operands = term
        terms[index].kind = capi.TERM_LEAF
        terms[index].condition = condition
        if len(operands) > 3:
            raise capi.HyriseB200Error(capi.HYB_ERR_INVALID, "a leaf takes at most three operands")
        for slot, nodes in enumerate(operands):
            if len(nodes) > capi.MAX_EXPR_NODES:
                raise capi.UnsupportedOnDevice(capi.HYB_ERR_UNSUPPORTED, "operand longer than MAX_EXPR_NODES")
            terms[index].node_counts[slot] = len(nodes)
            _fill_nodes(terms[index].operands[slot], nodes)
    struct = capi.ExpressionScanPredicate()
    struct.term_count = len(expression.terms)
    struct.terms = C.cast(terms, C.POINTER(capi.ExpressionTerm))
    return struct, terms


def build_expression_leaf_tests(table: Table, expression: ScanExpression) -> tuple[capi.ExpressionLeafTests, object]:
    """hyb_expression_leaf_tests of the column-test leaves of `expression`, in postfix order, with the value-ID bounds,
    LIKE bitmaps and IN bitmaps of the host table (build_scan_predicate / build_in_predicate), plus what must stay alive
    while the struct is in use."""
    leaves = [term for term in expression.terms if not isinstance(term, str)]
    scan_leaves = [leaf[1] for leaf in leaves if leaf[0] == "scan"]
    in_leaves = [leaf[1] for leaf in leaves if leaf[0] == "in"]
    scans = (capi.ScanPredicate * max(len(scan_leaves), 1))()
    ins = (capi.InPredicate * max(len(in_leaves), 1))()
    keepalive = [scans, ins]
    for index, predicate in enumerate(scan_leaves):
        scans[index], alive = build_scan_predicate(table, predicate)
        keepalive.append(alive)
    for index, in_list in enumerate(in_leaves):
        ins[index], alive = build_in_predicate(table, in_list)
        keepalive.append(alive)
    struct = capi.ExpressionLeafTests()
    struct.scan_count = len(scan_leaves)
    struct.in_count = len(in_leaves)
    struct.scans = C.cast(scans, C.POINTER(capi.ScanPredicate))
    struct.ins = C.cast(ins, C.POINTER(capi.InPredicate))
    return struct, keepalive


class DeviceTable:
    def __init__(self, context: "DeviceContext", handle: int, host_table: Table, holder: TableViewHolder):
        self.context = context
        self.handle = handle
        self.host_table = host_table
        self._holder = holder

    def drop(self) -> None:
        if self.handle:
            check(self.context.lib.hyb_table_drop(self.context.ptr, self.handle))
            self.handle = 0


class DevicePosList:
    """Device-resident output of hyb_table_scan: a RowIDPosList per input chunk."""

    def __init__(self, context: "DeviceContext", handle: int):
        self.context = context
        self.handle = handle

    def info(self) -> tuple[int, int]:
        total, chunks = C.c_uint64(), C.c_uint32()
        check(self.context.lib.hyb_pos_list_info(self.context.ptr, self.handle, C.byref(total), C.byref(chunks)))
        return total.value, chunks.value

    def chunk_offsets(self) -> np.ndarray:
        _, chunks = self.info()
        offsets = np.empty(chunks + 1, dtype=np.uint64)
        check(self.context.lib.hyb_pos_list_chunk_offsets(self.context.ptr, self.handle, offsets.ctypes.data))
        return offsets

    def to_host(self, out: np.ndarray | None = None) -> np.ndarray:
        total, _ = self.info()
        if out is None:
            out = np.empty(total, dtype=ROW_ID_DTYPE)
        check(self.context.lib.hyb_pos_list_copy(self.context.ptr, self.handle, 0, total, out.ctypes.data))
        return out[:total]

    def free(self) -> None:
        if self.handle:
            check(self.context.lib.hyb_pos_list_free(self.context.ptr, self.handle))
            self.handle = 0


class DeviceJoinResult:
    def __init__(self, context: "DeviceContext", handle: int, has_build_side: bool):
        self.context = context
        self.handle = handle
        self.has_build_side = has_build_side

    def info(self) -> tuple[int, int, int]:
        pairs, partitions, bits = C.c_uint64(), C.c_uint32(), C.c_int32()
        check(self.context.lib.hyb_join_result_info(self.context.ptr, self.handle, C.byref(pairs), C.byref(partitions),
                                                     C.byref(bits)))
        return pairs.value, partitions.value, bits.value

    def partition_offsets(self) -> np.ndarray:
        _, partitions, _ = self.info()
        offsets = np.empty(partitions + 1, dtype=np.uint64)
        check(self.context.lib.hyb_join_result_partition_offsets(self.context.ptr, self.handle, offsets.ctypes.data))
        return offsets

    def to_host(self, out_build: np.ndarray | None = None, out_probe: np.ndarray | None = None):
        pairs, _, _ = self.info()
        probe = np.empty(pairs, dtype=ROW_ID_DTYPE) if out_probe is None else out_probe
        build = None
        if self.has_build_side:
            build = np.empty(pairs, dtype=ROW_ID_DTYPE) if out_build is None else out_build
        check(self.context.lib.hyb_join_result_copy(self.context.ptr, self.handle, 0, pairs,
                                                    None if build is None else build.ctypes.data, probe.ctypes.data))
        return (None if build is None else build[:pairs]), probe[:pairs]

    def pos_list(self, side: int) -> "DevicePosList":
        """hyb_join_result_pos_list: one side (0 = build, 1 = probe) as a PosList on that side's table, in result order."""
        handle = C.c_uint64()
        check(self.context.lib.hyb_join_result_pos_list(self.context.ptr, self.handle, side, C.byref(handle)))
        return DevicePosList(self.context, handle.value)

    def output_chunks(self) -> np.ndarray:
        """hyb_join_result_output_chunks: offsets of the chunks write_output_chunks cuts the result into."""
        count = C.c_uint32()
        check(self.context.lib.hyb_join_result_output_chunks(self.context.ptr, self.handle, None, C.byref(count)))
        offsets = np.zeros(count.value + 1, dtype=np.uint64)
        check(self.context.lib.hyb_join_result_output_chunks(self.context.ptr, self.handle, offsets.ctypes.data, C.byref(count)))
        return offsets

    def free(self) -> None:
        if self.handle:
            check(self.context.lib.hyb_join_result_free(self.context.ptr, self.handle))
            self.handle = 0


@dataclass
class AggregateOutput:
    group_count: int
    used_immediate_keys: bool
    row_ids: np.ndarray
    values: list[np.ndarray | None]  # POSITION_DTYPE for string MIN / MAX; None for ANY (the column at row_ids)
    nulls: list[np.ndarray | None]
    value_types: list[int]           # ANY: the column's type
    result_handle: int = 0   # != 0: the device-side result is still alive (aggregate_hash(..., keep_result=True))


def string_values(host_table: Table, column_id: int, positions: np.ndarray, nulls: np.ndarray) -> list:
    """The strings a string MIN / MAX result names (bytes per group, None for NULL), read from the host table's
    dictionaries."""
    return [None if null else bytes(host_table.chunks[int(position["chunk_id"])].segments[column_id]
                                    .string_dictionary[int(position["value_id"])])
            for position, null in zip(positions, nulls)]


class DevicePeerGroup:
    """hyb_peer_group: this rank's exchange arena and its mappings of the peers' arenas. Distributed operators are one
    C-ABI call per rank; the host layer only moves the IPC handles once (hyrise_b200.distributed.connect_peer_group)."""

    def __init__(self, context: "DeviceContext", rank: int, world: int, tuple_capacity: int):
        self.context = context
        self.rank, self.world = rank, world
        handle = (C.c_ubyte * capi.IPC_HANDLE_BYTES)()
        group = C.c_uint64()
        check(context.lib.hyb_peer_group_create(context.ptr, rank, world, tuple_capacity, handle, C.byref(group)))
        self.handle = group.value
        self.ipc_handle = bytes(handle)

    def connect(self, all_ipc_handles: Sequence[bytes]) -> None:
        packed = (C.c_ubyte * (capi.IPC_HANDLE_BYTES * self.world)).from_buffer_copy(b"".join(all_ipc_handles))
        check(self.context.lib.hyb_peer_group_connect(self.context.ptr, self.handle, packed))

    def join_hash(self, build: "DeviceTable", build_column: int, probe: "DeviceTable", probe_column: int,
                  build_chunk_base: int, probe_chunk_base: int, radix_bits: int = -1) -> "DeviceJoinResult":
        build_side = capi.JoinSide(build.handle, build_column, 0)
        probe_side = capi.JoinSide(probe.handle, probe_column, 0)
        handle = C.c_uint64()
        check(self.context.lib.hyb_join_hash_distributed(self.context.ptr, self.handle, C.byref(build_side), C.byref(probe_side),
                                                         build_chunk_base, probe_chunk_base, radix_bits, C.byref(handle)))
        return DeviceJoinResult(self.context, handle.value, True)

    def aggregate_hash(self, table: "DeviceTable", groupby_column_ids: Sequence[int], aggregates: Sequence["Aggregate"],
                       predicates: Sequence["Predicate"] = (), chunk_id_base: int = 0, position_base: int = 0) -> "AggregateOutput":
        query, keepalive = self.context._aggregate_query(table, groupby_column_ids, aggregates, predicates, None)
        handle = C.c_uint64()
        check(self.context.lib.hyb_aggregate_hash_distributed(self.context.ptr, self.handle, C.byref(query), chunk_id_base,
                                                              position_base, C.byref(handle)))
        del keepalive
        return self.context._collect_aggregate(handle.value, len(aggregates))

    def stats(self) -> capi.DistributedStats:
        stats = capi.DistributedStats()
        check(self.context.lib.hyb_peer_group_stats(self.context.ptr, self.handle, C.byref(stats)))
        return stats

    def destroy(self) -> None:
        if self.handle:
            check(self.context.lib.hyb_peer_group_destroy(self.context.ptr, self.handle))
            self.handle = 0


class DeviceContext:
    """hyb_context: one per process and GPU."""

    def __init__(self, device_index: int = 0):
        self.lib = capi.load_library()
        ptr = C.c_void_p()
        check(self.lib.hyb_context_create(device_index, C.byref(ptr)))
        self.ptr = ptr
        self.device_index = device_index
        self._kept_sources: dict[int, Table] = {}  # result handle -> host table of a kept aggregate's input

    def close(self) -> None:
        if self.ptr:
            check(self.lib.hyb_context_destroy(self.ptr))
            self.ptr = None

    def __enter__(self) -> "DeviceContext":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def synchronize(self) -> None:
        check(self.lib.hyb_context_synchronize(self.ptr))

    def set_option(self, name: str, value: str) -> None:
        """hyb_context_set_option: tuning / test knobs (the HYB_* environment variables are read at context creation)."""
        check(self.lib.hyb_context_set_option(self.ptr, name.encode(), str(value).encode()))

    # device column pool ------------------------------------------------------------------------------------------
    def upload(self, table) -> DeviceTable:
        """`table`: storage.Table or tpch.GeneratedTable (anything with view() / column_definitions)."""
        holder = table.view()
        handle = C.c_uint64()
        check(self.lib.hyb_table_upload(self.ptr, holder.pointer(), C.byref(handle)))
        return DeviceTable(self, handle.value, table, holder)

    def upload_blocks(self, blocks) -> int:
        """hyb_blocks_upload: DMA whole host arena blocks; returns the block-set handle."""
        array = (capi.HostBlock * max(len(blocks), 1))(*blocks)
        handle = C.c_uint64()
        check(self.lib.hyb_blocks_upload(self.ptr, array, len(blocks), C.byref(handle)))
        return handle.value

    def upload_from_blocks(self, table, block_set: int) -> DeviceTable:
        holder = table.view()
        handle = C.c_uint64()
        check(self.lib.hyb_table_upload_from_blocks(self.ptr, holder.pointer(), block_set, C.byref(handle)))
        return DeviceTable(self, handle.value, table, holder)

    def free_blocks(self, block_set: int) -> None:
        check(self.lib.hyb_blocks_free(self.ptr, block_set))

    # operators ---------------------------------------------------------------------------------------------------
    def table_scan(self, table: DeviceTable, predicate: Predicate, input_filter: DevicePosList | None = None,
                   ) -> DevicePosList:
        struct, keepalive = build_scan_predicate(table.host_table, predicate)
        handle = C.c_uint64()
        check(self.lib.hyb_table_scan(self.ptr, table.handle, C.byref(struct),
                                      input_filter.handle if input_filter else 0, C.byref(handle)))
        del keepalive
        return DevicePosList(self, handle.value)

    def table_scan_columns(self, table: DeviceTable, comparison: ColumnComparison,
                           input_filter: DevicePosList | None = None, right_in_left: np.ndarray | None = None,
                           ) -> DevicePosList:
        """hyb_table_scan_columns: `left <condition> right` per row. String pairs build the right-in-left translation of
        the host table's dictionaries unless `right_in_left` is given (e.g. NativeBinaryTable.column_translation)."""
        struct, keepalive = build_column_scan_predicate(table.host_table, comparison, right_in_left)
        handle = C.c_uint64()
        check(self.lib.hyb_table_scan_columns(self.ptr, table.handle, C.byref(struct),
                                              input_filter.handle if input_filter else 0, C.byref(handle)))
        del keepalive
        return DevicePosList(self, handle.value)

    def table_scan_in(self, table: DeviceTable, in_list: InList, input_filter: DevicePosList | None = None,
                      dictionary_matches: np.ndarray | None = None) -> DevicePosList:
        """hyb_table_scan_in: `column [NOT] IN (elements)` per row. String columns build the dictionary bitmaps of the
        host table unless `dictionary_matches` is given (e.g. NativeBinaryTable.in_bitmaps)."""
        struct, keepalive = build_in_predicate(table.host_table, in_list, dictionary_matches)
        handle = C.c_uint64()
        check(self.lib.hyb_table_scan_in(self.ptr, table.handle, C.byref(struct),
                                         input_filter.handle if input_filter else 0, C.byref(handle)))
        del keepalive
        return DevicePosList(self, handle.value)

    def table_scan_expression(self, table: DeviceTable, expression: ScanExpression,
                              input_filter: DevicePosList | None = None) -> DevicePosList:
        """hyb_table_scan_expression: comparisons, BETWEEN and IS [NOT] NULL over arithmetic operands, with AND / OR.
        A tree with column-test leaves (ScanExpression.scan / in_list) runs through hyb_table_scan_expression_tests."""
        struct, keepalive = build_expression_scan_predicate(expression)
        handle = C.c_uint64()
        if expression.has_tests():
            tests, tests_keepalive = build_expression_leaf_tests(table.host_table, expression)
            check(self.lib.hyb_table_scan_expression_tests(self.ptr, table.handle, C.byref(struct), C.byref(tests),
                                                           input_filter.handle if input_filter else 0, C.byref(handle)))
            del tests_keepalive
        else:
            check(self.lib.hyb_table_scan_expression(self.ptr, table.handle, C.byref(struct),
                                                     input_filter.handle if input_filter else 0, C.byref(handle)))
        del keepalive
        return DevicePosList(self, handle.value)

    def table_scan_expression_tests(self, table: DeviceTable, expression: ScanExpression,
                                    input_filter: DevicePosList | None = None) -> DevicePosList:
        """hyb_table_scan_expression_tests for any tree, a tree of operand leaves only included."""
        struct, keepalive = build_expression_scan_predicate(expression)
        tests, tests_keepalive = build_expression_leaf_tests(table.host_table, expression)
        handle = C.c_uint64()
        check(self.lib.hyb_table_scan_expression_tests(self.ptr, table.handle, C.byref(struct), C.byref(tests),
                                                       input_filter.handle if input_filter else 0, C.byref(handle)))
        del keepalive, tests_keepalive
        return DevicePosList(self, handle.value)

    def join_hash(self, build: DeviceTable, build_column: int, probe: DeviceTable, probe_column: int, mode: int,
                  radix_bits: int = -1, build_filter: DevicePosList | None = None,
                  probe_filter: DevicePosList | None = None, secondary=None) -> DeviceJoinResult:
        """hyb_join_hash; with `secondary` = [(build column, probe column, condition), ...] (`build value <condition>
        probe value`, the list may be empty) hyb_join_hash_predicates."""
        build_side = capi.JoinSide(build.handle, build_column, build_filter.handle if build_filter else 0)
        probe_side = capi.JoinSide(probe.handle, probe_column, probe_filter.handle if probe_filter else 0)
        handle = C.c_uint64()
        if secondary is None:
            check(self.lib.hyb_join_hash(self.ptr, C.byref(build_side), C.byref(probe_side), mode, radix_bits,
                                         C.byref(handle)))
        else:
            predicates = (capi.JoinPredicate * max(len(secondary), 1))(
                *[capi.JoinPredicate(build_col, probe_col, condition, 0) for build_col, probe_col, condition in secondary])
            check(self.lib.hyb_join_hash_predicates(self.ptr, C.byref(build_side), C.byref(probe_side), mode, radix_bits,
                                                    predicates, len(secondary), C.byref(handle)))
        semi_or_anti = mode in (capi.JOIN_SEMI, capi.JOIN_ANTI_NULL_AS_TRUE, capi.JOIN_ANTI_NULL_AS_FALSE)
        return DeviceJoinResult(self, handle.value, not semi_or_anti)

    def _aggregate_query(self, table: DeviceTable, groupby_column_ids, aggregates, predicates, input_filter):
        """AggregateQuery struct + the objects that must stay alive while it is in use."""
        query = capi.AggregateQuery()
        query.table = table.handle
        query.filter = input_filter.handle if input_filter else 0
        keepalive = []
        predicate_structs = (capi.ScanPredicate * max(len(predicates), 1))()
        for index, predicate in enumerate(predicates):
            struct, alive = build_scan_predicate(table.host_table, predicate)
            predicate_structs[index] = struct
            keepalive.append(alive)
        query.predicate_count = len(predicates)
        query.predicates = C.cast(predicate_structs, C.POINTER(capi.ScanPredicate))
        groupby = (C.c_uint32 * max(len(groupby_column_ids), 1))(*groupby_column_ids)
        query.groupby_count = len(groupby_column_ids)
        query.groupby_column_ids = C.cast(groupby, C.POINTER(C.c_uint32))
        defs = build_aggregate_defs(aggregates)
        query.aggregate_count = len(aggregates)
        query.aggregates = C.cast(defs, C.POINTER(capi.AggregateDef))
        keepalive += [predicate_structs, groupby, defs]
        return query, keepalive

    def aggregate_top_k(self, result_handle: int, aggregate_index: int, k: int, descending: bool = True) -> np.ndarray:
        """hyb_aggregate_result_top_k on a result kept alive with aggregate_hash(..., keep_result=True)."""
        indexes = np.zeros(k, dtype=np.uint32)
        count = C.c_uint32()
        check(self.lib.hyb_aggregate_result_top_k(self.ptr, result_handle, aggregate_index, k, int(descending),
                                                  indexes.ctypes.data, C.byref(count)))
        return indexes[: count.value]

    def sort(self, table: DeviceTable, columns: Sequence[tuple[int, bool]],
             input_filter: DevicePosList | None = None) -> DevicePosList:
        """hyb_sort: the table's rows (or the filter's) ordered by `columns`, (column_id, descending) pairs, most significant
        first; NULLs first in every column, ties in input order. One chunk in result order."""
        array = (capi.SortColumn * max(len(columns), 1))(*[capi.SortColumn(column, int(bool(descending)))
                                                           for column, descending in columns])
        handle = C.c_uint64()
        check(self.lib.hyb_sort(self.ptr, table.handle, input_filter.handle if input_filter else 0, array, len(columns),
                                C.byref(handle)))
        return DevicePosList(self, handle.value)

    def aggregate_sort(self, result_handle: int, keys: Sequence[tuple[int, int, bool]]) -> np.ndarray:
        """hyb_aggregate_result_sort on a result kept alive with aggregate_hash(..., keep_result=True): every group index in
        sorted order. `keys`: (capi.SORT_KEY_AGGREGATE | capi.SORT_KEY_COLUMN, index, descending), most significant first."""
        groups, immediate = C.c_uint64(), C.c_int32()
        check(self.lib.hyb_aggregate_result_info(self.ptr, result_handle, C.byref(groups), C.byref(immediate)))
        array = (capi.AggregateSortKey * max(len(keys), 1))(*[capi.AggregateSortKey(kind, index, int(bool(descending)))
                                                                for kind, index, descending in keys])
        indexes = np.zeros(max(groups.value, 1), dtype=np.uint32)
        check(self.lib.hyb_aggregate_result_sort(self.ptr, result_handle, array, len(keys), indexes.ctypes.data))
        return indexes[: groups.value]

    def aggregate_table(self, result_handle: int, columns: Sequence[tuple[int, int]],
                        chunk_size: int = capi.DEFAULT_CHUNK_SIZE) -> DeviceTable:
        """hyb_aggregate_result_table on a result kept alive with aggregate_hash(..., keep_result=True): the result as a
        table of the pool, column c = columns[c], (capi.SORT_KEY_AGGREGATE, aggregate index) or (capi.SORT_KEY_COLUMN,
        column of the aggregated table at the representative RowIDs). Every operator takes it like an uploaded table.
        Its host_table holds the derived schema and chunking only; the values live on the device."""
        array = (capi.AggregateOutputColumn * max(len(columns), 1))(*[capi.AggregateOutputColumn(kind, index)
                                                                      for kind, index in columns])
        handle = C.c_uint64()
        check(self.lib.hyb_aggregate_result_table(self.ptr, result_handle, array, len(columns), chunk_size,
                                                  C.byref(handle)))
        groups, immediate = C.c_uint64(), C.c_int32()
        check(self.lib.hyb_aggregate_result_info(self.ptr, result_handle, C.byref(groups), C.byref(immediate)))
        source = self._kept_sources.get(result_handle)
        definitions = []
        for position, (kind, index) in enumerate(columns):
            if kind == capi.SORT_KEY_AGGREGATE:
                value_type = C.c_int32()
                check(self.lib.hyb_aggregate_result_values(self.ptr, result_handle, index, None, None, C.byref(value_type)))
                definitions.append(ColumnDefinition(f"aggregate_{index}", value_type.value, True))
            else:
                definitions.append(ColumnDefinition(source.column_definitions[index].name,
                                                    source.column_definitions[index].data_type, True))
        host_table = Table(definitions, target_chunk_size=chunk_size)
        for begin in range(0, groups.value, chunk_size):
            rows = min(chunk_size, groups.value - begin)
            host_table.chunks.append(Chunk([Segment(capi.ENC_UNENCODED, definition.data_type, rows)
                                            for definition in definitions]))
        return DeviceTable(self, handle.value, host_table, None)

    def free_aggregate_result(self, result_handle: int) -> None:
        check(self.lib.hyb_aggregate_result_free(self.ptr, result_handle))
        self._kept_sources.pop(result_handle, None)

    def set_string_order(self, table: DeviceTable, column_id: int, ranks: np.ndarray | None = None) -> None:
        """hyb_table_set_string_order: attach the order ranks MIN / MAX over a string column need; computed from the host
        table's dictionaries unless `ranks` is given (e.g. NativeBinaryTable.string_order_ranks)."""
        if ranks is None:
            ranks = table.host_table.string_order_ranks(column_id)
        ranks = np.ascontiguousarray(ranks, dtype=np.uint32)
        check(self.lib.hyb_table_set_string_order(self.ptr, table.handle, column_id,
                                                  ranks.ctypes.data_as(C.POINTER(C.c_uint32)), len(ranks)))

    def _collect_aggregate(self, handle: int, aggregate_count: int, keep_result: bool = False,
                           any_types: dict | None = None) -> AggregateOutput:
        try:
            groups, immediate = C.c_uint64(), C.c_int32()
            check(self.lib.hyb_aggregate_result_info(self.ptr, handle, C.byref(groups), C.byref(immediate)))
            count = groups.value
            row_ids = np.empty(count, dtype=ROW_ID_DTYPE)
            check(self.lib.hyb_aggregate_result_row_ids(self.ptr, handle, row_ids.ctypes.data))
            values, nulls, types = [], [], []
            for index in range(aggregate_count):
                if any_types and index in any_types:
                    values.append(None)
                    nulls.append(None)
                    types.append(any_types[index])
                    continue
                raw = np.zeros(max(count, 1), dtype=np.uint64)
                null = np.zeros(max(count, 1), dtype=np.uint8)
                value_type = C.c_int32()
                check(self.lib.hyb_aggregate_result_values(self.ptr, handle, index, raw.ctypes.data, null.ctypes.data,
                                                           C.byref(value_type)))
                dtype = POSITION_DTYPE if value_type.value == capi.TYPE_STRING else NUMPY_TYPES[value_type.value]
                values.append(raw.view(np.uint8)[: count * np.dtype(dtype).itemsize].view(dtype).copy())
                nulls.append(null[:count].astype(bool))
                types.append(value_type.value)
        finally:
            if not keep_result:
                check(self.lib.hyb_aggregate_result_free(self.ptr, handle))
        output = AggregateOutput(count, bool(immediate.value), row_ids, values, nulls, types)
        output.result_handle = handle if keep_result else 0
        return output

    def aggregate_hash(self, table: DeviceTable, groupby_column_ids: Sequence[int], aggregates: Sequence[Aggregate],
                       predicates: Sequence[Predicate] = (), input_filter: DevicePosList | None = None,
                       keep_result: bool = False, expression: ScanExpression | None = None) -> AggregateOutput:
        """hyb_aggregate_hash, or hyb_aggregate_hash_expression when `expression` is given: the rows must also satisfy
        that tree (operand leaves, and column-test leaves ScanExpression.scan / in_list), evaluated inside the aggregate."""
        query, keepalive = self._aggregate_query(table, groupby_column_ids, aggregates, predicates, input_filter)
        handle = C.c_uint64()
        if expression is None:
            check(self.lib.hyb_aggregate_hash(self.ptr, C.byref(query), C.byref(handle)))
        else:
            struct, tree_keepalive = build_expression_scan_predicate(expression)
            tests = None
            if expression.has_tests():
                tests_struct, tests_keepalive = build_expression_leaf_tests(table.host_table, expression)
                tests = C.byref(tests_struct)
                keepalive += [tests_struct, tests_keepalive]
            check(self.lib.hyb_aggregate_hash_expression(self.ptr, C.byref(query), C.byref(struct), tests, C.byref(handle)))
            del tree_keepalive
        del keepalive
        definitions = table.host_table.column_definitions
        any_types = {index: definitions[aggregate.expression.nodes[0][1]].data_type
                     for index, aggregate in enumerate(aggregates) if aggregate.function == capi.AGG_ANY}
        if keep_result:  # aggregate_table types its COLUMN outputs from the aggregated table's schema
            self._kept_sources[handle.value] = table.host_table
        return self._collect_aggregate(handle.value, len(aggregates), keep_result, any_types)

    def last_stats(self) -> capi.OperatorStats:
        stats = capi.OperatorStats()
        check(self.lib.hyb_last_operator_stats(self.ptr, C.byref(stats)))
        return stats

    # pinned host memory -------------------------------------------------------------------------------------------
    def pinned_empty(self, count: int, dtype) -> np.ndarray:
        """numpy array over hyb_host_alloc memory (freed with pinned_free)."""
        dtype = np.dtype(dtype)
        ptr = C.c_void_p()
        check(self.lib.hyb_host_alloc(max(count, 1) * dtype.itemsize, C.byref(ptr)))
        buffer = (C.c_uint8 * (max(count, 1) * dtype.itemsize)).from_address(ptr.value)
        array = np.frombuffer(buffer, dtype=dtype, count=count)
        self._pinned = getattr(self, "_pinned", {})
        self._pinned[array.ctypes.data] = ptr
        return array

    def pinned_free(self, array: np.ndarray) -> None:
        ptr = getattr(self, "_pinned", {}).pop(array.ctypes.data, None)
        if ptr is not None:
            check(self.lib.hyb_host_free(ptr))
