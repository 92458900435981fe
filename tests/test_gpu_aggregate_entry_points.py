"""The three AggregateHash entry points (hyb_aggregate_hash, _expression, _distributed) share one host driver. This pins
what it reports on every kernel path (hyb_operator_stats: path, kernel_launches, algorithmic_bytes, input and output
rows), and the status of every rejection, each followed by a call on the same context that still matches the oracle."""
import ctypes as C

import numpy as np
import pytest

import aggregate_layouts as layouts
import oracle_lib as orc
from helpers import assert_aggregate_outputs_equal
from hyrise_b200 import capi
from hyrise_b200.device import (Aggregate, DevicePeerGroup, DevicePosList, Expression, Predicate, ScanExpression,
                                build_expression_scan_predicate)
from hyrise_b200.storage import NUMPY_TYPES, ColumnDefinition, Table
from test_oracle_expression_scan import col, lit

pytestmark = pytest.mark.gpu
P = capi
CASES = {case.name: case for case in layouts.CASES}
leaf, scan = ScanExpression.leaf, ScanExpression.scan


def column_bytes(table, column_id):
    """What one unfiltered pass reads of a column: values or value-IDs, a numeric dictionary, FrameOfReference block
    minima, NULL flags."""
    total = 0
    for chunk in table.chunks:
        segment = chunk.segments[column_id]
        if segment.encoding == P.ENC_UNENCODED:
            total += segment.values.itemsize * segment.row_count
        else:
            total += segment.attribute_vector.nbytes
            if segment.encoding == P.ENC_DICTIONARY and segment.data_type != P.TYPE_STRING:
                total += np.dtype(NUMPY_TYPES[segment.data_type]).itemsize * segment.dictionary_size
            if segment.encoding == P.ENC_FRAME_OF_REFERENCE:
                total += 4 * ((segment.row_count + P.FOR_BLOCK_SIZE - 1) // P.FOR_BLOCK_SIZE)
        if segment.nulls is not None:
            total += segment.row_count
    return total


def columns_read(groupby, aggregates, predicates):
    columns = set(groupby) | {predicate.column_id for predicate in predicates}
    for aggregate in aggregates:
        if aggregate.expression is not None:
            columns |= {node[1] for node in aggregate.expression.nodes if isinstance(node, tuple) and node[0] == "col"}
    return columns


def check_stats(device, output, path, launches, input_rows, algorithmic_bytes=None):
    stats = device.last_stats()
    got = (stats.path, stats.kernel_launches, stats.input_rows, stats.output_rows)
    assert got == (path, launches, input_rows, output.group_count), got
    if algorithmic_bytes is not None:
        assert stats.algorithmic_bytes == algorithmic_bytes
    return stats.algorithmic_bytes


def upload_case(device, cache, case):
    if case.builder not in cache:
        table = case.builder().table
        cache[case.builder] = (table, device.upload(table))
    return cache[case.builder]


@pytest.fixture(scope="module")
def uploaded(device):
    cache = {}
    yield cache
    for _, device_table in cache.values():
        device_table.drop()


# case -> (path, launches): the fused predicates' tests (one launch each) and every fast-path attempt, overflowing ones
# included; the general path adds its sweep and the compaction
FAST_PATHS = {
    "q1_static": (P.AGG_PATH_STREAM_STATIC, 2),
    "mixed_widths": (P.AGG_PATH_STREAM_GENERIC, 2),
    "int32_immediate": (P.AGG_PATH_TILE_G4, 1),
    "late_groups": (P.AGG_PATH_TILE_G8, 3),
    "twelve_groups": (P.AGG_PATH_GENERAL, 5),
    "extremes": (P.AGG_PATH_GENERAL, 2),
}


@pytest.mark.parametrize("name", list(FAST_PATHS))
def test_stats_on_each_path(device, uploaded, name):
    case = CASES[name]
    table, device_table = upload_case(device, uploaded, case)
    path, launches = FAST_PATHS[name]
    read = sum(column_bytes(table, c) for c in columns_read(case.groupby, case.aggregates, case.predicates))
    for _ in range(2):  # the second call reads the plan memo
        output = device.aggregate_hash(device_table, case.groupby, case.aggregates, case.predicates)
        check_stats(device, output, path, launches, table.row_count, read)
    assert_aggregate_outputs_equal(output, orc.aggregate_hash(table, case.groupby, case.aggregates, case.predicates))


def test_stats_general_regrown(device):
    table = layouts.regrowth_keys().table
    device_table = device.upload(table)
    try:
        aggregates = [layouts.SUM(layouts.col(2)), layouts.MIN(3), layouts.STAR]
        output = device.aggregate_hash(device_table, [0, 1], aggregates)
        read = sum(column_bytes(table, c) for c in (0, 1, 2, 3))
        check_stats(device, output, P.AGG_PATH_GENERAL_REGROWN, 3, table.row_count, read)
    finally:
        device_table.drop()


def small_table(rng, rows=20_000):
    """g (int32 groups), s (string, NULLs), v (int32), d (float64, NULLs) in 4 000-row dictionary chunks."""
    words = np.array([b"w%03d" % i for i in rng.integers(0, 300, rows)], dtype="S")
    definitions = [ColumnDefinition("g", P.TYPE_INT32), ColumnDefinition("s", P.TYPE_STRING, True),
                   ColumnDefinition("v", P.TYPE_INT32), ColumnDefinition("d", P.TYPE_FLOAT64, True)]
    columns = [rng.integers(0, 7, rows).astype(np.int32), words, rng.integers(-500, 500, rows).astype(np.int32),
               rng.integers(-64, 64, rows) / 8.0]
    nulls = [None, rng.random(rows) < 0.1, None, rng.random(rows) < 0.1]
    return Table.from_columns(definitions, columns, nulls, chunk_size=4_000).encode("Dictionary")


@pytest.fixture(scope="module")
def small(device):
    table = small_table(np.random.default_rng(5))
    device_table = device.upload(table)
    device.set_string_order(device_table, 1)
    yield table, device_table
    device_table.drop()


def column(column_id):
    return Expression.column(column_id)


def test_stats_distinct_stddev_and_string_extremes(device, small):
    table, device_table = small
    read = sum(column_bytes(table, c) for c in (0, 1, 2, 3))
    distinct = [Aggregate(P.AGG_COUNT_DISTINCT, column(2)), Aggregate(P.AGG_STDDEV_SAMP, column(3)),
                Aggregate(P.AGG_COUNT, column(1))]
    output = device.aggregate_hash(device_table, [0], distinct)
    check_stats(device, output, P.AGG_PATH_GENERAL, 4, table.row_count, read)
    rank_words = 4 * sum(chunk.segments[1].dictionary_size for chunk in table.chunks)
    extremes = [Aggregate(P.AGG_MIN, column(1)), Aggregate(P.AGG_MAX, column(1)), Aggregate(P.AGG_SUM, column(2))]
    output = device.aggregate_hash(device_table, [0], extremes)
    check_stats(device, output, P.AGG_PATH_GENERAL, 3, table.row_count,
                sum(column_bytes(table, c) for c in (0, 1, 2)) + rank_words)


def test_stats_filtered(device, small):
    table, device_table = small
    other = Table.from_columns([ColumnDefinition("k", P.TYPE_INT32)], [np.arange(0, 7, 2, dtype=np.int32)],
                               chunk_size=3).encode("Dictionary")
    device_other = device.upload(other)
    ascending = device.table_scan(device_table, Predicate(2, P.PRED_LESS_THAN, 100))
    join = device.join_hash(device_table, 0, device_other, 0, P.JOIN_INNER, -1)
    unordered = join.pos_list(0)
    aggregates = [Aggregate(P.AGG_SUM, column(2)), Aggregate(P.AGG_MIN, column(1)), Aggregate(P.AGG_COUNT_STAR)]
    rank_words = 4 * sum(chunk.segments[1].dictionary_size for chunk in table.chunks)
    try:
        for source in (ascending, unordered):
            rows = source.info()[0]
            output = device.aggregate_hash(device_table, [0], aggregates, input_filter=source)
            # the sweep, the string extremes, the compaction and the RowID gather
            check_stats(device, output, P.AGG_PATH_GENERAL, 4, rows, 8 * rows + rank_words)
    finally:
        for handle in (ascending, unordered, join):
            handle.free()
        device_other.drop()


def test_stats_expression_trees(device, uploaded, small):
    case = CASES["mixed_widths"]
    table, device_table = upload_case(device, uploaded, case)
    tree = leaf(P.PRED_GREATER_THAN_EQUALS, col(2) + col(2) + ["+"], lit(0))  # d >= 0 everywhere: the same groups
    plain = device.aggregate_hash(device_table, case.groupby, case.aggregates, case.predicates)
    plain_bytes = device.last_stats().algorithmic_bytes
    excess = []
    for _ in range(2):
        output = device.aggregate_hash(device_table, case.groupby, case.aggregates, case.predicates, expression=tree)
        # a tree never takes the streaming kernels: the predicate's tests and aggregate_fast_tree_kernel
        excess.append(check_stats(device, output, P.AGG_PATH_TILE_G4, 2, table.row_count) - plain_bytes)
        assert_aggregate_outputs_equal(output, plain)
    assert excess[0] == excess[1] and excess[0] > 0

    table, device_table = small
    aggregates = [Aggregate(P.AGG_MIN, column(3)), Aggregate(P.AGG_COUNT_STAR)]
    tree = scan(Predicate(2, P.PRED_LESS_THAN, 200)) | leaf(P.PRED_IS_NULL, col(3))
    device.aggregate_hash(device_table, [0], aggregates)
    plain_bytes = device.last_stats().algorithmic_bytes
    excess = []
    for _ in range(2):
        output = device.aggregate_hash(device_table, [0], aggregates, expression=tree)
        # the scan leaf's tests, the sweep and the compaction
        excess.append(check_stats(device, output, P.AGG_PATH_GENERAL, 3, table.row_count) - plain_bytes)
    assert excess[0] == excess[1] and excess[0] > 0


def test_any_beside_other_aggregates(device, uploaded, small):
    case = CASES["mixed_widths"]
    table, device_table = upload_case(device, uploaded, case)
    with_any = [Aggregate(P.AGG_ANY, column(0))] + case.aggregates
    expected = device.aggregate_hash(device_table, case.groupby, case.aggregates, case.predicates)
    stats = device.last_stats()
    output = device.aggregate_hash(device_table, case.groupby, with_any, case.predicates)
    check_stats(device, output, stats.path, stats.kernel_launches, stats.input_rows, stats.algorithmic_bytes)
    assert output.values[0] is None and output.value_types[0] == P.TYPE_STRING
    assert all(np.array_equal(a, b) for a, b in zip(output.values[1:], expected.values))

    table, device_table = small
    aggregates = [Aggregate(P.AGG_MIN, column(3)), Aggregate(P.AGG_ANY, column(1)), Aggregate(P.AGG_SUM, column(2))]
    output = device.aggregate_hash(device_table, [0], aggregates)
    check_stats(device, output, P.AGG_PATH_GENERAL, 2, table.row_count)
    expected = orc.aggregate_hash(table, [0], [aggregates[0], aggregates[2]])
    assert np.array_equal(output.values[0], expected.values[0]) and np.array_equal(output.values[2], expected.values[1])
    assert output.value_types[1] == P.TYPE_STRING


# ---- rejections through the raw C-ABI ------------------------------------------------------------------------------
ENTRY_POINTS = ["hash", "expression", "distributed"]


@pytest.fixture(scope="module")
def peer_group(device):
    group = DevicePeerGroup(device, 0, 1, 1 << 16)
    yield group
    group.destroy()


def call(device, peer_group, entry, query):
    """The raw status of one entry point (the expression entry point with an always-true tree)."""
    handle = C.c_uint64()
    if entry == "hash":
        status = device.lib.hyb_aggregate_hash(device.ptr, C.byref(query) if query is not None else None, C.byref(handle))
    elif entry == "expression":
        struct, keepalive = build_expression_scan_predicate(leaf(P.PRED_EQUALS, lit(1), lit(1)))
        status = device.lib.hyb_aggregate_hash_expression(device.ptr, C.byref(query) if query is not None else None,
                                                          C.byref(struct), None, C.byref(handle))
        del keepalive
    else:
        status = device.lib.hyb_aggregate_hash_distributed(device.ptr, peer_group.handle,
                                                           C.byref(query) if query is not None else None, 0, 0,
                                                           C.byref(handle))
    if status == P.HYB_OK:
        device.free_aggregate_result(handle.value)
    return status


def still_works(device, small):
    table, device_table = small
    aggregates = [Aggregate(P.AGG_SUM, column(2)), Aggregate(P.AGG_COUNT, column(3))]
    output = device.aggregate_hash(device_table, [0], aggregates, [Predicate(2, P.PRED_GREATER_THAN, 0)])
    assert_aggregate_outputs_equal(output, orc.aggregate_hash(table, [0], aggregates, [Predicate(2, P.PRED_GREATER_THAN, 0)]))


def base_query(device, small, aggregates=None, groupby=(0,), predicates=(), input_filter=None):
    _, device_table = small
    aggregates = aggregates or [Aggregate(P.AGG_SUM, column(2))]
    return device._aggregate_query(device_table, list(groupby), aggregates, list(predicates), input_filter)


def shared_checks():
    """(field, value, status): the argument checks every entry point makes."""
    return [("groupby_count", P.MAX_GROUPBY_COLUMNS + 1, P.HYB_ERR_UNSUPPORTED),
            ("aggregate_count", P.MAX_AGGREGATES + 1, P.HYB_ERR_UNSUPPORTED),
            ("predicate_count", P.MAX_FUSED_PREDICATES + 1, P.HYB_ERR_UNSUPPORTED),
            ("groupby_column_ids", None, P.HYB_ERR_INVALID),
            ("aggregates", None, P.HYB_ERR_INVALID),
            ("predicates", None, P.HYB_ERR_INVALID)]


@pytest.mark.parametrize("entry", ENTRY_POINTS)
def test_argument_checks(device, small, peer_group, entry):
    assert call(device, peer_group, entry, None) == P.HYB_ERR_INVALID
    still_works(device, small)
    for field, value, status in shared_checks():
        query, keepalive = base_query(device, small, predicates=[Predicate(2, P.PRED_GREATER_THAN, 0)])
        if value is None:
            setattr(query, field, None)
            count = {"groupby_column_ids": "groupby_count", "aggregates": "aggregate_count",
                     "predicates": "predicate_count"}[field]
            setattr(query, count, 1)
        else:
            setattr(query, field, value)
        assert call(device, peer_group, entry, query) == status, field
        del keepalive
        still_works(device, small)


@pytest.mark.parametrize("entry", ENTRY_POINTS)
def test_tables_and_filters(device, small, peer_group, entry):
    table, device_table = small
    query, keepalive = base_query(device, small)
    query.table = 0x7FFF_FFFF
    assert call(device, peer_group, entry, query) == P.HYB_ERR_NOT_FOUND
    still_works(device, small)

    other = Table.from_columns([ColumnDefinition("k", P.TYPE_INT32)], [np.arange(0, 14, 2, dtype=np.int32)],
                               chunk_size=3).encode("Dictionary")
    device_other = device.upload(other)
    foreign = device.table_scan(device_other, Predicate(0, P.PRED_LESS_THAN, 5))
    left = device.join_hash(device_table, 0, device_other, 0, P.JOIN_LEFT, -1)
    with_null_rows = left.pos_list(0)
    try:
        for source, status in ((DevicePosList(device, 0x7FFF_FFFF), P.HYB_ERR_NOT_FOUND), (foreign, P.HYB_ERR_INVALID)):
            query, keepalive = base_query(device, small, input_filter=source)
            assert call(device, peer_group, entry, query) == status
            still_works(device, small)
        # keys 8, 10 and 12 of the other table find no row: their pairs hold NULL_ROW_IDs on this table's side
        assert (left.to_host()[0]["chunk_id"] == 0xFFFFFFFF).any()
        query, keepalive = base_query(device, small, input_filter=with_null_rows)
        assert call(device, peer_group, entry, query) == P.HYB_ERR_UNSUPPORTED
        still_works(device, small)
    finally:
        for handle in (foreign, with_null_rows, left):
            handle.free()
        device_other.drop()


@pytest.mark.parametrize("entry", ENTRY_POINTS)
def test_aggregate_checks(device, small, peer_group, entry):
    any_expression = Aggregate(P.AGG_ANY, Expression([("col", 2), ("col", 2), "+"]))
    # a distributed ANY is declined before the aggregates are checked
    for aggregates, groupby, status in (
            ([any_expression], [0], P.HYB_ERR_UNSUPPORTED if entry == "distributed" else P.HYB_ERR_INVALID),
            ([Aggregate(99, column(2))], [0], P.HYB_ERR_UNSUPPORTED),
            ([Aggregate(P.AGG_SUM, column(2))], [4], P.HYB_ERR_INVALID)):
        query, keepalive = base_query(device, small, aggregates, groupby)
        assert call(device, peer_group, entry, query) == status
        still_works(device, small)


@pytest.fixture(scope="module")
def wide(device):
    """81 int32 columns: sixteen aggregates over five columns each reference 80 distinct columns."""
    rng = np.random.default_rng(9)
    definitions = [ColumnDefinition(f"c{c}", P.TYPE_INT32) for c in range(81)]
    table = Table.from_columns(definitions, [rng.integers(0, 10, 3000).astype(np.int32) for _ in range(81)],
                               chunk_size=1000).encode("Unencoded")
    device_table = device.upload(table)
    yield table, device_table
    device_table.drop()


@pytest.mark.parametrize("entry", ENTRY_POINTS)
def test_too_many_distinct_aggregate_columns(device, small, wide, peer_group, entry):
    _, device_table = wide
    aggregates = [Aggregate(P.AGG_SUM, Expression([("col", 5 * a + 1)] + sum([[("col", 5 * a + k), "+"] for k in range(2, 6)],
                                                                                []))) for a in range(16)]
    query, keepalive = device._aggregate_query(device_table, [0], aggregates, [Predicate(0, P.PRED_LESS_THAN, 5)], None)
    assert call(device, peer_group, entry, query) == P.HYB_ERR_UNSUPPORTED
    still_works(device, small)
