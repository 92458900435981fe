"""hyb_aggregate_result_table on the H100: an aggregate result as a table of the pool, compared value by value and NULL by
NULL with the table aggregate_table_expected builds on the host, then used as the input of a HAVING scan, a semi and an
inner join, a sort and a further aggregate (each against the oracle over the expected table), and TPC-H Q18 / Q15 on
dbgen sf-0.01 against SQLite running the reference's query text (tpch_queries.cpp)."""
import ctypes as C
import os
import sqlite3
import subprocess

import numpy as np
import pytest

import oracle_lib as orc
import sort_oracle
from aggregate_cases import CASES
from aggregate_table_expected import expected_table
from helpers import assert_aggregate_outputs_equal, assert_pos_lists_equal, row_ids_equal, tbl
from hyrise_b200 import capi
from hyrise_b200.device import Aggregate, Expression, Predicate, ScanExpression
from hyrise_b200.storage import ColumnDefinition, Table

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AGG, COL = capi.SORT_KEY_AGGREGATE, capi.SORT_KEY_COLUMN
NULL_CHUNK = 0xFFFFFFFF
NUMERIC_CASES = [case for case in CASES
                 if all(tbl(case[2]).column_definitions[g].data_type != capi.TYPE_STRING for g in case[6])]


def on(column):
    return Expression.column(column)


def table_shape(device, table):
    chunks, rows = C.c_uint32(), C.c_uint64()
    capi.check(device.lib.hyb_table_info(device.ptr, table.handle, C.byref(chunks), None, C.byref(rows), None))
    return chunks.value, rows.value


def assert_table_content(device, derived, want, key_columns):
    """Every value and NULL of `derived` at its RowID equals `want`'s. Read through the public API: one aggregate over
    `derived` grouped by its key columns (unique per row) with MIN of every column; its representative RowIDs are the
    positions (a single row of a no-GROUP-BY table is row {0, 0})."""
    chunk_size = want.target_chunk_size
    assert table_shape(device, derived) == (want.chunk_count, want.row_count)
    if want.row_count == 0:
        return
    read = device.aggregate_hash(derived, key_columns, [Aggregate(capi.AGG_MIN, on(c)) for c in range(want.column_count)])
    assert read.group_count == want.row_count, "key columns are not unique per row"
    if key_columns:
        positions = read.row_ids["chunk_id"].astype(np.int64) * chunk_size + read.row_ids["chunk_offset"]
    else:
        positions = np.zeros(1, dtype=np.int64)
    for column in range(want.column_count):
        values, nulls = want.column_values(column)
        assert read.value_types[column] == want.column_definitions[column].data_type
        assert np.array_equal(read.nulls[column], nulls[positions]), f"column {column}: NULLs differ"
        got, expected = read.values[column][~read.nulls[column]], values[positions][~read.nulls[column]]
        assert got.dtype == expected.dtype
        if got.dtype.kind == "f":  # bit-identical, NaN included (any NaN: MIN may return another NaN payload)
            same = (got.view(f"u{got.itemsize}") == expected.view(f"u{got.itemsize}")) | (np.isnan(got) & np.isnan(expected))
            assert same.all(), f"column {column}: {got[~same][:8]} != {expected[~same][:8]}"
        else:
            assert np.array_equal(got, expected), f"column {column}: values differ"


def derive(device, source_host, source_dev, groupby, aggregates, columns, chunk_sizes, **query):
    """Aggregate, then one derived table per chunk size, each checked against the expected table; the last derived
    table, its expected table and the aggregate output are returned."""
    output = device.aggregate_hash(source_dev, groupby, aggregates, keep_result=True, **query)
    key_columns = [position for position, (kind, index) in enumerate(columns) if kind == COL and index in groupby]
    try:
        for chunk_size in chunk_sizes:
            derived = device.aggregate_table(output.result_handle, columns, chunk_size)
            stats = device.last_stats()
            assert stats.input_rows == stats.output_rows == output.group_count
            gathers = output.group_count > 0 and any(kind == COL for kind, _ in columns)
            assert stats.kernel_launches == (1 if gathers else 0) and stats.path == 0
            want = expected_table(source_host, output, columns, chunk_size)
            assert_table_content(device, derived, want, key_columns)
    finally:
        device.free_aggregate_result(output.result_handle)
    return derived, want, output


def standard_columns(groupby, aggregate_count, extra=()):
    return [(COL, g) for g in groupby] + [(AGG, a) for a in range(aggregate_count)] + list(extra)


def value_table(rng, rows, key_type=capi.TYPE_INT32, key_span=200, key_nulls=True, chunk_size=1000):
    """key (nullable, `key_type`, values in [0, key_span)), then int32, int64, float and double values with NULLs; the
    float and double columns hold -0.0 and NaN."""
    keys = rng.integers(0, key_span, rows)
    definitions = [ColumnDefinition("key", key_type, key_nulls), ColumnDefinition("i32", capi.TYPE_INT32, True),
                   ColumnDefinition("i64", capi.TYPE_INT64, True), ColumnDefinition("f32", capi.TYPE_FLOAT32, True),
                   ColumnDefinition("f64", capi.TYPE_FLOAT64, True)]
    floats = rng.normal(0, 100, rows)
    floats[rng.random(rows) < 0.01] = -0.0
    floats[rng.random(rows) < 0.005] = np.nan
    key_dtype = {capi.TYPE_INT32: np.int32, capi.TYPE_INT64: np.int64, capi.TYPE_FLOAT32: np.float32,
                 capi.TYPE_FLOAT64: np.float64}[key_type]
    if key_type == capi.TYPE_INT64:
        keys = keys * 2**33 + 7  # beyond int32
    columns = [keys.astype(key_dtype), rng.integers(-1000, 1000, rows).astype(np.int32),
               rng.integers(-2**40, 2**40, rows).astype(np.int64), floats.astype(np.float32), floats * 1.5]
    nulls = [rng.random(rows) < 0.02 if key_nulls else None] + [rng.random(rows) < 0.1 for _ in range(4)]
    return Table.from_columns(definitions, columns, nulls, chunk_size)


# ---- content ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", NUMERIC_CASES, ids=[f"{c[0]}@{c[1]}" for c in NUMERIC_CASES])
def test_golden_aggregate_fixtures(device, case):
    name, line, input_file, chunk_size, dictionary, definitions, groupby, expected_file, _ = case
    table = tbl(input_file, chunk_size)
    if dictionary:
        table.encode("Dictionary")
    aggregates = [Aggregate(function, None if column is None else on(column)) for column, function in definitions]
    derive(device, table, device.upload(table), groupby, aggregates, standard_columns(groupby, len(aggregates)), [2])


LAYOUTS = [("Unencoded", False, 200)] + [(encoding, bitpacking, span) for encoding in ("Dictionary", "FrameOfReference")
                                          for bitpacking in (False, True) for span in (200, 60_000, 1_000_000)]


@pytest.mark.parametrize("encoding,bitpacking,span", LAYOUTS, ids=[f"{e}-{'bp' if b else 'fw'}-{s}" for e, b, s in LAYOUTS])
def test_group_column_in_every_layout(device, encoding, bitpacking, span):
    """u8 / u16 / u32 vectors (dictionary sizes or FoR offsets below 2^8, 2^16 and above) and bit-packing; span 200 takes
    the immediate-key order with the NULL group first, span 1 000 000 first-appearance order."""
    rng = np.random.default_rng(span)
    table = value_table(rng, 90_000, key_span=span, chunk_size=30_000)
    table.encode([encoding, "Unencoded", "Unencoded", "Unencoded", "Unencoded"], bitpacking=bitpacking)
    aggregates = [Aggregate(capi.AGG_SUM, on(1)), Aggregate(capi.AGG_ANY, on(4))]
    _, _, output = derive(device, table, device.upload(table), [0], aggregates,
                          [(COL, 0), (AGG, 0), (COL, 4)], [capi.DEFAULT_CHUNK_SIZE])
    if span in (200, 1_000_000):  # dense keys, and keys spread over 11 times as many values as rows
        assert output.used_immediate_keys == (span == 200)


@pytest.mark.parametrize("key_type", [capi.TYPE_INT64, capi.TYPE_FLOAT32, capi.TYPE_FLOAT64])
def test_group_column_types_and_any(device, key_type):
    rng = np.random.default_rng(key_type)
    table = value_table(rng, 5_000, key_type=key_type, key_span=500)
    aggregates = [Aggregate(capi.AGG_ANY, on(column)) for column in (1, 2, 3, 4)]
    derive(device, table, device.upload(table), [0], aggregates, [(COL, c) for c in range(5)], [700])


@pytest.mark.parametrize("value_column", [1, 2, 3, 4], ids=["int32", "int64", "float", "double"])
def test_every_aggregate_function(device, value_column):
    """MIN / MAX (the column's type, -0.0 and NaN kept), SUM, AVG, COUNT, COUNT(*), COUNT(DISTINCT), STDDEV_SAMP (NULL for
    groups of fewer than two values: many groups are single rows)."""
    rng = np.random.default_rng(value_column)
    table = value_table(rng, 3_000, key_span=2_500, key_nulls=True)
    functions = [capi.AGG_MIN, capi.AGG_MAX, capi.AGG_SUM, capi.AGG_AVG, capi.AGG_COUNT, capi.AGG_COUNT_DISTINCT,
                 capi.AGG_STDDEV_SAMP]
    aggregates = [Aggregate(function, on(value_column)) for function in functions] + [Aggregate(capi.AGG_COUNT_STAR)]
    _, want, output = derive(device, table, device.upload(table), [0], aggregates,
                             standard_columns([0], len(aggregates)), [512])
    assert output.nulls[6].any(), "no STDDEV_SAMP NULL"


def test_scan_join_and_expression_inputs(device):
    rng = np.random.default_rng(7)
    table = value_table(rng, 20_000, key_span=3_000)
    table_dev = device.upload(table)
    aggregates = [Aggregate(capi.AGG_SUM, on(2)), Aggregate(capi.AGG_MAX, on(4)), Aggregate(capi.AGG_COUNT_STAR)]
    columns = standard_columns([0], len(aggregates), [(COL, 3)])
    scan = device.table_scan(table_dev, Predicate(1, capi.PRED_GREATER_THAN, 0))
    derive(device, table, table_dev, [0], aggregates, columns, [4_096], input_filter=scan)
    # a join's probe side in result order: rows whose i32 has a partner in a small dimension table
    dimension = Table.from_columns([ColumnDefinition("d", capi.TYPE_INT32)], [np.arange(-1000, 1000, 7, dtype=np.int32)])
    join = device.join_hash(device.upload(dimension), 0, table_dev, 1, capi.JOIN_INNER)
    derive(device, table, table_dev, [0], aggregates, columns, [4_096], input_filter=join.pos_list(1))
    tree = ScanExpression.leaf(capi.PRED_GREATER_THAN, [("col", 2), ("col", 1), "+"], [("lit", capi.TYPE_INT64, 0)])
    derive(device, table, table_dev, [0], aggregates, columns, [4_096], expression=tree)


def test_without_group_by_and_without_groups(device):
    table = value_table(np.random.default_rng(3), 1_000)
    table_dev = device.upload(table)
    aggregates = [Aggregate(capi.AGG_SUM, on(1)), Aggregate(capi.AGG_COUNT, on(3)), Aggregate(capi.AGG_AVG, on(4))]
    derive(device, table, table_dev, [], aggregates, standard_columns([], 3, [(COL, 2)]), [1, 5])
    nothing = device.table_scan(table_dev, Predicate(1, capi.PRED_GREATER_THAN, 10 ** 6))
    # the synthesised row of an empty input: COUNT 0, SUM / AVG NULL, the column at NULL_ROW_ID NULL
    _, want, output = derive(device, table, table_dev, [], aggregates, standard_columns([], 3, [(COL, 2)]), [4],
                             input_filter=nothing)
    assert output.group_count == 1 and output.row_ids[0]["chunk_id"] == NULL_CHUNK
    nothing = device.table_scan(table_dev, Predicate(1, capi.PRED_GREATER_THAN, 10 ** 6))
    derived, want, output = derive(device, table, table_dev, [0], aggregates, standard_columns([0], 3), [4],
                                   input_filter=nothing)
    assert output.group_count == 0 and table_shape(device, derived) == (0, 0)
    # every operator over a table without chunks returns its empty result
    assert device.table_scan(derived, Predicate(1, capi.PRED_GREATER_THAN, 0)).info()[0] == 0
    assert device.sort(derived, [(1, True)]).info()[0] == 0
    assert device.aggregate_hash(derived, [0], [Aggregate(capi.AGG_SUM, on(1))]).group_count == 0
    assert device.join_hash(derived, 0, table_dev, 0, capi.JOIN_SEMI).info()[0] == 0


def test_chunk_sizes_around_the_group_count(device):
    table = value_table(np.random.default_rng(11), 4_000, key_span=1_000_000, key_nulls=False)
    table_dev = device.upload(table)
    output = device.aggregate_hash(table_dev, [0], [Aggregate(capi.AGG_SUM, on(1))])
    groups = output.group_count
    aggregates = [Aggregate(capi.AGG_SUM, on(1)), Aggregate(capi.AGG_MIN, on(3))]
    derive(device, table, table_dev, [0], aggregates, standard_columns([0], 2, [(COL, 4)]),
           [1, groups - 1, groups, groups + 1, 65_535])


# ---- composition --------------------------------------------------------------------------------------------------------
@pytest.fixture
def composed(device):
    rng = np.random.default_rng(5)
    table = value_table(rng, 30_000, key_span=5_000)
    table.encode(["Dictionary", "Unencoded", "FrameOfReference", "Unencoded", "Dictionary"])
    table_dev = device.upload(table)
    aggregates = [Aggregate(capi.AGG_SUM, on(4)), Aggregate(capi.AGG_COUNT_STAR), Aggregate(capi.AGG_SUM, on(1)),
                  Aggregate(capi.AGG_MAX, on(1))]
    derived, want, _ = derive(device, table, table_dev, [0], aggregates, standard_columns([0], 4), [1_000])
    return table, table_dev, derived, want


CONDITIONS = [capi.PRED_EQUALS, capi.PRED_NOT_EQUALS, capi.PRED_LESS_THAN, capi.PRED_LESS_THAN_EQUALS,
              capi.PRED_GREATER_THAN, capi.PRED_GREATER_THAN_EQUALS, capi.PRED_BETWEEN_INCLUSIVE, capi.PRED_BETWEEN_EXCLUSIVE,
              capi.PRED_IS_NULL, capi.PRED_IS_NOT_NULL]
# (column, lower, upper): SUM(f64) double, COUNT(*) int64, SUM(i32) int64, MAX(i32) int32
BOUNDS = [(1, 100, 1_000), (2, 6, 8), (3, -50, 300), (4, 10, 200)]
HAVING = [(column, condition, lower, upper) for column, lower, upper in BOUNDS for condition in CONDITIONS]


@pytest.mark.parametrize("column,condition,lower,upper", HAVING)
def test_having_scan(device, composed, column, condition, lower, upper):
    """int literals against the double SUM (column 1) and the int64 COUNT / SUM columns, int32 against MAX."""
    _, _, derived, want = composed
    between = condition in (capi.PRED_BETWEEN_INCLUSIVE, capi.PRED_BETWEEN_EXCLUSIVE)
    predicate = Predicate(column, condition, lower, upper if between else None)
    got = device.table_scan(derived, predicate)
    assert_pos_lists_equal(got.to_host(), got.chunk_offsets(), orc.table_scan(want, predicate))


def sorted_pairs(build, probe):
    keys = [tuple(row) for row in probe] if build is None else [tuple(a) + tuple(b) for a, b in zip(build, probe)]
    return sorted(keys)


@pytest.mark.parametrize("mode", [capi.JOIN_SEMI, capi.JOIN_INNER])
def test_join_onto_the_table_under_a_having(device, composed, mode):
    table, table_dev, derived, want = composed
    having = Predicate(2, capi.PRED_GREATER_THAN, 6)
    got = device.join_hash(derived, 0, table_dev, 0, mode, build_filter=device.table_scan(derived, having))
    expected = orc.join_hash(want, 0, table, 0, mode, build_filter=orc.table_scan(want, having))
    build, probe = got.to_host()
    assert got.info()[0] == expected.pair_count > 0
    assert sorted_pairs(build, probe) == sorted_pairs(expected.build, expected.probe)


def test_sort_and_aggregate_over_the_table(device, composed):
    _, _, derived, want = composed
    definitions = [(2, True), (1, False), (0, False)]
    got = device.sort(derived, definitions)
    assert row_ids_equal(got.to_host(), sort_oracle.sort_table(want, definitions))
    # a view's aggregate: GROUP BY the COUNT column
    aggregates = [Aggregate(capi.AGG_SUM, on(3)), Aggregate(capi.AGG_COUNT_STAR), Aggregate(capi.AGG_MAX, on(4))]
    assert_aggregate_outputs_equal(device.aggregate_hash(derived, [2], aggregates), orc.aggregate_hash(want, [2], aggregates))


def test_table_outlives_the_result_and_the_aggregated_table(device):
    table = value_table(np.random.default_rng(9), 5_000, key_span=800)
    table_dev = device.upload(table)
    output = device.aggregate_hash(table_dev, [0], [Aggregate(capi.AGG_SUM, on(1))], keep_result=True)
    columns = [(COL, 0), (AGG, 0), (COL, 4)]
    derived = device.aggregate_table(output.result_handle, columns, 300)
    want = expected_table(table, output, columns, 300)
    device.free_aggregate_result(output.result_handle)
    table_dev.drop()
    device.synchronize()
    assert_table_content(device, derived, want, [0])
    predicate = Predicate(1, capi.PRED_GREATER_THAN, 0)
    got = device.table_scan(derived, predicate)
    assert_pos_lists_equal(got.to_host(), got.chunk_offsets(), orc.table_scan(want, predicate))
    derived.drop()


# ---- errors -------------------------------------------------------------------------------------------------------------
def test_errors(device):
    definitions = [ColumnDefinition("k", capi.TYPE_INT32), ColumnDefinition("v", capi.TYPE_INT32),
                   ColumnDefinition("s", capi.TYPE_STRING)]
    table = Table.from_columns(definitions, [np.array([1, 2, 1], dtype=np.int32), np.array([4, 5, 6], dtype=np.int32),
                                             np.array([b"x", b"y", b"z"])]).encode("Dictionary")
    table_dev = device.upload(table)
    device.set_string_order(table_dev, 2)
    aggregates = [Aggregate(capi.AGG_SUM, on(1)), Aggregate(capi.AGG_ANY, on(1)), Aggregate(capi.AGG_MIN, on(2))]
    output = device.aggregate_hash(table_dev, [0], aggregates, keep_result=True)
    handle, lib, ptr = output.result_handle, device.lib, device.ptr

    def status(columns, chunk_size=16, result=handle, out=True):
        array = (capi.AggregateOutputColumn * max(len(columns), 1))(*[capi.AggregateOutputColumn(k, i) for k, i in columns])
        table_handle = C.c_uint64()
        code = lib.hyb_aggregate_result_table(ptr, result, array, len(columns), chunk_size,
                                              C.byref(table_handle) if out else None)
        if code == capi.HYB_OK:
            capi.check(lib.hyb_table_drop(ptr, table_handle.value))
        return code

    assert status([(AGG, 0), (COL, 0)]) == capi.HYB_OK
    assert status([]) == capi.HYB_ERR_INVALID
    assert status([(7, 0)]) == capi.HYB_ERR_INVALID
    assert status([(AGG, 3)]) == capi.HYB_ERR_INVALID
    assert status([(COL, 3)]) == capi.HYB_ERR_INVALID
    assert status([(AGG, 0)], chunk_size=0) == capi.HYB_ERR_INVALID
    assert status([(AGG, 0)], result=handle + 1000) == capi.HYB_ERR_INVALID
    assert status([(AGG, 0)], out=False) == capi.HYB_ERR_INVALID
    assert lib.hyb_aggregate_result_table(ptr, handle, None, 1, 16, C.byref(C.c_uint64())) == capi.HYB_ERR_INVALID
    assert status([(AGG, 1)]) == capi.HYB_ERR_INVALID  # ANY: through COL instead
    assert status([(COL, 1)]) == capi.HYB_OK
    assert status([(AGG, 2)]) == capi.HYB_ERR_UNSUPPORTED  # string MIN
    assert status([(COL, 2)]) == capi.HYB_ERR_UNSUPPORTED  # string column
    table_dev.drop()
    assert status([(COL, 0)]) == capi.HYB_ERR_INVALID  # the aggregated table is gone
    assert status([(AGG, 0)]) == capi.HYB_OK
    device.free_aggregate_result(handle)
    assert status([(AGG, 0)]) == capi.HYB_ERR_INVALID


def test_cpp_mirror():
    build = subprocess.run(["make", "-C", REPO, "build/aggregate_table_check"], capture_output=True, text=True)
    assert build.returncode == 0, build.stdout + build.stderr
    run = subprocess.run([os.path.join(REPO, "build", "aggregate_table_check")], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0, run.stdout + run.stderr
    assert "aggregate_table_check: ok" in run.stdout


# ---- TPC-H ----------------------------------------------------------------------------------------------------------------
def load(name, columns, chunk_size, encoding="Automatic"):
    data = np.load(os.path.join(REPO, "tests", "golden", "tpch", f"sf-0.01_{name}.npz"))
    types = {"S": capi.TYPE_STRING, "f": capi.TYPE_FLOAT32, "i": capi.TYPE_INT32}
    definitions = [ColumnDefinition(column, types[data[column].dtype.kind]) for column in columns]
    return Table.from_columns(definitions, [data[column] for column in columns], chunk_size=chunk_size).encode(encoding), data


Q18_SQL = """SELECT c_custkey, o_orderkey, o_orderdate, o_totalprice, SUM(l_quantity)
      FROM customer, orders, lineitem WHERE o_orderkey in (SELECT l_orderkey FROM lineitem
      GROUP BY l_orderkey having SUM(l_quantity) > ?) AND c_custkey = o_custkey AND o_orderkey = l_orderkey
      GROUP BY c_custkey, o_orderkey, o_orderdate, o_totalprice ORDER BY o_totalprice DESC, o_orderdate
      LIMIT 100"""


@pytest.mark.parametrize("quantity,expected_orders", [(300, 2), (250, 67)])
def test_q18_against_sqlite(device, quantity, expected_orders):
    """The reference's Q18 text without c_name (it follows c_custkey; the fixtures hold no names)."""
    lineitem, lineitem_data = load("lineitem", ["l_orderkey", "l_quantity"], 10_000)
    orders, orders_data = load("orders_totalprice", ["o_orderkey", "o_custkey", "o_orderdate", "o_totalprice"], 4_000)
    lineitem_dev, orders_dev = device.upload(lineitem), device.upload(orders)
    device.set_string_order(orders_dev, 2)
    sum_quantity = [Aggregate(capi.AGG_SUM, on(1))]
    # SELECT l_orderkey ... GROUP BY l_orderkey HAVING SUM(l_quantity) > quantity, as a table
    per_order = device.aggregate_hash(lineitem_dev, [0], sum_quantity, keep_result=True)
    per_order_table = device.aggregate_table(per_order.result_handle, [(COL, 0), (AGG, 0)])
    device.free_aggregate_result(per_order.result_handle)
    having = device.table_scan(per_order_table, Predicate(1, capi.PRED_GREATER_THAN, quantity))
    # o_orderkey IN (...): a semi join of orders onto the HAVING rows
    big_orders = device.join_hash(per_order_table, 0, orders_dev, 0, capi.JOIN_SEMI, build_filter=having).pos_list(1)
    assert big_orders.info()[0] == expected_orders
    # orders |x| lineitem, then GROUP BY o_orderkey, SUM(l_quantity) as a table joined back to orders
    lines = device.join_hash(orders_dev, 0, lineitem_dev, 0, capi.JOIN_INNER, build_filter=big_orders).pos_list(1)
    per_big_order = device.aggregate_hash(lineitem_dev, [0], sum_quantity, input_filter=lines, keep_result=True)
    sums_table = device.aggregate_table(per_big_order.result_handle, [(COL, 0), (AGG, 0)])
    device.free_aggregate_result(per_big_order.result_handle)
    back = device.join_hash(sums_table, 0, orders_dev, 0, capi.JOIN_INNER, probe_filter=big_orders)
    sums_rows, order_rows = back.to_host()
    ordered = device.sort(orders_dev, [(3, True), (2, False)], input_filter=back.pos_list(1)).to_host()[:100]
    # read the result rows on the host: the sums through the derived table's RowIDs of each joined pair
    sums_values = expected_table(lineitem, per_big_order, [(COL, 0), (AGG, 0)], capi.DEFAULT_CHUNK_SIZE).column_values(1)[0]
    sum_of_order_row = {(int(o["chunk_id"]), int(o["chunk_offset"])):
                        sums_values[int(s["chunk_id"]) * capi.DEFAULT_CHUNK_SIZE + int(s["chunk_offset"])]
                        for s, o in zip(sums_rows, order_rows)}
    got = []
    for row in ordered:
        position = int(row["chunk_id"]) * 4_000 + int(row["chunk_offset"])
        got.append((int(orders_data["o_custkey"][position]), int(orders_data["o_orderkey"][position]),
                    orders_data["o_orderdate"][position].decode(), float(orders_data["o_totalprice"][position]),
                    float(sum_of_order_row[(int(row["chunk_id"]), int(row["chunk_offset"]))])))

    connection = sqlite3.connect(":memory:")
    customer_data = np.load(os.path.join(REPO, "tests", "golden", "tpch", "sf-0.01_customer.npz"))
    connection.execute("CREATE TABLE customer (c_custkey INTEGER)")
    connection.executemany("INSERT INTO customer VALUES (?)", [(int(k),) for k in customer_data["c_custkey"]])
    connection.execute("CREATE TABLE orders (o_orderkey INTEGER, o_custkey INTEGER, o_orderdate TEXT, o_totalprice REAL)")
    connection.executemany("INSERT INTO orders VALUES (?, ?, ?, ?)", zip(
        orders_data["o_orderkey"].tolist(), orders_data["o_custkey"].tolist(),
        [d.decode() for d in orders_data["o_orderdate"]], orders_data["o_totalprice"].astype(np.float64).tolist()))
    connection.execute("CREATE TABLE lineitem (l_orderkey INTEGER, l_quantity REAL)")
    connection.executemany("INSERT INTO lineitem VALUES (?, ?)", zip(
        lineitem_data["l_orderkey"].tolist(), lineitem_data["l_quantity"].astype(np.float64).tolist()))
    want = connection.execute(Q18_SQL, (quantity,)).fetchall()
    assert len(got) == len(want) == expected_orders
    assert [row[:4] for row in got] == [tuple(row[:4]) for row in want]
    assert np.allclose([row[4] for row in got], [row[4] for row in want], rtol=1e-9, atol=0)


Q15_SQL = """WITH revenue_view (supplier_no, total_revenue) AS (SELECT l_suppkey,
      SUM(l_extendedprice * (1 - l_discount)) FROM lineitem WHERE l_shipdate >= '1996-01-01'
      AND l_shipdate < '1996-04-01' GROUP BY l_suppkey)
      SELECT s_suppkey, s_name, total_revenue FROM supplier, revenue_view
      WHERE s_suppkey = supplier_no AND total_revenue = (SELECT max(total_revenue)
      FROM revenue_view) ORDER BY s_suppkey"""


def test_q15_against_sqlite(device):
    """The reference's Q15 view as a WITH clause (SQLite), without s_address / s_phone (not in the fixtures)."""
    keys = np.load(os.path.join(REPO, "tests", "golden", "tpch", "sf-0.01_lineitem_keys.npz"))
    base, data = load("lineitem", ["l_extendedprice", "l_discount", "l_shipdate"], 10_000)
    definitions = base.column_definitions + [ColumnDefinition("l_suppkey", capi.TYPE_INT32)]
    lineitem = Table.from_columns(definitions, [data["l_extendedprice"], data["l_discount"], data["l_shipdate"],
                                                keys["l_suppkey"]], chunk_size=10_000).encode("Automatic")
    supplier, supplier_data = load("supplier", ["s_suppkey", "s_name"], 40)
    lineitem_dev, supplier_dev = device.upload(lineitem), device.upload(supplier)
    revenue = Aggregate(capi.AGG_SUM, Expression([("col", 0), ("lit", capi.TYPE_FLOAT64, 1.0), ("col", 1), "-", "*"]))
    window = device.table_scan(lineitem_dev, Predicate(2, capi.PRED_BETWEEN_UPPER_EXCLUSIVE, b"1996-01-01", b"1996-04-01"))
    view = device.aggregate_hash(lineitem_dev, [3], [revenue], input_filter=window, keep_result=True)
    view_table = device.aggregate_table(view.result_handle, [(COL, 3), (AGG, 0)])
    device.free_aggregate_result(view.result_handle)
    # SELECT max(total_revenue) FROM revenue_view, read back as the literal of an equality scan
    maximum = device.aggregate_hash(view_table, [], [Aggregate(capi.AGG_MAX, on(1))])
    top = device.table_scan(view_table, Predicate(1, capi.PRED_EQUALS, float(maximum.values[0][0])))
    joined = device.join_hash(view_table, 0, supplier_dev, 0, capi.JOIN_INNER, build_filter=top)
    ordered = device.sort(supplier_dev, [(0, False)], input_filter=joined.pos_list(1)).to_host()
    got = [(int(supplier_data["s_suppkey"][int(r["chunk_id"]) * 40 + int(r["chunk_offset"])]),
            supplier_data["s_name"][int(r["chunk_id"]) * 40 + int(r["chunk_offset"])].decode(), float(maximum.values[0][0]))
           for r in ordered]

    connection = sqlite3.connect(":memory:")
    connection.execute("CREATE TABLE lineitem (l_suppkey INTEGER, l_extendedprice REAL, l_discount REAL, l_shipdate TEXT)")
    connection.executemany("INSERT INTO lineitem VALUES (?, ?, ?, ?)", zip(
        keys["l_suppkey"].tolist(), data["l_extendedprice"].astype(np.float64).tolist(),
        data["l_discount"].astype(np.float64).tolist(), [d.decode() for d in data["l_shipdate"]]))
    connection.execute("CREATE TABLE supplier (s_suppkey INTEGER, s_name TEXT)")
    connection.executemany("INSERT INTO supplier VALUES (?, ?)", zip(
        supplier_data["s_suppkey"].tolist(), [n.decode() for n in supplier_data["s_name"]]))
    want = connection.execute(Q15_SQL).fetchall()
    assert len(got) == len(want) >= 1
    assert [row[:2] for row in got] == [tuple(row[:2]) for row in want]
    assert np.allclose([row[2] for row in got], [row[2] for row in want], rtol=1e-6, atol=0)
