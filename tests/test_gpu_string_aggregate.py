"""MIN / MAX / COUNT over string columns and the ANY pseudo-aggregate on the device. Expected values are computed with
Python bytes (unsigned, a proper prefix first, as char_traits<char>::compare) per group; groups, their order and the
representative RowIDs must equal those of the same call without the string aggregates."""
import ctypes as C

import numpy as np
import pytest

from helpers import row_ids_equal
from hyrise_b200 import capi
from hyrise_b200.device import Aggregate, DevicePeerGroup, Expression, Predicate, string_values
from hyrise_b200.storage import ColumnDefinition, Table
from test_oracle_aggregate import Q1_AGGREGATES, Q1_PREDICATES, lineitem_table

pytestmark = pytest.mark.gpu

WORDS = [b"", b"a\0b", b"a", b"ab", b"abc", b"\xff", b"\xff\xff", b"\x7f", b"\x80", b"b", b"A", b"zz", b"\0x"]


def make_table(rows, chunk_size, distinct, seed, bitpacking=False, null_every=5, all_null_chunk=False):
    rng = np.random.default_rng(seed)
    pool = WORDS + [b"w%06d" % i for i in range(max(distinct - len(WORDS), 0))]
    picks = rng.permutation(rows) % len(pool) if rows >= len(pool) else rng.integers(0, len(pool), rows)
    strings = np.array([pool[i] for i in picks], dtype=object)
    groups = rng.integers(0, 4, rows).astype(np.int32)
    values = rng.integers(-50, 50, rows).astype(np.int32)
    nulls = np.zeros(rows, dtype=bool)
    if null_every:
        nulls[::null_every] = True
        nulls[groups == 3] = True  # group 3: no non-NULL string
    if all_null_chunk and rows > chunk_size:
        nulls[:chunk_size] = True
    definitions = [ColumnDefinition("g", capi.TYPE_INT32), ColumnDefinition("s", capi.TYPE_STRING, True),
                   ColumnDefinition("v", capi.TYPE_INT32), ColumnDefinition("l", capi.TYPE_INT64),
                   ColumnDefinition("f", capi.TYPE_FLOAT32), ColumnDefinition("d", capi.TYPE_FLOAT64)]
    columns = [groups, np.array(list(strings), dtype="S"), values, values.astype(np.int64) * 3, values.astype(np.float32) / 4,
               values.astype(np.float64) / 8]
    table = Table.from_columns(definitions, columns, [None, nulls, None, None, None, None], chunk_size=chunk_size)
    return table.encode("Dictionary", bitpacking=bitpacking)


def expected_strings(table, output, groupby, column, function, positions=None):
    """Per group of `output`: MIN / MAX (bytes or None) or COUNT of the string column over the rows in `positions`."""
    keys = [table.column_values(g) for g in groupby]
    strings, nulls = table.column_values(column)
    starts = np.cumsum([0] + [chunk.size for chunk in table.chunks])
    group_of = {(): 0}
    for index, row_id in enumerate(output.row_ids if groupby else []):
        position = starts[row_id["chunk_id"]] + row_id["chunk_offset"]
        group_of[tuple((bool(k[1][position]), k[0][position] if not k[1][position] else None) for k in keys)] = index
    rows = range(len(strings)) if positions is None else positions
    per_group = [[] for _ in range(output.group_count)]
    for position in rows:
        key = tuple((bool(k[1][position]), k[0][position] if not k[1][position] else None) for k in keys)
        if not nulls[position]:
            per_group[group_of[key]].append(bytes(strings[position]))
    if function == capi.AGG_COUNT:
        return [len(values) for values in per_group]
    pick = min if function == capi.AGG_MIN else max
    return [pick(values) if values else None for values in per_group]


def check_strings(device, table, device_table, groupby, predicates=(), input_filter=None, positions=None):
    aggregates = [Aggregate(capi.AGG_MIN, Expression.column(1)), Aggregate(capi.AGG_MAX, Expression.column(1)),
                  Aggregate(capi.AGG_COUNT, Expression.column(1))]
    baseline = device.aggregate_hash(device_table, groupby, [Aggregate(capi.AGG_COUNT_STAR)], predicates, input_filter)
    got = device.aggregate_hash(device_table, groupby, aggregates, predicates, input_filter)
    assert device.last_stats().path in (capi.AGG_PATH_GENERAL, capi.AGG_PATH_GENERAL_REGROWN)
    assert got.group_count == baseline.group_count and row_ids_equal(got.row_ids, baseline.row_ids)
    if got.group_count == 0:
        return got
    assert got.value_types[:2] == [capi.TYPE_STRING, capi.TYPE_STRING] and got.value_types[2] == capi.TYPE_INT64
    for index, function in enumerate((capi.AGG_MIN, capi.AGG_MAX)):
        assert string_values(table, 1, got.values[index], got.nulls[index]) == \
            expected_strings(table, got, groupby, 1, function, positions)
    assert got.values[2].tolist() == expected_strings(table, got, groupby, 1, capi.AGG_COUNT, positions)
    return got


LAYOUTS = [  # rows, chunk size, distinct strings, bitpacking
    (5_000, 1_000, 40, False),      # FixedWidth 1 byte
    (9_000, 3_000, 2_000, False),   # FixedWidth 2 bytes
    (80_000, 80_000, 80_000, False),  # FixedWidth 4 bytes (no NULLs, every string distinct)
    (7_000, 700, 300, True),        # BitPacking
]


@pytest.mark.parametrize("layout", LAYOUTS, ids=["fixed1", "fixed2", "fixed4", "bitpacked"])
def test_layouts(device, layout):
    rows, chunk_size, distinct, bitpacking = layout
    table = make_table(rows, chunk_size, distinct, seed=rows, bitpacking=bitpacking, all_null_chunk=True,
                       null_every=0 if distinct > 65_536 else 5)
    device_table = device.upload(table)
    try:
        device.set_string_order(device_table, 1)
        for groupby in ([0], [], [0, 2]):
            check_strings(device, table, device_table, groupby)
    finally:
        device_table.drop()


def test_overlapping_chunks_and_filters(device):
    table = make_table(20_000, 1_500, 120, seed=7)
    device_table = device.upload(table)
    try:
        device.set_string_order(device_table, 1)
        check_strings(device, table, device_table, [0])
        # scan PosList
        predicate = Predicate(2, capi.PRED_GREATER_THAN, 10)
        scan = device.table_scan(device_table, predicate)
        values, _ = table.column_values(2)
        check_strings(device, table, device_table, [0], input_filter=scan, positions=np.flatnonzero(values > 10))
        # fused predicates, LIKE included
        like = Predicate(1, capi.PRED_LIKE, b"a%")
        strings, nulls = table.column_values(1)
        keep = [i for i in range(len(strings)) if not nulls[i] and bytes(strings[i]).startswith(b"a") and values[i] > 10]
        check_strings(device, table, device_table, [0], predicates=[like, predicate], positions=keep)
        # the probe side of an inner join with the rows v == 0 (join order, repeated rows)
        zero = device.table_scan(device_table, Predicate(2, capi.PRED_EQUALS, 0))
        join = device.join_hash(device_table, 2, device_table, 2, capi.JOIN_INNER, build_filter=zero)
        probe = join.pos_list(1)
        starts = np.cumsum([0] + [c.size for c in table.chunks])
        check_strings(device, table, device_table, [0], input_filter=probe,
                      positions=[int(starts[r["chunk_id"]] + r["chunk_offset"]) for r in probe.to_host()])
    finally:
        device_table.drop()


def test_empty_input(device):
    table = make_table(1_000, 500, 10, seed=3)
    device_table = device.upload(table)
    try:
        device.set_string_order(device_table, 1)
        none = Predicate(2, capi.PRED_GREATER_THAN, 1000)
        got = check_strings(device, table, device_table, [], predicates=[none], positions=[])
        assert got.group_count == 1 and got.nulls[0][0] and got.nulls[1][0] and got.values[2][0] == 0
        assert check_strings(device, table, device_table, [0], predicates=[none], positions=[]).group_count == 0
    finally:
        device_table.drop()


def test_any(device):
    table = make_table(12_000, 2_000, 50, seed=11)
    device_table = device.upload(table)
    try:
        any_columns = [Aggregate(capi.AGG_ANY, Expression.column(c)) for c in (1, 2, 3, 4, 5)]
        baseline = device.aggregate_hash(device_table, [0], [])
        path = device.last_stats().path
        got = device.aggregate_hash(device_table, [0], any_columns)
        assert device.last_stats().path == path
        assert got.group_count == baseline.group_count and row_ids_equal(got.row_ids, baseline.row_ids)
        assert got.values == [None] * 5 and got.value_types == [capi.TYPE_STRING, capi.TYPE_INT32, capi.TYPE_INT64,
                                                                   capi.TYPE_FLOAT32, capi.TYPE_FLOAT64]
        # mixed: the other aggregates equal the call without ANY, in the same kernel
        plain = [Aggregate(capi.AGG_SUM, Expression.column(2)), Aggregate(capi.AGG_MIN, Expression.column(5))]
        without = device.aggregate_hash(device_table, [0], plain)
        path = device.last_stats().path
        mixed = device.aggregate_hash(device_table, [0], [any_columns[0], plain[0], any_columns[3], plain[1]])
        assert device.last_stats().path == path
        assert row_ids_equal(mixed.row_ids, without.row_ids)
        assert mixed.values[1].tolist() == without.values[0].tolist() and mixed.values[3].tolist() == without.values[1].tolist()
        # no group-by: one group for a non-empty input, none for an empty one
        only = device.aggregate_hash(device_table, [], any_columns[:1])
        assert only.group_count == 1 and only.row_ids[0]["chunk_id"] == 0 and only.row_ids[0]["chunk_offset"] == 0
        none = Predicate(2, capi.PRED_GREATER_THAN, 1000)
        assert device.aggregate_hash(device_table, [], any_columns[:1], predicates=[none]).group_count == 0
        # ANY must name a single column
        with pytest.raises(capi.HyriseB200Error) as error:
            device.aggregate_hash(device_table, [0], [Aggregate(capi.AGG_ANY, Expression([("col", 2), ("col", 2), "+"]))])
        assert error.value.status == capi.HYB_ERR_INVALID
    finally:
        device_table.drop()


def test_q1_with_any_keeps_its_path(device):
    table, _ = lineitem_table()
    device_table = device.upload(table)
    try:
        plain = device.aggregate_hash(device_table, [5, 6], Q1_AGGREGATES, predicates=Q1_PREDICATES)
        path = device.last_stats().path
        got = device.aggregate_hash(device_table, [5, 6], Q1_AGGREGATES + [Aggregate(capi.AGG_ANY, Expression.column(5))],
                                    predicates=Q1_PREDICATES)
        assert device.last_stats().path == path
        assert row_ids_equal(got.row_ids, plain.row_ids)
        for a, b in zip(got.values[:-1], plain.values):
            assert np.array_equal(a, b)
    finally:
        device_table.drop()


def test_declines_and_validation(device):
    table = make_table(3_000, 1_000, 30, seed=5)
    device_table = device.upload(table)
    try:
        min_string = [Aggregate(capi.AGG_MIN, Expression.column(1))]
        with pytest.raises(capi.UnsupportedOnDevice):  # no ranks attached
            device.aggregate_hash(device_table, [0], min_string)
        device.aggregate_hash(device_table, [0], [Aggregate(capi.AGG_COUNT, Expression.column(1))])  # COUNT needs none
        for function in (capi.AGG_SUM, capi.AGG_AVG):
            with pytest.raises(capi.UnsupportedOnDevice):
                device.aggregate_hash(device_table, [0], [Aggregate(function, Expression.column(1))])
        ranks = table.string_order_ranks(1)

        def attach(words, column=1):
            words = np.ascontiguousarray(words, dtype=np.uint32)
            return device.lib.hyb_table_set_string_order(device.ptr, device_table.handle, column,
                                                         words.ctypes.data_as(C.POINTER(C.c_uint32)), len(words))

        bad = ranks.copy()
        bad[1], bad[0] = bad[0], bad[1]
        big = ranks.copy()
        big[-1] = 1 << 31
        for status in (attach(ranks[:-1]), attach(bad), attach(big), attach(ranks, column=2)):
            assert status == capi.HYB_ERR_INVALID
        assert attach(ranks) == capi.HYB_OK
        device.aggregate_hash(device_table, [0], min_string)
        # appending a chunk drops the ranks
        holder = table.view()
        assert device.lib.hyb_table_append_chunk(device.ptr, device_table.handle, holder.chunk_descs(0)) == capi.HYB_OK
        with pytest.raises(capi.UnsupportedOnDevice):
            device.aggregate_hash(device_table, [0], min_string)
        device.set_string_order(device_table, 1, np.concatenate([ranks, ranks[: table.chunks[0].segments[1].dictionary_size]]))
        device.aggregate_hash(device_table, [0], min_string)
        # ANY has no values; its index in hyb_aggregate_result_values is an error
        result = device.aggregate_hash(device_table, [0], [Aggregate(capi.AGG_ANY, Expression.column(1))], keep_result=True)
        raw = np.zeros(max(result.group_count, 1), dtype=np.uint64)
        kind = C.c_int32()
        assert device.lib.hyb_aggregate_result_values(device.ptr, result.result_handle, 0, raw.ctypes.data, None,
                                                      C.byref(kind)) == capi.HYB_ERR_INVALID
        assert b"hyb_aggregate_result_row_ids" in device.lib.hyb_last_error()
        device.free_aggregate_result(result.result_handle)
        # a one-rank peer group declines the new forms before any exchange
        group = DevicePeerGroup(device, 0, 1, 1 << 16)
        try:
            for aggregates in (min_string, [Aggregate(capi.AGG_COUNT, Expression.column(1))],
                               [Aggregate(capi.AGG_ANY, Expression.column(2))]):
                with pytest.raises(capi.UnsupportedOnDevice):
                    group.aggregate_hash(device_table, [0], aggregates)
        finally:
            group.destroy()
    finally:
        device_table.drop()


# ---- the aggregate_test.cpp cases against the restatement (string_aggregate_oracle), on base and scan-output tables ----
import sqlite3  # noqa: E402

import oracle_lib as orc  # noqa: E402
import string_aggregate_oracle as sorc  # noqa: E402
from helpers import assert_rows_match_unordered, column_values_at  # noqa: E402
from string_aggregate_cases import CASES  # noqa: E402
from test_oracle_string_aggregate import case_expected, case_inputs, case_rows, make_aggregates  # noqa: E402


def device_output_rows(device, table, device_table, groupby, aggregates, predicates=(), input_filter=None):
    """The device's result in the restatement's form (strings as bytes, ANY through the representative RowIDs)."""
    got = device.aggregate_hash(device_table, groupby, aggregates, predicates, input_filter)
    for index, aggregate in enumerate(aggregates):
        column = aggregate.expression.nodes[0][1] if aggregate.expression else None
        if aggregate.function == capi.AGG_ANY:
            got.values[index] = column_values_at(table, column, got.row_ids) if got.group_count else []
            got.nulls[index] = np.array([cell is None for cell in got.values[index]], dtype=bool)
        elif got.value_types[index] == capi.TYPE_STRING:
            got.values[index] = string_values(table, column, got.values[index], got.nulls[index])
    return got



@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}@{c[1]}" for c in CASES])
def test_reference_cases(device, case):
    _, _, _, _, _, definitions, groupby, _, on_reference_table, prefilter = case
    table, host_prefilter = case_inputs(case)
    aggregates = make_aggregates(definitions)
    device_table = device.upload(table)
    try:
        for column, function in definitions:
            if function in (capi.AGG_MIN, capi.AGG_MAX) and table.column_definitions[column].data_type == capi.TYPE_STRING:
                device.set_string_order(device_table, column)
        device_prefilter = device.table_scan(device_table, Predicate(*prefilter)) if prefilter else None
        inputs = [(device_prefilter, host_prefilter)]
        if on_reference_table and table.column_definitions[0].data_type != capi.TYPE_STRING:
            positive = Predicate(0, capi.PRED_GREATER_THAN, 0)
            inputs.append((device.table_scan(device_table, positive, device_prefilter),
                           orc.table_scan(table, positive, host_prefilter)))
        for device_filter, host_filter in inputs:
            expected = sorc.aggregate_hash(table, groupby, aggregates, input_filter=host_filter)
            got = device_output_rows(device, table, device_table, groupby, aggregates, input_filter=device_filter)
            assert got.group_count == expected.group_count and row_ids_equal(got.row_ids, expected.row_ids)
            assert sorc.rows(table, groupby, got) == sorc.rows(table, groupby, expected)
            assert_rows_match_unordered(case_rows(case, table, got), case_expected(case))
    finally:
        device_table.drop()


def test_first_entry_of_each_rank(device):
    """Dictionaries built to be disjoint, overlapping and late-only: a string MIN / MAX names the first {chunk, value-ID}
    in chunk order whose dictionary holds the string, whichever rows of the group held it."""
    strings = [b"m", b"n", b"m", b"b", b"z", b"b", b"a", b"zz", b"a", b"a", b"zzz", b"q"]
    groups = np.array([0, 0, 0, 1, 1, 1, 1, 1, 1, 0, 0, 0], dtype=np.int32)
    definitions = [ColumnDefinition("g", capi.TYPE_INT32), ColumnDefinition("s", capi.TYPE_STRING)]
    table = Table.from_columns(definitions, [groups, np.array(strings, dtype="S")], chunk_size=3).encode("Dictionary")
    device_table = device.upload(table)
    try:
        device.set_string_order(device_table, 1)
        got = device.aggregate_hash(device_table, [0], [Aggregate(capi.AGG_MIN, Expression.column(1)),
                                                         Aggregate(capi.AGG_MAX, Expression.column(1))])
        assert got.group_count == 2
        positions = [[(int(p["chunk_id"]), int(p["value_id"])) for p in values] for values in got.values]
        # group 0 = chunks 0 and 3: "a" first held by chunk 2, "zzz" only by chunk 3; group 1 = chunks 1 and 2
        assert positions[0] == [(2, 0), (2, 0)] and positions[1] == [(3, 2), (2, 1)]
        assert string_values(table, 1, got.values[1], got.nulls[1]) == [b"zzz", b"zz"]
    finally:
        device_table.drop()


def assert_sqlite(device, table, device_table, groupby, aggregates, sql, connection, predicates=(), input_filter=None):
    got = device_output_rows(device, table, device_table, groupby, aggregates, predicates, input_filter)
    want = [tuple(cell.encode() if isinstance(cell, str) else cell for cell in row) for row in connection.execute(sql)]
    assert_rows_match_unordered(sorc.rows(table, groupby, got), want)


def test_tpch_against_sqlite(device):
    """SQLite's BINARY collation compares with memcmp, the order of char_traits<char>::compare."""
    connection = sqlite3.connect(":memory:")
    text = lambda column: [v.decode() for v in column]  # noqa: E731

    dates = np.load("tests/golden/tpch/sf-0.01_lineitem_dates.npz")
    names = ["l_shipmode", "l_shipdate", "l_receiptdate", "l_commitdate"]
    table = Table.from_columns([ColumnDefinition(n, capi.TYPE_STRING) for n in names], [dates[n] for n in names],
                               chunk_size=10_000).encode("Dictionary")
    connection.execute("create table lineitem (l_shipmode text, l_shipdate text, l_receiptdate text, l_commitdate text)")
    connection.executemany("insert into lineitem values (?,?,?,?)", zip(*[text(dates[n]) for n in names]))
    device_table = device.upload(table)
    device.set_string_order(device_table, 1)
    device.set_string_order(device_table, 2)
    assert_sqlite(device, table, device_table, [0], make_aggregates([(1, capi.AGG_MIN), (2, capi.AGG_MAX), (3, capi.AGG_COUNT)]),
                  "select l_shipmode, min(l_shipdate), max(l_receiptdate), count(l_commitdate) from lineitem group by 1",
                  connection)
    device_table.drop()

    comments = np.load("tests/golden/tpch/sf-0.01_orders_comment.npz")
    table = Table.from_columns([ColumnDefinition("o_comment", capi.TYPE_STRING)], [comments["o_comment"]],
                               chunk_size=4_000).encode("Dictionary")
    connection.execute("create table orders_comment (o_comment text)")
    connection.executemany("insert into orders_comment values (?)", [(v,) for v in text(comments["o_comment"])])
    device_table = device.upload(table)
    device.set_string_order(device_table, 0)
    assert_sqlite(device, table, device_table, [], make_aggregates([(0, capi.AGG_MIN), (0, capi.AGG_MAX)]),
                  "select min(o_comment), max(o_comment) from orders_comment where o_comment like '%special%requests%'",
                  connection, predicates=[Predicate(0, capi.PRED_LIKE, b"%special%requests%")])
    device_table.drop()

    part = np.load("tests/golden/tpch/sf-0.01_part.npz")
    names = ["p_container", "p_name", "p_type"]
    table = Table.from_columns([ColumnDefinition(n, capi.TYPE_STRING) for n in names], [part[n] for n in names],
                               chunk_size=700).encode("Dictionary")
    connection.execute("create table part (p_container text, p_name text, p_type text)")
    connection.executemany("insert into part values (?,?,?)", zip(*[text(part[n]) for n in names]))
    device_table = device.upload(table)
    device.set_string_order(device_table, 1)
    device.set_string_order(device_table, 2)
    assert_sqlite(device, table, device_table, [0], make_aggregates([(1, capi.AGG_MIN), (2, capi.AGG_MAX)]),
                  "select p_container, min(p_name), max(p_type) from part group by 1", connection)
    device_table.drop()

    # Q3 shape: GROUP BY o_orderkey with ANY(o_orderdate), ANY(o_shippriority) over customer ⋈ orders
    customer = np.load("tests/golden/tpch/sf-0.01_customer.npz")
    orders = np.load("tests/golden/tpch/sf-0.01_orders.npz")
    customers = Table.from_columns([ColumnDefinition("c_custkey", capi.TYPE_INT32), ColumnDefinition("c_mktsegment", capi.TYPE_STRING)],
                                   [customer["c_custkey"], customer["c_mktsegment"]], chunk_size=500).encode("Dictionary")
    order_names = ["o_orderkey", "o_custkey", "o_orderdate", "o_shippriority"]
    order_types = [capi.TYPE_INT32, capi.TYPE_INT32, capi.TYPE_STRING, capi.TYPE_INT32]
    order_table = Table.from_columns([ColumnDefinition(n, t) for n, t in zip(order_names, order_types)],
                                     [orders[n] for n in order_names], chunk_size=4_000).encode("Automatic")
    connection.execute("create table customer (c_custkey int, c_mktsegment text)")
    connection.executemany("insert into customer values (?,?)", zip(customer["c_custkey"].tolist(), text(customer["c_mktsegment"])))
    connection.execute("create table orders (o_orderkey int, o_custkey int, o_orderdate text, o_shippriority int)")
    connection.executemany("insert into orders values (?,?,?,?)", zip(orders["o_orderkey"].tolist(), orders["o_custkey"].tolist(),
                                                                     text(orders["o_orderdate"]), orders["o_shippriority"].tolist()))
    device_customers, device_orders = device.upload(customers), device.upload(order_table)
    building = device.table_scan(device_customers, Predicate(1, capi.PRED_EQUALS, b"BUILDING"))
    join = device.join_hash(device_customers, 0, device_orders, 1, capi.JOIN_INNER, build_filter=building)
    orders_side = join.pos_list(1)
    any_columns = [Aggregate(capi.AGG_ANY, Expression.column(2)), Aggregate(capi.AGG_ANY, Expression.column(3))]
    assert_sqlite(device, order_table, device_orders, [0], any_columns,
                  "select o_orderkey, o_orderdate, o_shippriority from customer join orders on c_custkey = o_custkey "
                  "where c_mktsegment = 'BUILDING' group by o_orderkey", connection, input_filter=orders_side)
    device_customers.drop()
    device_orders.drop()


def test_cpp_mirror_string_aggregate():
    import os
    import subprocess

    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    build = subprocess.run(["make", "-C", repo, "build/string_aggregate_check"], capture_output=True, text=True)
    assert build.returncode == 0, build.stdout + build.stderr
    environment = dict(os.environ, HYB_BINARY_FIXTURE=os.path.join(repo, "tests", "golden", "bin",
                                                                   "FixedStringDictionaryMultipleChunks.bin"))
    run = subprocess.run([os.path.join(repo, "build", "string_aggregate_check")], capture_output=True, text=True, timeout=120,
                         env=environment)
    assert run.returncode == 0 and run.stdout.strip() == "OK", run.stdout + run.stderr
