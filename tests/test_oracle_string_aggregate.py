"""Pins the string MIN / MAX / COUNT and ANY restatement (string_aggregate_oracle) to the reference's golden tables of
aggregate_test.cpp and to the DISTINCT path's groups. CPU only."""
import numpy as np
import pytest

import oracle_lib as orc
import string_aggregate_oracle as sorc
from helpers import assert_rows_match_unordered, expected_rows, tbl
from hyrise_b200 import capi
from hyrise_b200.device import Aggregate, Expression, Predicate
from string_aggregate_cases import ANY_MULTIPLE_ENTRIES_VALUE, CASES


def make_aggregates(definitions):
    return [Aggregate(function, Expression.column(column)) for column, function in definitions]


def case_inputs(case):
    """(table, input filter of the *OnRef tests or None) of a restated case."""
    _, _, input_file, chunk_size, dictionary, _, _, _, _, prefilter = case
    table = tbl(input_file, chunk_size)
    if dictionary:
        table.encode("Dictionary")
    return table, (orc.table_scan(table, Predicate(*prefilter)) if prefilter else None)


def case_rows(case, table, output):
    """The rows to compare with the golden table (AnyOnGroupWithMultipleEntries: the ANY value of each group)."""
    groupby = case[6]
    if case[7] is None:
        return [(row[-1],) for row in sorc.rows(table, groupby, output)]
    return sorc.rows(table, groupby, output)


def case_expected(case):
    return [(ANY_MULTIPLE_ENTRIES_VALUE,)] if case[7] is None else expected_rows(tbl(case[7]))


@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}@{c[1]}" for c in CASES])
def test_reference_golden_tables(case):
    _, _, _, _, _, definitions, groupby, _, on_reference_table, _ = case
    table, prefilter = case_inputs(case)
    output = sorc.aggregate_hash(table, groupby, make_aggregates(definitions), input_filter=prefilter)
    assert_rows_match_unordered(case_rows(case, table, output), case_expected(case))
    if on_reference_table and table.column_definitions[0].data_type != capi.TYPE_STRING:
        scan = orc.table_scan(table, Predicate(0, capi.PRED_GREATER_THAN, 0), prefilter)
        output = sorc.aggregate_hash(table, groupby, make_aggregates(definitions), input_filter=scan)
        assert_rows_match_unordered(case_rows(case, table, output), case_expected(case))


def test_any_only_is_the_distinct_path():
    """An all-ANY query has the groups, group order and representative RowIDs of the group-by-only query. Without a
    group-by column every row has the empty key: one group, represented by the first input row, and no group for an
    empty input (no aggregate functions, so no row is synthesised, aggregate_hash.cpp:1209-1217, :1422)."""
    table = tbl("aggregateoperator/groupby_int_1gb_1agg/input.tbl", 2)
    any_b = [Aggregate(capi.AGG_ANY, Expression.column(1))]
    for groupby in ([0], []):
        distinct = orc.aggregate_hash(table, groupby, [])
        output = sorc.aggregate_hash(table, groupby, any_b)
        assert output.group_count == distinct.group_count
        assert np.array_equal(output.row_ids, distinct.row_ids)
    output = sorc.aggregate_hash(table, [], any_b)
    assert output.group_count == 1 and output.row_ids[0]["chunk_id"] == 0 and output.row_ids[0]["chunk_offset"] == 0
    none = Predicate(0, capi.PRED_GREATER_THAN, 10 ** 6)
    assert sorc.aggregate_hash(table, [], any_b, predicates=[none]).group_count == 0


def test_bytes_order_is_char_traits():
    """Python bytes order: unsigned, a proper prefix first, embedded NUL an ordinary byte."""
    assert sorted([b"\xff", b"a", b"", b"a\0", b"a\0b", b"\x80", b"A"]) == [b"", b"A", b"a", b"a\0", b"a\0b", b"\x80", b"\xff"]
