"""Pins the expected aggregate table (aggregate_table_expected.expected_table: the oracle's AggregateHash result with its
GROUP BY columns read at the representative rows, then the aggregates) to the reference's golden result tables
(src/test/lib/operators/aggregate_test.cpp -> resources/test_data/tbl/aggregateoperator/**). The device's
hyb_aggregate_result_table is compared with this table in test_gpu_aggregate_table.py. CPU only."""
import pytest

import oracle_lib as orc
from aggregate_cases import CASES
from aggregate_table_expected import expected_table
from helpers import assert_rows_match_unordered, expected_rows, tbl
from hyrise_b200 import capi
from hyrise_b200.device import Aggregate, Expression, Predicate

# the derived table holds numeric GROUP BY columns only (string columns share no dictionary across source chunks)
NUMERIC_CASES = [case for case in CASES
                 if all(tbl(case[2]).column_definitions[g].data_type != capi.TYPE_STRING for g in case[6])]


def make_aggregates(definitions):
    return [Aggregate(function, None if column is None else Expression.column(column)) for column, function in definitions]


def table_columns(groupby, aggregate_count):
    return [(capi.SORT_KEY_COLUMN, g) for g in groupby] + [(capi.SORT_KEY_AGGREGATE, a) for a in range(aggregate_count)]


@pytest.mark.parametrize("case", NUMERIC_CASES, ids=[f"{c[0]}@{c[1]}" for c in NUMERIC_CASES])
@pytest.mark.parametrize("chunk_size", [1, 3, capi.DEFAULT_CHUNK_SIZE])
def test_expected_table_equals_reference_golden_output(case, chunk_size):
    name, line, input_file, input_chunk_size, dictionary, definitions, groupby, expected_file, _ = case
    table = tbl(input_file, input_chunk_size)
    if dictionary:
        table.encode("Dictionary")
    output = orc.aggregate_hash(table, groupby, make_aggregates(definitions))
    derived = expected_table(table, output, table_columns(groupby, len(definitions)), chunk_size)
    assert derived.row_count == output.group_count
    assert all(chunk.size == chunk_size for chunk in derived.chunks[:-1])
    assert_rows_match_unordered(expected_rows(derived), expected_rows(tbl(expected_file)))


def test_expected_table_of_an_empty_input():
    """No GROUP BY over no rows: one row whose COUNT is 0 and whose column read at NULL_ROW_ID is NULL; with a GROUP BY:
    a table without chunks."""
    table = tbl("aggregateoperator/groupby_int_1gb_1agg/input.tbl", 2)
    nothing = orc.table_scan(table, Predicate(0, capi.PRED_GREATER_THAN, 10 ** 9))
    aggregates = make_aggregates([(1, capi.AGG_COUNT)])
    output = orc.aggregate_hash(table, [], aggregates, input_filter=nothing)
    derived = expected_table(table, output, [(capi.SORT_KEY_COLUMN, 1), (capi.SORT_KEY_AGGREGATE, 0)], 4)
    assert expected_rows(derived) == [(None, 0)]
    output = orc.aggregate_hash(table, [0], aggregates, input_filter=nothing)
    derived = expected_table(table, output, [(capi.SORT_KEY_COLUMN, 0), (capi.SORT_KEY_AGGREGATE, 0)], 4)
    assert derived.chunk_count == 0 and derived.row_count == 0
