"""The string MIN / MAX / COUNT and ANY cases of src/test/lib/operators/aggregate_test.cpp (hyrise/hyrise @ 2f7bedf3),
restated like aggregate_distinct_cases.py (line numbers kept). Each case: (reference test name, source line, input .tbl,
chunk size, dictionary-encode the input?, [(column id, function)], group-by column ids, expected result .tbl, also run
on a TableScan-produced reference table?, scan that produced the test's input or None).

AnyOnGroupWithMultipleEntries has no result table: the test reads the ANY value of the one remaining group, 20
(ANY_MULTIPLE_ENTRIES_VALUE), from the output of TableScan(column 0 = 123) over the 2-group-by fixture.
"""
from hyrise_b200 import capi
from hyrise_b200.capi import AGG_ANY, AGG_COUNT, AGG_MAX, AGG_MIN

D = "aggregateoperator/"
LESS_THAN_100 = (0, capi.PRED_LESS_THAN, 100)
EQUALS_123 = (0, capi.PRED_EQUALS, 123)
ANY_MULTIPLE_ENTRIES_VALUE = 20

CASES = [
    ("AnyOnGroupWithMultipleEntries", 262, D + "groupby_int_2gb_2agg/input.tbl", 2, False, [(2, AGG_ANY)], [0, 1], None, False, EQUALS_123),
    ("AnyAndNulls", 280, D + "groupby_int_1gb_0agg/input_null.tbl", 2, False, [(0, AGG_ANY)], [1], D + "groupby_int_1gb_0agg/result_any_null.tbl", False, None),
    ("CanCountStringColumns", 285, D + "groupby_string_1gb_1agg/input.tbl", 2, False, [(0, AGG_COUNT)], [0], D + "groupby_string_1gb_1agg/count_str.tbl", True, None),
    ("StringSingleAggregateStringMax", 342, D + "groupby_string_1gb_1agg/input.tbl", 2, False, [(0, AGG_MAX)], [], D + "groupby_string_1gb_1agg/max_str.tbl", True, None),
    ("StringSingleAggregateStringMin", 347, D + "groupby_string_1gb_1agg/input.tbl", 2, False, [(0, AGG_MIN)], [], D + "groupby_string_1gb_1agg/min_str.tbl", True, None),
    ("DictionarySingleAggregateAnyOnRef", 812, D + "groupby_int_1gb_1agg/input.tbl", 2, True, [(1, AGG_ANY)], [0], D + "groupby_int_1gb_1agg/any_filtered.tbl", True, LESS_THAN_100),
]
