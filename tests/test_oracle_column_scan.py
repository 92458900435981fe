"""Column-vs-column TableScan without a GPU: the numeric oracle against hand-derived expectations on the reference's .tbl
fixtures and on the rounding cases of C++'s arithmetic conversions; the host translation of string dictionaries
(hyb_dictionary_translate, hyb_binary_table_column_translation) against bisect."""
import bisect
import os
import random

import numpy as np
import pytest

import column_scan_oracle as cso
from helpers import tbl
from hyrise_b200 import capi
from hyrise_b200.binary_table import NativeBinaryTable, write_binary_table
from hyrise_b200.device import ColumnComparison
from hyrise_b200.storage import ColumnDefinition, Table

P = capi
CONDITIONS = [P.PRED_EQUALS, P.PRED_NOT_EQUALS, P.PRED_LESS_THAN, P.PRED_LESS_THAN_EQUALS, P.PRED_GREATER_THAN,
              P.PRED_GREATER_THAN_EQUALS]
# `a <op> b` == `b <flip(op)> a`
FLIPPED = {P.PRED_EQUALS: P.PRED_EQUALS, P.PRED_NOT_EQUALS: P.PRED_NOT_EQUALS, P.PRED_LESS_THAN: P.PRED_GREATER_THAN,
           P.PRED_LESS_THAN_EQUALS: P.PRED_GREATER_THAN_EQUALS, P.PRED_GREATER_THAN: P.PRED_LESS_THAN,
           P.PRED_GREATER_THAN_EQUALS: P.PRED_LESS_THAN_EQUALS}

# (fixture, left column, right column, matching rows per condition) — read off the fixture files by hand
FIXTURE_CASES = [
    ("int_int.tbl", 0, 1, {P.PRED_EQUALS: [], P.PRED_NOT_EQUALS: [0, 1, 2], P.PRED_LESS_THAN: [],
                           P.PRED_LESS_THAN_EQUALS: [], P.PRED_GREATER_THAN: [0, 1, 2],
                           P.PRED_GREATER_THAN_EQUALS: [0, 1, 2]}),
    ("int_float.tbl", 0, 1, {P.PRED_EQUALS: [], P.PRED_NOT_EQUALS: [0, 1, 2], P.PRED_LESS_THAN: [1],
                             P.PRED_LESS_THAN_EQUALS: [1], P.PRED_GREATER_THAN: [0, 2],
                             P.PRED_GREATER_THAN_EQUALS: [0, 2]}),
    ("float_int.tbl", 0, 1, {P.PRED_EQUALS: [], P.PRED_NOT_EQUALS: [0, 1, 2], P.PRED_LESS_THAN: [0, 2],
                             P.PRED_LESS_THAN_EQUALS: [0, 2], P.PRED_GREATER_THAN: [1],
                             P.PRED_GREATER_THAN_EQUALS: [1]}),
    *[("int_float_double_string.tbl", left, right,
       {P.PRED_EQUALS: list(range(6)), P.PRED_NOT_EQUALS: [], P.PRED_LESS_THAN: [],
        P.PRED_LESS_THAN_EQUALS: list(range(6)), P.PRED_GREATER_THAN: [], P.PRED_GREATER_THAN_EQUALS: list(range(6))})
      for left, right in [(0, 1), (0, 2), (1, 2), (0, 0), (2, 2)]],
    ("int_int_int_null.tbl", 0, 1, {P.PRED_EQUALS: [], P.PRED_NOT_EQUALS: [0], P.PRED_LESS_THAN: [0],
                                    P.PRED_LESS_THAN_EQUALS: [0], P.PRED_GREATER_THAN: [],
                                    P.PRED_GREATER_THAN_EQUALS: []}),
    ("int_int_int_null.tbl", 1, 2, {P.PRED_EQUALS: [1], P.PRED_NOT_EQUALS: [0], P.PRED_LESS_THAN: [0],
                                    P.PRED_LESS_THAN_EQUALS: [0, 1], P.PRED_GREATER_THAN: [],
                                    P.PRED_GREATER_THAN_EQUALS: [1]}),
    ("int_int_int_null.tbl", 0, 2, {P.PRED_EQUALS: [2], P.PRED_NOT_EQUALS: [0], P.PRED_LESS_THAN: [0],
                                    P.PRED_LESS_THAN_EQUALS: [0, 2], P.PRED_GREATER_THAN: [],
                                    P.PRED_GREATER_THAN_EQUALS: [2]}),
    ("int_float_with_null.tbl", 0, 1, {P.PRED_EQUALS: [], P.PRED_NOT_EQUALS: [0, 3], P.PRED_LESS_THAN: [],
                                       P.PRED_LESS_THAN_EQUALS: [], P.PRED_GREATER_THAN: [0, 3],
                                       P.PRED_GREATER_THAN_EQUALS: [0, 3]}),
]


def row_ids(rows, chunk_size):
    return [(row // chunk_size, row % chunk_size) for row in rows]


def as_tuples(pos_list):
    return [(int(r["chunk_id"]), int(r["chunk_offset"])) for r in pos_list.row_ids]


@pytest.mark.parametrize("encoding", ["Unencoded", "Dictionary", "Automatic"])
@pytest.mark.parametrize("chunk_size", [2, 3])
@pytest.mark.parametrize("case", FIXTURE_CASES, ids=lambda case: f"{case[0]}:{case[1]}-{case[2]}")
def test_numeric_fixtures(case, chunk_size, encoding):
    source, left, right, expected = case
    table = tbl(source, chunk_size).encode(encoding)
    for condition in CONDITIONS:
        got = cso.table_scan_columns(table, ColumnComparison(left, condition, right))
        assert as_tuples(got) == row_ids(expected[condition], chunk_size), condition
        # both operand orders: `right <flip(op)> left` selects the same rows
        swapped = cso.table_scan_columns(table, ColumnComparison(right, FLIPPED[condition], left))
        assert as_tuples(swapped) == row_ids(expected[condition], chunk_size), condition
        offsets = got.chunk_offsets
        assert len(offsets) == table.chunk_count + 1 and offsets[-1] == len(got.row_ids)


def test_string_and_number_is_invalid():
    table = tbl("int_float_double_string.tbl", 2).encode("Dictionary")
    with pytest.raises(capi.HyriseB200Error):
        cso.table_scan_columns(table, ColumnComparison(3, P.PRED_EQUALS, 0))


def pair_table(left_type, left, right_type, right, left_nulls=None, right_nulls=None, chunk_size=3):
    definitions = [ColumnDefinition("l", left_type, left_nulls is not None),
                   ColumnDefinition("r", right_type, right_nulls is not None)]
    return Table.from_columns(definitions, [np.array(left), np.array(right)], [left_nulls, right_nulls], chunk_size)


def matching_rows(table, condition):
    return [offset + chunk * table.target_chunk_size for chunk, offset in
            as_tuples(cso.table_scan_columns(table, ColumnComparison(0, condition, 1)))]


def test_int_float_rounds_the_integer_to_float():
    # 16777217 is not a float: it rounds to 16777216.0f, so the pair is equal in float (never compared in double)
    left = np.array([16777217, 16777216, 16777218, 16777219, -16777217], dtype=np.int32)
    right = np.array([16777216.0, 16777216.0, 16777216.0, 16777220.0, -16777216.0], dtype=np.float32)
    for encoding in ("Unencoded", "Dictionary"):
        table = pair_table(P.TYPE_INT32, left, P.TYPE_FLOAT32, right).encode(encoding)
        assert matching_rows(table, P.PRED_EQUALS) == [0, 1, 3, 4]
        assert matching_rows(table, P.PRED_GREATER_THAN) == [2]
        assert matching_rows(table, P.PRED_LESS_THAN) == []
    int64 = np.array([2 ** 24 + 1, 2 ** 40 + 1], dtype=np.int64)
    table = pair_table(P.TYPE_INT64, int64, P.TYPE_FLOAT32, np.array([2.0 ** 24, 2.0 ** 40], dtype=np.float32))
    assert matching_rows(table.encode("Dictionary"), P.PRED_EQUALS) == [0, 1]


def test_int64_double_rounds_the_integer_and_int32_double_is_exact():
    left = np.array([2 ** 53 + 1, 2 ** 53, 2 ** 53 + 2, -(2 ** 53) - 1], dtype=np.int64)
    right = np.array([2.0 ** 53, 2.0 ** 53, 2.0 ** 53, -(2.0 ** 53)], dtype=np.float64)
    table = pair_table(P.TYPE_INT64, left, P.TYPE_FLOAT64, right).encode("Unencoded")
    assert matching_rows(table, P.PRED_EQUALS) == [0, 1, 3]
    assert matching_rows(table, P.PRED_GREATER_THAN) == [2]
    # int32 x double: exact; int32 x int64: exact in int64
    ints = np.array([16777217, 2 ** 31 - 1, -(2 ** 31)], dtype=np.int32)
    table = pair_table(P.TYPE_INT32, ints, P.TYPE_FLOAT64, np.array([16777216.0, 2.0 ** 31 - 1, -(2.0 ** 31)]))
    assert matching_rows(table, P.PRED_EQUALS) == [1, 2]
    assert matching_rows(table, P.PRED_GREATER_THAN) == [0]
    table = pair_table(P.TYPE_INT32, ints, P.TYPE_INT64, np.array([16777216, 2 ** 31 - 1, -(2 ** 31) + 1]))
    assert matching_rows(table, P.PRED_EQUALS) == [1]
    assert matching_rows(table, P.PRED_LESS_THAN) == [2]


@pytest.mark.parametrize("left_type,right_type", [(P.TYPE_FLOAT32, P.TYPE_FLOAT32), (P.TYPE_FLOAT64, P.TYPE_FLOAT64),
                                                  (P.TYPE_FLOAT32, P.TYPE_FLOAT64)])
def test_ieee_special_values(left_type, right_type):
    nan, inf = float("nan"), float("inf")
    left = [nan, 1.0, nan, -0.0, 0.0, inf, -inf, inf, 2.0]
    right = [nan, nan, 1.0, 0.0, -0.0, inf, inf, 3.0, -inf]
    table = pair_table(left_type, left, right_type, right, chunk_size=4).encode("Unencoded")
    assert matching_rows(table, P.PRED_EQUALS) == [3, 4, 5]
    assert matching_rows(table, P.PRED_NOT_EQUALS) == [0, 1, 2, 6, 7, 8]  # NaN != everything
    assert matching_rows(table, P.PRED_LESS_THAN) == [6]
    assert matching_rows(table, P.PRED_LESS_THAN_EQUALS) == [3, 4, 5, 6]
    assert matching_rows(table, P.PRED_GREATER_THAN) == [7, 8]
    assert matching_rows(table, P.PRED_GREATER_THAN_EQUALS) == [3, 4, 5, 7, 8]


def test_nulls_on_either_side_never_match():
    left = np.array([1, 2, 3, 4, 5, 6], dtype=np.int32)
    right = np.array([1, 5, 3, 0, 5, 6], dtype=np.int64)
    left_nulls = np.array([0, 0, 1, 0, 0, 1], dtype=bool)
    right_nulls = np.array([0, 1, 0, 0, 1, 1], dtype=bool)
    for encoding in ("Unencoded", "Dictionary"):
        table = pair_table(P.TYPE_INT32, left, P.TYPE_INT64, right, left_nulls, right_nulls).encode(encoding)
        assert matching_rows(table, P.PRED_EQUALS) == [0]
        assert matching_rows(table, P.PRED_NOT_EQUALS) == [3]
        assert matching_rows(table, P.PRED_GREATER_THAN_EQUALS) == [0, 3]


# --- string dictionaries: the host translation ----------------------------------------------------------------------------
def random_strings(rng: random.Random, count: int) -> list[bytes]:
    alphabet = [b"a", b"b", b"\x00", b"\x7f", b"\x80", b"\xff", b"A"]
    values = {b""}
    while len(values) < count:
        values.add(b"".join(rng.choice(alphabet) for _ in range(rng.randint(0, 5))))
    return sorted(values)[:count] if count else []


def sign(x: int) -> int:
    return (x > 0) - (x < 0)


def cmp(a: bytes, b: bytes) -> int:
    return (a > b) - (a < b)


def check_translation(left: list[bytes], right: list[bytes]) -> None:
    words = capi.dictionary_translate(left, right)
    assert len(words) == len(right)
    for j, value in enumerate(right):
        position = bisect.bisect_left(left, value)
        found = position < len(left) and left[position] == value
        assert int(words[j]) == 2 * position + int(found), (value, position, found)
        for i, entry in enumerate(left):  # order and equality of the keys are those of the strings
            assert sign(cmp(entry, value)) == sign((2 * i + 1) - int(words[j]))


@pytest.mark.parametrize("seed", range(6))
def test_dictionary_translate_against_bisect(seed):
    rng = random.Random(seed)
    pool = random_strings(rng, 80)  # sorted: the empty string, proper prefixes, bytes >= 0x80 and embedded NUL
    left = sorted(rng.sample(pool, rng.randint(0, 60)))
    right = sorted(rng.sample(pool, rng.randint(0, 60)))
    check_translation(left, right)
    check_translation(right, left)
    check_translation(left, left)  # a column compared with itself: right_in_left[j] = 2j + 1
    assert list(capi.dictionary_translate(left, left)) == [2 * j + 1 for j in range(len(left))]


def test_dictionary_translate_small_dictionaries():
    check_translation([], [])
    check_translation([], [b"a"])
    assert list(capi.dictionary_translate([], [b"a", b"b"])) == [0, 0]
    assert list(capi.dictionary_translate([b"b"], [])) == []
    assert list(capi.dictionary_translate([b"b"], [b"a", b"b", b"c"])) == [0, 1, 2]
    assert list(capi.dictionary_translate([b""], [b""])) == [1]  # empty strings only: no characters at all
    assert list(capi.dictionary_translate([b"ab"], [b"a", b"ab\x00", b"\x80"])) == [0, 2, 2]


def test_binary_table_translation_equals_the_python_one(tmp_path):
    rng = random.Random(7)
    pool = [value for value in random_strings(rng, 60) if not value.endswith(b"\x00")]  # 'S' arrays drop trailing NULs
    rows = 50
    left = [rng.choice(pool) for _ in range(rows)]
    right = [rng.choice(pool[10:40]) for _ in range(rows)]
    table = Table.from_columns([ColumnDefinition("l", P.TYPE_STRING), ColumnDefinition("r", P.TYPE_STRING),
                                ColumnDefinition("k", P.TYPE_INT32)],
                               [np.array(left, dtype="S8"), np.array(right, dtype="S8"), np.arange(rows, dtype=np.int32)],
                               chunk_size=7).encode("Dictionary")
    path = os.path.join(tmp_path, "pairs.bin")
    write_binary_table(table, path)
    native = NativeBinaryTable(path)
    try:
        for a, b in [(0, 1), (1, 0), (0, 0)]:
            assert np.array_equal(native.column_translation(a, b), table.string_column_translation(a, b))
            assert len(native.column_translation(a, b)) == sum(len(chunk.segments[b].string_dictionary)
                                                               for chunk in table.chunks)
        with pytest.raises(capi.HyriseB200Error):
            native.column_translation(0, 2)
    finally:
        native.close()
