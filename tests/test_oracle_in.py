"""`<column> [NOT] IN (<literal>, ...)` without a GPU: the row-by-row restatement (in_scan_oracle.py) against the
reference's own expectations, the library's list normaliser against the restatement's std::equal_to for every column and
element type, and the string dictionary bitmaps against Python set membership."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import in_scan_oracle as ino
from conftest import GOLDEN
from helpers import tbl
from hyrise_b200 import capi
from hyrise_b200.device import InList, build_in_predicate, literal_type
from hyrise_b200.storage import ColumnDefinition, Table

P = capi
I32, I64, F32, F64 = np.int32, np.int64, np.float32, float
NUMERIC = [P.TYPE_INT32, P.TYPE_INT64, P.TYPE_FLOAT32, P.TYPE_FLOAT64]
NUMPY = {P.TYPE_INT32: np.int32, P.TYPE_INT64: np.int64, P.TYPE_FLOAT32: np.float32, P.TYPE_FLOAT64: np.float64}


def scalar(value, elements, negated):
    """`<literal> [NOT] IN (elements)` as a one-row column; None = the NULL literal. Returns 1, 0 or None (NULL),
    reading NULL off the restatement as "neither the row nor its negation is selected" for a non-degenerate list."""
    if value is None or isinstance(value, int):
        column_type, values, nulls = P.TYPE_INT32, np.array([0 if value is None else value], np.int32), [value is None]
    else:
        column_type, values, nulls = P.TYPE_STRING, [value.encode()], [False]
    got = bool(ino.selected(column_type, values, nulls, elements, negated)[0])
    flipped = bool(ino.selected(column_type, values, nulls, elements, not negated)[0])
    if not got and not flipped:
        return None
    return int(got)


# (left, list, expected IN, expected NOT IN): the literal-list cases of ExpressionEvaluatorToValuesTest.InListLiterals
# and NotInListLiterals (expression_evaluator_to_values_test.cpp:579-597, 752-770) whose elements are all literals.
LITERAL_CASES = [
    (None, [None], None, None),
    (None, [None, 3], None, None),
    (None, [], 0, 1),
    (None, [1, 2, 3, 4], None, None),
    (None, [None, 2, 3, 4], None, None),
    (5, [None, 5, None], 1, 0),
    (5, [], 0, 1),
    (5, [None, 6, None], None, None),
    (5, [1, 3], 0, 1),
    (5, [1.0, 3.0], 0, 1),
    (5, ["Hello", 1.0, "You", 3.0], 0, 1),
    ("You", ["Hello", 1.0, "You", 3.0], 1, 0),
    (5, [1.0, 5.0], 1, 0),
]
# Cases with computed elements (add_) are evaluated expressions, not literal lists a TableScan receives.
COMPUTED_CASES = ["in_(5, list_(null_(), add_(2, 3), null_()))", "in_(5, list_(1.0, add_(1.0, 3.0)))",
                  "in_(5, list_(1.0, add_(2.0, 3.0)))", "not_in_(5, list_(null_(), add_(2, 3), null_()))",
                  "not_in_(5, list_(1.0, add_(1.0, 3.0)))", "not_in_(5, list_(1.0, add_(2.0, 3.0)))",
                  "in_(sub_(mul_(a, 2), 2), list_(b, 6, null_(), 0))",
                  "not_in_(sub_(mul_(a, 2), 2), list_(b, 6, null_(), 0))"]


@pytest.mark.parametrize("left,elements,expected_in,expected_not_in", LITERAL_CASES)
def test_reference_literal_lists(left, elements, expected_in, expected_not_in):
    assert scalar(left, elements, False) == expected_in
    assert scalar(left, elements, True) == expected_not_in


@pytest.mark.parametrize("case", COMPUTED_CASES)
def test_reference_computed_elements(case):
    pytest.skip(f"{case}: an element is an expression or a column, not a literal; such lists stay on the CPU")


@pytest.mark.parametrize("chunk_size", [2, 5])
def test_reference_series(chunk_size):
    # InListSeries / NotInListSeries on table_a (input_a.tbl), column a = 1, 2, 3, 4
    table = tbl("expression_evaluator_input_a.tbl", chunk_size)
    column = table.column_id_by_name("a")
    cases = [([1.0, 3.0], [0, 2], [1, 3]),
             ([None, 1.0, 3.0], [0, 2], [])]  # NULL rows 1 and 3 of IN / NOT IN are not selected
    for elements, in_rows, not_in_rows in cases:
        for condition, rows in ((P.PRED_IN, in_rows), (P.PRED_NOT_IN, not_in_rows)):
            result = ino.table_scan_in(table, InList(column, condition, elements))
            flat = [int(r["chunk_id"]) * chunk_size + int(r["chunk_offset"]) for r in result.row_ids]
            assert flat == rows, (elements, condition)


def test_string_column_rules():
    values = [b"a", b"b", b"", b"ab"]
    nulls = [False, False, False, True]
    # NULL elements are dropped on a string column: `s NOT IN ('a', NULL)` is `s NOT IN ('a')`
    assert ino.selected(P.TYPE_STRING, values, nulls, ["a", None], True).tolist() == [False, True, True, False]
    assert ino.selected(P.TYPE_STRING, values, nulls, ["a", None], False).tolist() == [True, False, False, False]
    # no string element: IN selects nothing, NOT IN every row, the NULL row included
    assert ino.selected(P.TYPE_STRING, values, nulls, [1, None, 2.5], False).tolist() == [False] * 4
    assert ino.selected(P.TYPE_STRING, values, nulls, [1, None, 2.5], True).tolist() == [True] * 4
    assert ino.null_row_selected(P.TYPE_STRING, [], True) and not ino.null_row_selected(P.TYPE_STRING, ["a"], True)
    # numeric column: string elements are dropped, NULL elements stay
    ints = np.array([1, 2, 3], np.int32)
    assert ino.selected(P.TYPE_INT32, ints, [False] * 3, ["x", 2], True).tolist() == [True, False, True]
    assert ino.selected(P.TYPE_INT32, ints, [False] * 3, [None, 2], True).tolist() == [False] * 3
    assert ino.selected(P.TYPE_INT32, ints, [False] * 3, ["x"], True).tolist() == [True] * 3


def test_rule_four_examples():
    floats = np.array([0.05, 0.0], np.float32)
    assert ino.selected(P.TYPE_FLOAT32, floats, [False, False], [0.05], False).tolist() == [False, False]
    assert capi.in_list_normalize(P.TYPE_FLOAT32, [literal_type(0.05)]) == []
    big = np.array([2**53, 2**53 + 1, 2**53 + 2, 2**53 - 1], np.int64)
    assert ino.selected(P.TYPE_INT64, big, [False] * 4, [9007199254740992.0], False).tolist() == [True, True, False, False]
    assert capi.in_list_normalize(P.TYPE_INT64, [literal_type(9007199254740992.0)]) == [(2**53, 2**53 + 1)]
    ints = np.array([16777216, 16777217, 16777218, 16777215], np.int32)
    assert ino.selected(P.TYPE_INT32, ints, [False] * 4, [np.float32(16777216.0)], False).tolist() == \
        [True, True, False, False]
    assert capi.in_list_normalize(P.TYPE_INT32, [literal_type(np.float32(16777216.0))]) == [(16777216, 16777217)]


# ---------------------------------------------------------------------------------------------------------------------
# hyb_in_list_normalize against the restatement's std::equal_to
# ---------------------------------------------------------------------------------------------------------------------
EDGE_ELEMENTS = [
    I32(0), I32(1), I32(-1), I32(-2**31), I32(2**31 - 1), I32(2**24 - 1), I32(2**24), I32(2**24 + 1), I32(7),
    I64(-2**63), I64(2**63 - 1), I64(2**53 - 1), I64(2**53), I64(2**53 + 1), I64(2**31), I64(-2**31 - 1), I64(2**24 + 1),
    F32(0.0), F32(-0.0), F32(np.nan), F32(np.inf), F32(-np.inf), F32(1e-45), F32(-1e-45), F32(3.4028235e38),
    F32(-3.4028235e38), F32(16777216.0), F32(0.05), F32(2.5), F32(9.223372e18), F32(-2147483648.0), F32(2147483648.0),
    F64(0.0), F64(-0.0), F64(math.nan), F64(math.inf), F64(-math.inf), F64(5e-324), F64(0.05), F64(2.5),
    F64(2**53), F64(2**53 + 2), F64(2**63), F64(-2**63), F64(2**31 - 1), F64(2**31), F64(-2**31), F64(16777217.0),
    F64(float(np.float32(3.4028235e38))), F64(1e300), F64(float(np.float32(0.05))), F64(1.5e-45),
]


def neighbours(column_type, value):
    if column_type in (P.TYPE_INT32, P.TYPE_INT64):
        info = np.iinfo(NUMPY[column_type])
        return [v for v in (value - 1, value, value + 1) if info.min <= v <= info.max]
    dtype = NUMPY[column_type]
    value = dtype(value)
    with np.errstate(over="ignore"):
        return [np.nextafter(value, dtype(-np.inf)), value, np.nextafter(value, dtype(np.inf))]


def probes(column_type, elements, intervals, rng):
    values = []
    for lo, hi in intervals:
        values += neighbours(column_type, lo) + neighbours(column_type, hi)
    for element in elements:
        data_type, value = literal_type(element)
        if data_type is None or (isinstance(value, float) and not math.isfinite(value)):
            continue
        if column_type in (P.TYPE_INT32, P.TYPE_INT64):
            info = np.iinfo(NUMPY[column_type])
            center = int(min(max(value, info.min), info.max))
            values += neighbours(column_type, center)
            values += [int(min(max(center + int(d), info.min), info.max)) for d in rng.integers(-3, 4, 6)]
        else:
            with np.errstate(over="ignore"):
                values += neighbours(column_type, NUMPY[column_type](value))
    if column_type in (P.TYPE_INT32, P.TYPE_INT64):
        info = np.iinfo(NUMPY[column_type])
        values += [info.min, info.max, 0, 1, -1] + [int(v) for v in rng.integers(info.min, info.max, 40, dtype=np.int64)]
    else:
        values += [0.0, -0.0, np.nan, np.inf, -np.inf, np.finfo(NUMPY[column_type]).max]
        values += list(rng.standard_normal(20) * 10.0 ** rng.integers(-40, 38, 20))
    with np.errstate(over="ignore"):
        return np.array(values, dtype=NUMPY[column_type])


def members(intervals, values):
    out = np.zeros(len(values), dtype=bool)
    for lo, hi in intervals:
        out |= (values >= lo) & (values <= hi)
    return out


def check_normal_form(column_type, intervals):
    integral = column_type in (P.TYPE_INT32, P.TYPE_INT64)
    for (lo, hi) in intervals:
        assert lo <= hi
        if lo == 0:
            assert math.copysign(1.0, lo) > 0, "zero is stored as +0.0"
    for (_, hi), (lo, _) in zip(intervals, intervals[1:]):
        if integral:
            assert lo > hi + 1, "touching intervals are merged"
        else:
            assert lo > np.nextafter(NUMPY[column_type](hi), NUMPY[column_type](np.inf)), "touching intervals are merged"


@pytest.mark.parametrize("column_type", NUMERIC)
def test_normalize_each_element_against_equal_to(column_type):
    rng = np.random.default_rng(column_type)
    for element in EDGE_ELEMENTS:
        intervals = capi.in_list_normalize(column_type, [literal_type(element)])
        check_normal_form(column_type, intervals)
        values = probes(column_type, [element], intervals, rng)
        expected = ino.selected(column_type, values, np.zeros(len(values), bool), [element], False)
        assert np.array_equal(members(intervals, values), expected), (column_type, element, intervals)


@pytest.mark.parametrize("column_type", NUMERIC)
def test_normalize_lists_against_equal_to(column_type):
    rng = np.random.default_rng(100 + column_type)
    for trial in range(30):
        count = int(rng.integers(1, 12))
        picks = [EDGE_ELEMENTS[int(i)] for i in rng.integers(0, len(EDGE_ELEMENTS), count)]
        picks += picks[: int(rng.integers(0, 3))]  # duplicates
        rng.shuffle(picks)
        intervals = capi.in_list_normalize(column_type, [literal_type(e) for e in picks])
        check_normal_form(column_type, intervals)
        values = probes(column_type, picks, intervals, rng)
        for negated in (False, True):
            expected = ino.selected(column_type, values, np.zeros(len(values), bool), picks, negated)
            got = members(intervals, values)
            if negated:  # NOT IN without NULL element: not a member (NaN rows included)
                got = ~got
            assert np.array_equal(got, expected), (column_type, picks, intervals)


def test_normalize_merges_and_rejects():
    assert capi.in_list_normalize(P.TYPE_INT32, [(P.TYPE_INT32, 3), (P.TYPE_INT32, 1), (P.TYPE_INT32, 2),
                                                 (P.TYPE_INT32, 2), (P.TYPE_INT32, 7)]) == [(1, 3), (7, 7)]
    assert capi.in_list_normalize(P.TYPE_FLOAT64, [(P.TYPE_FLOAT64, -0.0), (P.TYPE_FLOAT64, 0.0)]) == [(0.0, 0.0)]
    assert capi.in_list_normalize(P.TYPE_FLOAT64, [(P.TYPE_FLOAT64, math.nan)]) == []
    assert capi.in_list_normalize(P.TYPE_INT32, [(P.TYPE_INT64, 2**40)]) == []
    assert capi.in_list_normalize(P.TYPE_INT32, [(P.TYPE_FLOAT64, 2.5)]) == []
    lib = capi.load_library()
    count = C.c_uint32(4)
    literal = capi.literal_array([(P.TYPE_INT32, 1)])
    assert lib.hyb_in_list_normalize(P.TYPE_STRING, literal, 1, None, C.byref(count)) == P.HYB_ERR_INVALID
    bad = capi.literal_array([(P.TYPE_STRING, 0)])
    bad[0].data_type = P.TYPE_STRING
    assert lib.hyb_in_list_normalize(P.TYPE_INT32, bad, 1, None, C.byref(count)) == P.HYB_ERR_INVALID
    two = capi.literal_array([(P.TYPE_INT32, 1), (P.TYPE_INT32, 5)])
    bounds = (capi.Value * 2)()
    count = C.c_uint32(1)  # room for one interval, two are needed
    assert lib.hyb_in_list_normalize(P.TYPE_INT32, two, 2, bounds, C.byref(count)) == P.HYB_ERR_INVALID


# ---------------------------------------------------------------------------------------------------------------------
# String dictionary bitmaps against Python set membership
# ---------------------------------------------------------------------------------------------------------------------
def expected_words(entries, elements, condition):
    bits = [(bytes(entry) in set(elements)) != (condition == P.PRED_NOT_IN) for entry in entries]
    words = np.zeros((len(entries) + 31) // 32, dtype=np.uint32)
    for index, bit in enumerate(bits):
        if bit:
            words[index >> 5] |= np.uint32(1 << (index & 31))
    return words


def random_dictionary(rng, count):
    alphabet = [b"a", b"b", b"\x80", b"\xff", b"\x00x", b"ab"]
    entries = {b""}
    while len(entries) < count:
        entries.add(b"".join(alphabet[int(i)] for i in rng.integers(0, len(alphabet), int(rng.integers(0, 5)))))
    return sorted(entries)


@pytest.mark.parametrize("condition", [P.PRED_IN, P.PRED_NOT_IN])
def test_dictionary_matches(condition):
    rng = np.random.default_rng(7 + condition)
    for trial in range(40):
        entries = random_dictionary(rng, int(rng.integers(1, 90)))
        elements = [entries[int(i)] for i in rng.integers(0, len(entries), int(rng.integers(1, 6)))]
        elements += [b"absent", entries[-1] + b"z", entries[-1][:-1]]  # absent, a proper extension, a proper prefix
        rng.shuffle(elements)
        got = capi.in_dictionary_matches(condition, elements, entries)
        assert np.array_equal(got, expected_words(entries, elements, condition)), (entries, elements)
    # a dictionary holding only the empty string, and a list holding only the empty string: NULL characters
    assert capi.in_dictionary_matches(condition, [b""], [b""]).tolist() == ([1] if condition == P.PRED_IN else [0])
    assert capi.in_dictionary_matches(condition, [b"a"], [b""]).tolist() == ([0] if condition == P.PRED_IN else [1])
    assert capi.in_dictionary_matches(condition, [b""], []).tolist() == []


def test_dictionary_matches_rejects_other_conditions():
    lib = capi.load_library()
    offsets = np.zeros(2, dtype=np.uint64)
    words = np.zeros(1, dtype=np.uint32)
    for condition in (P.PRED_EQUALS, P.PRED_LIKE):
        assert lib.hyb_in_dictionary_matches(condition, None, offsets.ctypes.data_as(C.POINTER(C.c_uint64)), 1, None,
                                             offsets.ctypes.data_as(C.POINTER(C.c_uint64)), 1,
                                             words.ctypes.data_as(C.POINTER(C.c_uint32)), None) == P.HYB_ERR_INVALID


def test_table_bitmaps_and_predicate_struct():
    rng = np.random.default_rng(3)
    strings = np.array(random_dictionary(rng, 60)[1:], dtype="S")
    values = strings[rng.integers(0, len(strings), 600)]
    nulls = rng.random(600) < 0.1
    nulls[100:150] = True  # chunk 2 (chunk size 50) has no dictionary entry
    table = Table.from_columns([ColumnDefinition("s", P.TYPE_STRING, True), ColumnDefinition("i", P.TYPE_INT32)],
                               [values, np.arange(600, dtype=np.int32)], [nulls, None], chunk_size=50)
    table.encode("Dictionary")
    elements = [bytes(strings[0]), "ab", None, 5, bytes(strings[3])]
    for condition in (P.PRED_IN, P.PRED_NOT_IN):
        string_elements = [bytes(strings[0]), b"ab", bytes(strings[3])]
        words = table.string_in_bitmaps(0, condition, string_elements)
        expected = np.concatenate([expected_words([bytes(e) for e in chunk.segments[0].string_dictionary],
                                                  string_elements, condition) for chunk in table.chunks])
        assert np.array_equal(words, expected)
        struct, keepalive = build_in_predicate(table, InList(0, condition, elements))
        assert struct.dictionary_matches == keepalive.ctypes.data and np.array_equal(keepalive[: len(words)], words)
        # no string element: no bitmaps
        struct, _ = build_in_predicate(table, InList(0, condition, [1, None]))
        assert not struct.dictionary_matches
        # a numeric column takes its numeric elements and the NULL flag; strings are dropped
        struct, _ = build_in_predicate(table, InList(1, condition, elements))
        assert struct.element_count == 1 and struct.has_null_element == 1 and not struct.dictionary_matches
        assert struct.elements[0].data_type == P.TYPE_INT32 and struct.elements[0].value.i32 == 5


def test_literal_types():
    assert literal_type(5) == (P.TYPE_INT32, 5)
    assert literal_type(2**31) == (P.TYPE_INT64, 2**31)
    assert literal_type(-2**31) == (P.TYPE_INT32, -2**31)
    assert literal_type(2.5) == (P.TYPE_FLOAT64, 2.5)
    assert literal_type(np.float32(2.5)) == (P.TYPE_FLOAT32, 2.5)
    assert literal_type(np.int64(5)) == (P.TYPE_INT64, 5)
    assert literal_type("x") == (P.TYPE_STRING, b"x") and literal_type(b"\xff") == (P.TYPE_STRING, b"\xff")
    assert literal_type(None) == (None, None)
    with pytest.raises(OverflowError):
        literal_type(2**63)
    with pytest.raises(TypeError):
        literal_type(True)


def test_binary_table_in_bitmaps(tmp_path):
    from hyrise_b200.binary_table import NativeBinaryTable, write_binary_table

    checked = 0
    for name in ("StringSegment/Dictionary.bin", "FixedStringDictionaryMultipleChunks.bin",
                 "FixedStringDictionaryNullValue.bin", "AllTypesMixColumn/Dictionary.bin"):
        native = NativeBinaryTable(os.path.join(GOLDEN, "bin", name))
        try:
            for column, definition in enumerate(native.table.column_definitions):
                if definition.data_type != P.TYPE_STRING:
                    if checked == 0:
                        with pytest.raises(capi.HyriseB200Error):
                            native.in_bitmaps(column, P.PRED_IN, [b"a"])
                    continue
                for elements in ([b"a"], [b"This", b"test", b"zzz"], [b""], [b"is", b"is"]):
                    for condition in (P.PRED_IN, P.PRED_NOT_IN):
                        expected = np.concatenate(
                            [expected_words([bytes(e) for e in chunk.segments[column].string_dictionary], elements,
                                            condition) for chunk in native.table.chunks] + [np.zeros(0, np.uint32)])
                        assert np.array_equal(native.in_bitmaps(column, condition, elements), expected), (name, elements)
                        checked += 1
        finally:
            native.close()
    assert checked > 0
    # a chunk whose dictionary holds only "" has no characters in the parsed file
    values = np.array([b"", b"", b"a_b", b"", b"xyz", b""], dtype="S")
    table = Table.from_columns([ColumnDefinition("s", P.TYPE_STRING)], [values], chunk_size=2).encode("Dictionary")
    path = str(tmp_path / "empty_strings.bin")
    write_binary_table(table, path)
    native = NativeBinaryTable(path)
    try:
        for elements in ([b""], [b"xyz", b"q"]):
            for condition in (P.PRED_IN, P.PRED_NOT_IN):
                expected = np.concatenate([expected_words([bytes(e) for e in chunk.segments[0].string_dictionary],
                                                          elements, condition) for chunk in native.table.chunks])
                assert np.array_equal(native.in_bitmaps(0, condition, elements), expected)
    finally:
        native.close()
