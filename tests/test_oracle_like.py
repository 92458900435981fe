"""LIKE without a GPU: the oracle against the reference's own expectations, and the library's dictionary matcher
(hyb_like_dictionary_matches, hyb_binary_table_like_bitmaps) against the oracle, bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest

import like_oracle as lo
from conftest import GOLDEN
from helpers import row_ids_equal, tbl
from hyrise_b200 import capi
from hyrise_b200.device import Predicate, build_scan_predicate
from hyrise_b200.storage import ColumnDefinition, Table

P = capi
LIKES = list(capi.LIKE_CONDITIONS)
ANY, ONE = lo.ANY, lo.SINGLE


# --- like_matcher_test.cpp --------------------------------------------------------------------------------------------
def test_pattern_to_tokens():
    # PatternToTokens (like_matcher_test.cpp:20-36)
    assert lo.tokens(b"") == []
    assert lo.tokens(b"%abc%_def__Hello%") == [ANY, b"abc", ANY, ONE, b"def", ONE, ONE, b"Hello", ANY]


# (value, pattern, Like, NotLike, LikeInsensitive, NotLikeInsensitive), like_matcher_test.cpp:38-116. The Like / NotLike
# rows use the value as written there; the insensitive tests (:78-116) write `heLlo` for `Hello`.
MATCHER_CASES = [
    (b"Hello", b"Hello", True), (b"Hello", b"Hello%", True), (b"Hello", b"%Hello%", True), (b"Hello", b"%H%%", True),
    (b"Hello", b"H%ello%", True), (b"Hello", b"%H%ello%", True), (b"Hello", b"H%el%l%o%", True),
    (b"Hello", b"%H%el%l%o%", True), (b"Hello World", b"%_%", True), (b"Hello World", b"%_World", True),
    (b"Hello World!! (Nice day)", b"H%(%day)", True), (b"Smiley: ^-^", b"%^_^%", True),
    (b"Questionmark: ?", b"%_?%", True),
    (b"hello", b"Hello", False), (b"Hello", b"Hello_", False), (b"Hello", b"He_o", False),
]


@pytest.mark.parametrize("value,pattern,expected", MATCHER_CASES)
def test_like_matcher_expectations(value, pattern, expected):
    assert lo.match(value, pattern, P.PRED_LIKE) == expected                   # :38-56
    assert lo.match(value, pattern, P.PRED_NOT_LIKE) == (not expected)         # :58-76
    insensitive_value = value.replace(b"Hello", b"heLlo") if value.startswith(b"Hello") else value
    insensitive_expected = True if value == b"hello" else expected             # :93 `hello` ILIKE `Hello`
    assert lo.match(insensitive_value, pattern, P.PRED_LIKE_INSENSITIVE) == insensitive_expected          # :78-96
    assert lo.match(insensitive_value, pattern, P.PRED_NOT_LIKE_INSENSITIVE) == (not insensitive_expected)  # :98-116
    for condition, (v, want) in zip(LIKES, [(value, expected), (value, not expected), (insensitive_value, insensitive_expected),
                                            (insensitive_value, not insensitive_expected)]):
        assert bool(capi.like_dictionary_matches(pattern, condition, [v])[0] & 1) == want, (v, pattern, condition)


def test_special_form_choice():
    # pattern_string_to_pattern_variant (like_matcher.cpp:125-182): the first three shapes, then the alternating check
    assert lo.form(b"abc%") == ("starts_with", b"abc")
    assert lo.form(b"%abc") == ("ends_with", b"abc")
    assert lo.form(b"%abc%") == ("contains", b"abc")
    assert lo.form(b"%a%b%c%") == ("multiple_contains", [b"a", b"b", b"c"])
    assert lo.form(b"%a%b") == ("multiple_contains", [b"a", b"b"])   # need not end with %
    assert lo.form(b"%") == ("multiple_contains", [])
    assert lo.form(b"") == ("multiple_contains", [])
    for pattern in (b"abc", b"a%b", b"%%", b"abc%%", b"%a_b%", b"_", b"a%b%"):
        assert lo.form(pattern)[0] == "regex", pattern


def test_newlines_differ_between_forms():
    # the regex `.` does not match '\n' / '\r'; the special forms compare bytes
    for terminator in (b"\n", b"\r"):
        value = b"a" + terminator + b"b"
        assert not lo.match(value, b"a%b", P.PRED_LIKE)
        assert lo.match(value, b"%a%b%", P.PRED_LIKE)
        assert lo.match(value, b"a%", P.PRED_LIKE)
        assert not lo.match(value, b"a_b", P.PRED_LIKE)
        words = capi.like_dictionary_matches(b"a%b", P.PRED_LIKE, [value, b"axb"])
        assert words[0] == 0b10
        assert capi.like_dictionary_matches(b"%a%b%", P.PRED_LIKE, [value, b"axb"])[0] == 0b11
        assert capi.like_dictionary_matches(b"a%b", P.PRED_NOT_LIKE, [value, b"axb"])[0] == 0b01


def test_insensitive_lowers_ascii_only():
    assert lo.match(b"\xc4BC", b"\xc4bc", P.PRED_LIKE_INSENSITIVE)
    assert not lo.match(b"\xe4bc", b"\xc4bc", P.PRED_LIKE_INSENSITIVE)  # bytes >= 0x80 stay as they are
    assert capi.like_dictionary_matches(b"\xc4bc", P.PRED_LIKE_INSENSITIVE, [b"\xc4BC", b"\xe4bc"])[0] == 0b01


def test_dictionary_of_empty_strings_without_characters():
    # a dictionary that holds only "" has no characters: the C path gets chars == NULL and must accept it
    assert capi.like_dictionary_matches(b"%", P.PRED_LIKE, [b""])[0] == 1
    assert capi.like_dictionary_matches(b"_%", P.PRED_LIKE, [b""])[0] == 0
    assert capi.like_dictionary_matches(b"", P.PRED_NOT_LIKE, [b""])[0] == 0
    offsets = np.zeros(2, dtype=np.uint64)
    offsets[1] = 1  # one character claimed but none given: still an error
    words = np.zeros(1, dtype=np.uint32)
    lib = capi.load_library()
    assert lib.hyb_like_dictionary_matches(b"%", 1, P.PRED_LIKE, None, offsets.ctypes.data_as(C.POINTER(C.c_uint64)), 1,
                                           words.ctypes.data_as(C.POINTER(C.c_uint32)), None) == capi.HYB_ERR_INVALID


# Bracket expressions. sql_like_to_regex (like_matcher.cpp:32-55) escapes neither `[` nor `]`, so in a pattern of the
# regex form they open an ECMAScript character class; like_oracle.py does not restate those. These expectations follow
# ECMAScript by hand: [bc] is one of b / c; `^` is escaped like every other character of the table, so [^a] is the class
# of `^` and `a`, not a negation; a `.` inside a class is escaped to a literal `\.`, and `%` / `_` inside a class become
# the characters `.`, `*` / `.`. In the special forms (abc%, %abc,
# %abc%, %a%b%) brackets are plain characters.
BRACKET_CASES = [
    (b"a[bc]_", [(b"abx", True), (b"acx", True), (b"adx", False), (b"ab", False), (b"ab\n", False)]),
    (b"[^a]_%", [(b"ab", True), (b"^bc", True), (b"bc", False), (b"a", False), (b"ab\n", False)]),
    (b"%[.]_", [(b"x.y", True), (b"x.", False), (b"xyz", False)]),
    (b"x[%]y", [(b"x.y", True), (b"x*y", True), (b"x%y", False), (b"xzy", False)]),
    (b"x[_]y", [(b"x.y", True), (b"x_y", False)]),
    (b"[a-c]_", [(b"bz", True), (b"dz", False), (b"-z", False)]),
    (b"[a-c]%", [(b"[a-c]x", True), (b"bx", False)]),   # starts-with: the brackets are literal
    (b"%[x]%", [(b"a[x]b", True), (b"axb", False)]),    # contains
]


@pytest.mark.parametrize("pattern,cases", BRACKET_CASES, ids=[case[0].decode() for case in BRACKET_CASES])
def test_library_bracket_expressions(pattern, cases):
    values = [value for value, _ in cases]
    words = capi.like_dictionary_matches(pattern, P.PRED_LIKE, values)
    got = [bool(words[i >> 5] >> (i & 31) & 1) for i in range(len(values))]
    assert got == [want for _, want in cases]
    try:
        kind = lo.form(pattern)[0]
    except NotImplementedError:  # regex form with a bracket expression: not restated by the oracle
        kind = "regex"
    if kind != "regex":
        assert [lo.match(value, pattern, P.PRED_LIKE) for value in values] == got
    inverted = capi.like_dictionary_matches(pattern, P.PRED_NOT_LIKE, values)
    assert [bool(inverted[i >> 5] >> (i & 31) & 1) for i in range(len(values))] == [not want for _, want in cases]


def test_library_rejects_bad_input():
    with pytest.raises(capi.HyriseB200Error) as error:
        capi.like_dictionary_matches(b"a%", P.PRED_EQUALS, [b"a"])
    assert error.value.status == capi.HYB_ERR_INVALID
    with pytest.raises(capi.HyriseB200Error) as error:  # std::regex rejects the unbalanced bracket, as in the reference
        capi.like_dictionary_matches(b"a[_", P.PRED_LIKE, [b"a"])
    assert error.value.status == capi.HYB_ERR_INVALID
    assert len(capi.like_dictionary_matches(b"%", P.PRED_LIKE, [])) == 0


# --- table_scan_string_test.cpp ---------------------------------------------------------------------------------------
# (test, input, column, condition, pattern, expected .tbl or None for an empty result)
SCAN_CASES = [
    ("ScanLikeEmptyString", "int_string_like.tbl", P.PRED_LIKE, b"%", "int_string_like_without_null.tbl"),
    ("ScanLikeUnderscoreWildcard", "int_string_like.tbl", P.PRED_LIKE, b"%D%_m_f%", "int_string_like_starting.tbl"),
    ("ScanLike_Starting", "int_string_like.tbl", P.PRED_LIKE, b"Dampf%", "int_string_like_starting.tbl"),
    ("ScanLikeEnding", "int_string_like.tbl", P.PRED_LIKE, b"%gesellschaft", "int_string_like_ending.tbl"),
    ("ScanLikeOnSpecialChars/1", "int_string_like_special_chars.tbl", P.PRED_LIKE, b"%2^2%",
     "int_string_like_special_chars_1.tbl"),
    ("ScanLikeOnSpecialChars/2", "int_string_like_special_chars.tbl", P.PRED_LIKE, b"%$%$%",
     "int_string_like_special_chars_1.tbl"),
    ("ScanLikeOnSpecialChars/3", "int_string_like_special_chars.tbl", P.PRED_LIKE, b"%(%)%",
     "int_string_like_special_chars_2.tbl"),
    ("ScanLikeOnSpecialChars/4", "int_string_like_special_chars.tbl", P.PRED_LIKE, b"%la\\.^$+?)({}.*__bl%",
     "int_string_like_special_chars_3.tbl"),
    ("ScanLikeContainingWildcard", "int_string_like.tbl", P.PRED_LIKE, b"Schiff%schaft",
     "int_string_like_containing_wildcard.tbl"),
    ("ScanLikeContaining", "int_string_like.tbl", P.PRED_LIKE, b"%schifffahrtsgesellschaft%",
     "int_string_like_containing.tbl"),
    ("ScanLikeNotFound", "int_string_like.tbl", P.PRED_LIKE, b"%not_there%", None),
    ("ScanNotLikeEmptyString", "int_string_like.tbl", P.PRED_NOT_LIKE, b"%", None),
    ("ScanNotLikeAllRows", "int_string_like.tbl", P.PRED_NOT_LIKE, b"%foo%", "int_string_like_without_null.tbl"),
    ("ScanNotLikeUnderscoreWildcard", "int_string_like.tbl", P.PRED_NOT_LIKE, b"D_m_f%",
     "int_string_like_not_starting.tbl"),
]


def expected_rows(name):
    if name is None:
        return []
    table = tbl(name)
    ints, _ = table.column_values(0)
    strings, _ = table.column_values(1)
    return sorted(zip(ints.tolist(), [bytes(s) for s in strings]))


def result_rows(table, pos_list):
    out = []
    for row in pos_list.row_ids:
        segments = table.chunks[int(row["chunk_id"])].segments
        offset = int(row["chunk_offset"])
        out.append((int(segments[0].decode()[offset]), bytes(segments[1].decode()[offset])))
    return sorted(out)


@pytest.mark.parametrize("case", SCAN_CASES, ids=[case[0] for case in SCAN_CASES])
@pytest.mark.parametrize("chunk_size", [2, 5])
def test_oracle_reproduces_table_scan_string_test(case, chunk_size):
    _, source, condition, pattern, expected = case
    table = tbl(source, chunk_size).encode("Dictionary")
    result = lo.table_scan(table, 1, pattern, condition)
    assert result_rows(table, result) == expected_rows(expected)
    # ...OnReferencedDictSegment: the same LIKE on the output of `a > 0`
    first = lo.HostPosList(*_all_rows_with_positive_a(table))
    filtered = lo.table_scan(table, 1, pattern, condition, first)
    assert row_ids_equal(filtered.row_ids, result.row_ids)


def _all_rows_with_positive_a(table):
    rows, offsets = [], [0]
    for chunk_id, chunk in enumerate(table.chunks):
        values = chunk.segments[0].decode()
        rows.extend((chunk_id, offset) for offset in range(chunk.size) if values[offset] > 0)
        offsets.append(len(rows))
    from hyrise_b200.device import ROW_ID_DTYPE
    return np.array(rows, dtype=ROW_ID_DTYPE).reshape(-1), np.array(offsets, dtype=np.uint64)


def test_like_on_non_string_column_is_invalid():
    # ScanLikeNonStringColumn (table_scan_string_test.cpp:92-95): a hard error, not a CPU fallback
    table = tbl("int_float.tbl", 2).encode("Dictionary")
    with pytest.raises(capi.HyriseB200Error) as error:
        build_scan_predicate(table, Predicate(0, P.PRED_LIKE, b"%test"))
    assert error.value.status == capi.HYB_ERR_INVALID and not isinstance(error.value, capi.UnsupportedOnDevice)


# --- library matcher against the oracle -------------------------------------------------------------------------------
ALPHABET = [b"a", b"b", b"A", b"B", b"%", b"_", b".", b"^", b"$", b"+", b"?", b"(", b")", b"{", b"}", b"|", b"*", b"\\",
            b"\n", b"\r", b" ", b"\xc4", b"\xe4", b"\xff"]


def random_strings(rng, count, max_length=8):
    out = {b""}
    while len(out) < count:
        length = int(rng.integers(0, max_length + 1))
        out.add(b"".join(ALPHABET[i] for i in rng.integers(0, len(ALPHABET), length)))
    return sorted(out)


def random_patterns(rng, count):
    """Every special form and regex forms, with literals drawn from the same alphabet (wildcards excluded)."""
    literals = [a for a in ALPHABET if a not in (b"%", b"_")]

    def literal():
        return b"".join(literals[i] for i in rng.integers(0, len(literals), int(rng.integers(1, 3))))

    patterns = [b"", b"%", b"%%", b"_", b"__", b"%_%", b"a%b", b"%a%b", b"A%", b"%a", b"%\n%", b"_%_"]
    for _ in range(count):
        shape = int(rng.integers(0, 6))
        if shape == 0:
            patterns.append(literal() + b"%")
        elif shape == 1:
            patterns.append(b"%" + literal())
        elif shape == 2:
            patterns.append(b"%" + literal() + b"%")
        elif shape == 3:
            patterns.append(b"%" + b"%".join(literal() for _ in range(int(rng.integers(2, 4)))) + b"%")
        else:  # regex form: wildcards mixed into literals
            parts = [literal() if rng.random() < 0.5 else [b"%", b"_"][int(rng.integers(0, 2))]
                     for _ in range(int(rng.integers(1, 6)))]
            patterns.append(b"".join(parts))
    return patterns


def fixture_strings():
    out = set()
    for name in ("int_string_like.tbl", "int_string_like_special_chars.tbl", "int_string_like_containing2.tbl"):
        strings, nulls = tbl(name).column_values(1)
        out.update(bytes(s) for s, n in zip(strings, nulls) if not n)
    return sorted(out)


@pytest.mark.parametrize("condition", LIKES)
def test_library_matches_oracle_on_fixture_strings(condition):
    entries = fixture_strings()
    patterns = [case[3] for case in SCAN_CASES] + [b"%SCHIFF%", b"d%", b"%_?%", b"Dampf%kapit_n%", b"%\xc3\xa4n"]
    for pattern in patterns:
        expected = lo.dictionary_matches(entries, pattern, condition)
        assert np.array_equal(capi.like_dictionary_matches(pattern, condition, entries), expected), pattern


@pytest.mark.parametrize("condition", LIKES)
def test_library_matches_oracle_on_random_strings(condition):
    rng = np.random.default_rng(2024 + condition)
    entries = random_strings(rng, 700)
    for pattern in random_patterns(rng, 150):
        expected = lo.dictionary_matches(entries, pattern, condition)
        got = capi.like_dictionary_matches(pattern, condition, entries)
        assert np.array_equal(got, expected), (pattern, condition)


def test_table_bitmaps_layout():
    # storage.Table.string_like_bitmaps: ceil(dictionary size / 32) words per chunk, chunk order, empty dictionaries
    rng = np.random.default_rng(3)
    strings = np.array(random_strings(rng, 300), dtype="S")
    values = strings[rng.integers(0, len(strings), 1000)]
    nulls = rng.random(1000) < 0.1
    nulls[200:260] = True  # chunk 4 (chunk size 50) has no dictionary entry
    table = Table.from_columns([ColumnDefinition("s", capi.TYPE_STRING, True)], [values], [nulls], chunk_size=50)
    table.encode("Dictionary")
    assert table.chunks[4].segments[0].dictionary_size == 0
    predicate = Predicate(0, P.PRED_LIKE, b"%a%")
    words = table.string_like_bitmaps(predicate)
    expected = [lo.dictionary_matches(chunk.segments[0].string_dictionary, b"%a%", P.PRED_LIKE) for chunk in table.chunks]
    assert np.array_equal(words, np.concatenate(expected))
    struct, keepalive = build_scan_predicate(table, predicate)
    assert struct.value_id_bounds == keepalive.ctypes.data and len(keepalive) == len(words)


def test_binary_table_like_bitmaps():
    from hyrise_b200.binary_table import NativeBinaryTable

    checked = 0
    for name in ("StringSegment/Dictionary.bin", "FixedStringDictionaryMultipleChunks.bin",
                 "FixedStringDictionaryNullValue.bin", "AllTypesMixColumn/Dictionary.bin"):
        native = NativeBinaryTable(os.path.join(GOLDEN, "bin", name))
        try:
            for column, definition in enumerate(native.table.column_definitions):
                if definition.data_type != capi.TYPE_STRING:
                    continue
                for pattern in (b"%", b"a%", b"%a%b%", b"_b%", b"%e"):
                    for condition in LIKES:
                        expected = np.concatenate(
                            [lo.dictionary_matches(chunk.segments[column].string_dictionary, pattern, condition)
                             for chunk in native.table.chunks] + [np.zeros(0, dtype=np.uint32)])
                        assert np.array_equal(native.like_bitmaps(column, pattern, condition), expected), (name, pattern)
                        checked += 1
        finally:
            native.close()
    assert checked > 0
    lib = capi.load_library()
    count = C.c_uint32()
    native = NativeBinaryTable(os.path.join(GOLDEN, "bin", "StringSegment/Dictionary.bin"))
    try:
        int_columns = [c for c, d in enumerate(native.table.column_definitions) if d.data_type != capi.TYPE_STRING]
        if int_columns:
            assert lib.hyb_binary_table_like_bitmaps(native.ptr, int_columns[0], b"%", 1, P.PRED_LIKE, None,
                                                     C.byref(count)) == capi.HYB_ERR_INVALID
    finally:
        native.close()


def test_binary_table_dictionary_of_empty_strings(tmp_path):
    # a chunk whose dictionary holds only "" has no characters in the parsed file (chars.data() == NULL)
    from hyrise_b200.binary_table import NativeBinaryTable, write_binary_table

    values = np.array([b"", b"", b"a_b", b"", b"xyz", b""], dtype="S")
    table = Table.from_columns([ColumnDefinition("s", capi.TYPE_STRING)], [values], chunk_size=2).encode("Dictionary")
    assert table.chunks[0].segments[0].dictionary_size == 1
    path = str(tmp_path / "empty_strings.bin")
    write_binary_table(table, path)
    native = NativeBinaryTable(path)
    try:
        for pattern in (b"%", b"_%", b"", b"%b"):
            for condition in LIKES:
                expected = np.concatenate([lo.dictionary_matches(chunk.segments[0].string_dictionary, pattern, condition)
                                           for chunk in native.table.chunks])
                assert np.array_equal(native.like_bitmaps(0, pattern, condition), expected), (pattern, condition)
    finally:
        native.close()
