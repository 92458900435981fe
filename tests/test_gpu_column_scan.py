"""Column-vs-column TableScans on the device (hyb_table_scan_columns): PosLists and per-chunk offsets bit-exact against
the CPU restatement (column_scan_oracle.py) for every numeric type pair, condition and encoding, string pairs with
partly, not or fully overlapping dictionaries, position-filtered and chained inputs; TPC-H sf-0.01 Q4 / Q12 / Q21
predicates against SQLite; the error codes; the C++ mirror."""
import ctypes as C
import os
import sqlite3
import subprocess

import numpy as np
import pytest

import column_scan_oracle as cso
import oracle_lib as orc
from conftest import GOLDEN, REPO
from helpers import assert_pos_lists_equal
from hyrise_b200 import capi
from hyrise_b200.binary_table import NativeBinaryTable, write_binary_table
from hyrise_b200.device import ColumnComparison, Predicate, build_column_scan_predicate
from hyrise_b200.storage import ColumnDefinition, Table

pytestmark = pytest.mark.gpu
P = capi
CONDITIONS = [P.PRED_EQUALS, P.PRED_NOT_EQUALS, P.PRED_LESS_THAN, P.PRED_LESS_THAN_EQUALS, P.PRED_GREATER_THAN,
              P.PRED_GREATER_THAN_EQUALS]
TYPES = [P.TYPE_INT32, P.TYPE_INT64, P.TYPE_FLOAT32, P.TYPE_FLOAT64]
NUMPY = {P.TYPE_INT32: np.int32, P.TYPE_INT64: np.int64, P.TYPE_FLOAT32: np.float32, P.TYPE_FLOAT64: np.float64}


def check(device, table, device_table, comparison, device_filter=None, oracle_filter=None, ascending=True, strings=None,
          right_in_left=None):
    expected = cso.table_scan_columns(table, comparison, oracle_filter, ascending, strings)
    result = device.table_scan_columns(device_table, comparison, device_filter, right_in_left)
    try:
        assert_pos_lists_equal(result.to_host(), result.chunk_offsets(), expected)
    except AssertionError as error:
        raise AssertionError(f"{comparison}: {error}") from error
    return result, expected


def ragged_table(definitions, chunks, spec, bitpacking=False) -> Table:
    """One chunk per entry of `chunks` (a list of [(values, nulls) per column]), encoded with `spec`."""
    table = Table.from_columns(definitions, [np.zeros(0, dtype=NUMPY.get(d.data_type, "S8")) for d in definitions],
                               [np.zeros(0, dtype=bool) if d.nullable else None for d in definitions])
    table._raw = chunks
    return table.encode(spec, bitpacking=bitpacking)


def numeric_values(rng, data_type, rows, wide):
    """Values that collide across types: integers in a small range, and for floats also halves and large integers
    (16777217 and its neighbours), so that equal, unequal and rounding-equal pairs all occur."""
    if wide:
        base = rng.integers(-600, 600, rows)
    else:
        base = rng.integers(-12, 12, rows)
    if data_type in (P.TYPE_FLOAT32, P.TYPE_FLOAT64):
        values = base.astype(np.float64) + np.where(rng.random(rows) < 0.25, 0.5, 0.0)
    else:
        values = base.astype(np.int64)
    special = rng.random(rows) < 0.02
    values = values.astype(np.float64) if data_type in (P.TYPE_FLOAT32, P.TYPE_FLOAT64) else values
    values[special] = 16777217 if data_type != P.TYPE_FLOAT32 else 16777216
    return values.astype(NUMPY[data_type])


# Encodings of the numeric columns: every type unencoded and dictionary-encoded, int32 also FrameOfReference; each with
# a NULL-free and a nullable (about 10 % NULL) column of a narrow domain, plus a NULL-free wide (2-byte value-ID) one.
def numeric_layout():
    columns = []
    for data_type in TYPES:
        encodings = ["Unencoded", "Dictionary"] + (["FrameOfReference"] if data_type == P.TYPE_INT32 else [])
        for encoding in encodings:
            for domain in ("narrow", "nullable", "wide"):
                columns.append((data_type, encoding, domain))
    return columns


def numeric_table(rng, chunk_sizes, bitpacking=False, all_null_chunk=None):
    layout = numeric_layout()
    definitions = [ColumnDefinition(f"c{i}", t, domain == "nullable") for i, (t, _, domain) in enumerate(layout)]
    chunks = []
    for chunk_id, rows in enumerate(chunk_sizes):
        raw = []
        for data_type, _, domain in layout:
            values = numeric_values(rng, data_type, rows, domain == "wide")
            nulls = None
            if domain == "nullable":
                nulls = np.ones(rows, dtype=bool) if chunk_id == all_null_chunk else rng.random(rows) < 0.1
            raw.append((values, nulls))
        chunks.append(raw)
    return ragged_table(definitions, chunks, [encoding for _, encoding, _ in layout], bitpacking), layout


@pytest.fixture(scope="module")
def numeric_tables():
    rng = np.random.default_rng(11)
    return {
        # chunk sizes 2 and 5, and around the 16 384-row tile (a tile never straddles chunks)
        "fixed-width": numeric_table(rng, [2, 5, 16_383, 16_384, 16_385, 700], all_null_chunk=5),
        "bitpacking": numeric_table(rng, [5, 2, 16_385, 333], bitpacking=True, all_null_chunk=0),
    }


def pairs_of(layout):
    """Every ordered pair of columns whose domains match (narrow values meet nullable ones), and each column with
    itself."""
    for left, (_, _, left_domain) in enumerate(layout):
        for right, (_, _, right_domain) in enumerate(layout):
            if (left_domain == "wide") == (right_domain == "wide"):
                yield left, right


@pytest.mark.parametrize("variant", ["fixed-width", "bitpacking"])
def test_numeric_pairs(device, numeric_tables, variant):
    table, layout = numeric_tables[variant]
    kinds = {(segment.encoding, segment.vector_type) for chunk in table.chunks for segment in chunk.segments}
    if variant == "fixed-width":
        assert {(P.ENC_DICTIONARY, P.VEC_FIXED_1B), (P.ENC_DICTIONARY, P.VEC_FIXED_2B),
                (P.ENC_FRAME_OF_REFERENCE, P.VEC_FIXED_1B), (P.ENC_FRAME_OF_REFERENCE, P.VEC_FIXED_2B)} <= kinds
    else:
        assert {(P.ENC_DICTIONARY, P.VEC_BITPACKED), (P.ENC_FRAME_OF_REFERENCE, P.VEC_BITPACKED)} <= kinds
    device_table = device.upload(table)
    type_pairs = set()
    for left, right in pairs_of(layout):
        type_pairs.add((layout[left][0], layout[right][0]))
        for condition in CONDITIONS:
            check(device, table, device_table, ColumnComparison(left, condition, right))[0].free()
    assert len(type_pairs) == 16
    device_table.drop()


def test_four_byte_value_ids_and_empty_chunk(device):
    # a 70 000-distinct-value chunk (4-byte value-IDs) next to a chunk without rows
    rng = np.random.default_rng(5)
    definitions = [ColumnDefinition("a", P.TYPE_INT64), ColumnDefinition("b", P.TYPE_FLOAT64, True)]
    rows = 70_000
    a = rng.permutation(rows).astype(np.int64)
    b = rng.permutation(rows).astype(np.float64) + np.where(rng.random(rows) < 0.3, 0.0, 0.5)
    chunks = [[(a, None), (b, rng.random(rows) < 0.05)],
              [(np.zeros(0, dtype=np.int64), None), (np.zeros(0), np.zeros(0, dtype=bool))],
              [(a[:9], None), (b[:9], np.zeros(9, dtype=bool))]]
    table = ragged_table(definitions, chunks, "Dictionary")
    assert table.chunks[0].segments[0].vector_type == P.VEC_FIXED_4B and table.chunks[1].size == 0
    device_table = device.upload(table)
    for condition in CONDITIONS:
        for left, right in [(0, 1), (1, 0), (0, 0)]:
            check(device, table, device_table, ColumnComparison(left, condition, right))[0].free()
    device_table.drop()


def test_two_pass_option_does_not_matter(device, numeric_tables):
    table, layout = numeric_tables["fixed-width"]
    device_table = device.upload(table)
    comparisons = [ColumnComparison(0, P.PRED_LESS_THAN, 4), ColumnComparison(len(layout) - 1, P.PRED_EQUALS, 2)]
    reference = []
    for comparison in comparisons:
        result, _ = check(device, table, device_table, comparison)
        reference.append((result.to_host().copy(), result.chunk_offsets().copy()))
        result.free()
    device.set_option("scan_two_pass", "0")
    device.set_option("scan_bulk", "1")
    try:
        for comparison, (rows, offsets) in zip(comparisons, reference):
            result = device.table_scan_columns(device_table, comparison)
            assert np.array_equal(result.to_host(), rows) and np.array_equal(result.chunk_offsets(), offsets)
            result.free()
    finally:
        device.set_option("scan_two_pass", "1")
        device.set_option("scan_bulk", "0")
    device_table.drop()


# --- strings ------------------------------------------------------------------------------------------------------------
def string_table(rng, overlap, chunk_sizes=(3, 16_390, 5, 2_000), bitpacking=False):
    """Two nullable string columns. overlap: 'partial' (shared and own values), 'none' (disjoint pools), 'full' (the same
    pool). Values include the empty string, proper prefixes and bytes >= 0x80 (no trailing NUL: 'S' arrays drop it)."""
    shared = [b"", b"a", b"ab", b"abc", b"b", b"\x80", b"\x80\x01", b"a\x00b", b"zz", b"1994-01-01", b"1994-01-02"]
    left_own = [b"aa", b"abd", b"\xff", b"m", b"1994-01-015"]
    right_own = [b"ac", b"abb", b"\xfe", b"n", b"1993-12-31"]
    if overlap == "partial":
        left_pool, right_pool = shared + left_own, shared + right_own
    elif overlap == "none":
        left_pool, right_pool = left_own + [b"c"], right_own + [b"d"]
    else:
        left_pool = right_pool = shared
    definitions = [ColumnDefinition("l", P.TYPE_STRING, True), ColumnDefinition("r", P.TYPE_STRING, True),
                   ColumnDefinition("k", P.TYPE_INT32)]
    chunks, strings = [], {0: [], 1: []}
    for chunk_id, rows in enumerate(chunk_sizes):
        raw = []
        for column, pool in ((0, left_pool), (1, right_pool)):
            values = [pool[i] for i in rng.integers(0, len(pool), rows)]
            nulls = rng.random(rows) < 0.08
            if chunk_id == 2 and column == 1:
                nulls[:] = True  # an all-NULL chunk: no dictionary entry on the right
            strings[column] += [None if null else value for value, null in zip(values, nulls)]
            raw.append((np.array(values, dtype="S12"), nulls))
        raw.append((np.arange(rows, dtype=np.int32), None))
        chunks.append(raw)
    return ragged_table(definitions, chunks, "Dictionary", bitpacking), strings


@pytest.mark.parametrize("bitpacking", [False, True])
@pytest.mark.parametrize("overlap", ["partial", "none", "full"])
def test_string_pairs(device, overlap, bitpacking):
    table, strings = string_table(np.random.default_rng(3), overlap, bitpacking=bitpacking)
    device_table = device.upload(table)
    for condition in CONDITIONS:
        for left, right in [(0, 1), (1, 0), (0, 0), (1, 1)]:
            check(device, table, device_table, ColumnComparison(left, condition, right), strings=strings)[0].free()
    device_table.drop()


# --- filtered inputs --------------------------------------------------------------------------------------------------
def test_filtered_inputs(device, numeric_tables):
    table, layout = numeric_tables["fixed-width"]
    device_table = device.upload(table)
    nullable_int, nullable_double = 1, [i for i, c in enumerate(layout) if c == (P.TYPE_FLOAT64, "Dictionary", "nullable")][0]
    # from a previous scan's output (ascending)
    first = device.table_scan(device_table, Predicate(0, P.PRED_GREATER_THAN, -3))
    first_expected = orc.table_scan(table, Predicate(0, P.PRED_GREATER_THAN, -3))
    for condition in CONDITIONS:
        check(device, table, device_table, ColumnComparison(nullable_int, condition, nullable_double), first,
              first_expected)[0].free()
    # chained: one column-vs-column scan's output is the input of another
    second, second_expected = check(device, table, device_table, ColumnComparison(0, P.PRED_LESS_THAN_EQUALS, 3), first,
                                    first_expected)
    third, _ = check(device, table, device_table, ColumnComparison(nullable_int, P.PRED_NOT_EQUALS, nullable_double),
                     second, second_expected)
    unfiltered, unfiltered_expected = check(device, table, device_table, ColumnComparison(2, P.PRED_GREATER_THAN, 5))
    check(device, table, device_table, ColumnComparison(0, P.PRED_EQUALS, 3), unfiltered, unfiltered_expected)[0].free()
    for result in (first, second, third, unfiltered):
        result.free()

    # from a join's PosList: input order, one chunk, NULL_ROW_IDs of a Left join never match
    rng = np.random.default_rng(1)
    probe = Table.from_columns([ColumnDefinition("p", P.TYPE_INT32)], [rng.integers(-15, 15, 3_000).astype(np.int32)],
                               chunk_size=1_000).encode("Dictionary")
    probe_device = device.upload(probe)
    join = device.join_hash(device_table, 0, probe_device, 0, P.JOIN_LEFT, -1)
    build_rows, _ = join.to_host()
    assert (build_rows["chunk_id"] == 0xFFFFFFFF).any()
    side = join.pos_list(0)
    host_side = orc.HostPosList(build_rows, np.array([0, len(build_rows)], dtype=np.uint64))
    for condition in CONDITIONS:
        check(device, table, device_table, ColumnComparison(nullable_int, condition, nullable_double), side, host_side,
              ascending=False)[0].free()
    side.free()
    join.free()
    probe_device.drop()
    device_table.drop()


def test_string_pairs_filtered(device):
    table, strings = string_table(np.random.default_rng(9), "partial")
    device_table = device.upload(table)
    first, first_expected = check(device, table, device_table, ColumnComparison(0, P.PRED_LESS_THAN, 1), strings=strings)
    for condition in CONDITIONS:
        check(device, table, device_table, ColumnComparison(1, condition, 0), first, first_expected,
              strings=strings)[0].free()
    first.free()
    device_table.drop()


# --- TPC-H sf-0.01 lineitem against SQLite -----------------------------------------------------------------------------
LINEITEM_COLUMNS = ["l_orderkey", "l_linenumber", "l_shipdate", "l_commitdate", "l_receiptdate", "l_shipmode"]
CHUNK = 1_000


@pytest.fixture(scope="module")
def lineitem():
    data = np.load(os.path.join(GOLDEN, "tpch", "sf-0.01_lineitem_dates.npz"))
    types = {"int": P.TYPE_INT32, "string": P.TYPE_STRING}
    definitions = [ColumnDefinition(c, types[str(data["type__" + c])]) for c in LINEITEM_COLUMNS]
    table = Table.from_columns(definitions, [data[c] for c in LINEITEM_COLUMNS], chunk_size=CHUNK).encode("Dictionary")
    raw = {c: [bytes(v) if isinstance(v, bytes) else int(v) for v in data[c].tolist()] for c in LINEITEM_COLUMNS}
    connection = sqlite3.connect(":memory:")
    connection.execute("CREATE TABLE lineitem (l_orderkey INTEGER, l_linenumber INTEGER, l_shipdate BLOB, "
                       "l_commitdate BLOB, l_receiptdate BLOB, l_shipmode BLOB)")  # BLOBs compare with memcmp
    connection.executemany("INSERT INTO lineitem VALUES (?, ?, ?, ?, ?, ?)", zip(*[raw[c] for c in LINEITEM_COLUMNS]))
    yield table, raw, connection
    connection.close()


def keys_of(raw, pos_list_rows):
    positions = [int(r["chunk_id"]) * CHUNK + int(r["chunk_offset"]) for r in pos_list_rows]
    return sorted((raw["l_orderkey"][p], raw["l_linenumber"][p]) for p in positions)


def sqlite_keys(connection, where):
    return sorted(connection.execute(f"SELECT l_orderkey, l_linenumber FROM lineitem WHERE {where}").fetchall())


def column(name):
    return LINEITEM_COLUMNS.index(name)


def test_tpch_q4_q21_dates(device, lineitem):
    table, raw, connection = lineitem
    strings = {column(c): raw[c] for c in ("l_shipdate", "l_commitdate", "l_receiptdate")}
    device_table = device.upload(table)
    want = sqlite_keys(connection, "l_commitdate < l_receiptdate")
    assert 0 < len(want) < table.row_count
    q4, _ = check(device, table, device_table,
                  ColumnComparison(column("l_commitdate"), P.PRED_LESS_THAN, column("l_receiptdate")), strings=strings)
    q21, _ = check(device, table, device_table,
                   ColumnComparison(column("l_receiptdate"), P.PRED_GREATER_THAN, column("l_commitdate")), strings=strings)
    assert keys_of(raw, q4.to_host()) == want
    assert np.array_equal(q21.to_host(), q4.to_host())  # the operands swapped: the same rows
    q4.free()
    q21.free()
    device_table.drop()


def q12_chain(device, table, device_table, raw, right_in_left=None):
    strings = {column(c): raw[c] for c in ("l_shipdate", "l_commitdate", "l_receiptdate")}
    mail = device.table_scan(device_table, Predicate(column("l_shipmode"), P.PRED_EQUALS, b"MAIL"))
    mail_expected = orc.table_scan(table, Predicate(column("l_shipmode"), P.PRED_EQUALS, b"MAIL"))
    translations = right_in_left or {}
    commit_receipt = ColumnComparison(column("l_commitdate"), P.PRED_LESS_THAN, column("l_receiptdate"))
    second, second_expected = check(device, table, device_table, commit_receipt, mail, mail_expected, strings=strings,
                                     right_in_left=translations.get("commit_receipt"))
    ship_commit = ColumnComparison(column("l_shipdate"), P.PRED_LESS_THAN, column("l_commitdate"))
    third, third_expected = check(device, table, device_table, ship_commit, second, second_expected, strings=strings,
                                  right_in_left=translations.get("ship_commit"))
    fourth = device.table_scan(device_table, Predicate(column("l_receiptdate"), P.PRED_GREATER_THAN_EQUALS, b"1994-01-01"),
                               third)
    rows = fourth.to_host()
    for result in (mail, second, third, fourth):
        result.free()
    return rows


def test_tpch_q12_chain(device, lineitem):
    table, raw, connection = lineitem
    device_table = device.upload(table)
    rows = q12_chain(device, table, device_table, raw)
    want = sqlite_keys(connection, "l_shipmode = CAST('MAIL' AS BLOB) AND l_commitdate < l_receiptdate AND "
                                   "l_shipdate < l_commitdate AND l_receiptdate >= CAST('1994-01-01' AS BLOB)")
    assert len(want) > 0 and keys_of(raw, rows) == want
    device_table.drop()


def test_tpch_through_binary_table(device, lineitem, tmp_path):
    table, raw, connection = lineitem
    path = os.path.join(tmp_path, "lineitem_dates.bin")
    write_binary_table(table, path)
    native = NativeBinaryTable(path, pinned=True)
    try:
        device_table = native.upload(device)
        translations = {
            "commit_receipt": native.column_translation(column("l_commitdate"), column("l_receiptdate")),
            "ship_commit": native.column_translation(column("l_shipdate"), column("l_commitdate")),
        }
        assert np.array_equal(translations["commit_receipt"],
                              table.string_column_translation(column("l_commitdate"), column("l_receiptdate")))
        rows = q12_chain(device, native.table, device_table, raw, translations)
        want = sqlite_keys(connection, "l_shipmode = CAST('MAIL' AS BLOB) AND l_commitdate < l_receiptdate AND "
                                       "l_shipdate < l_commitdate AND l_receiptdate >= CAST('1994-01-01' AS BLOB)")
        assert keys_of(raw, rows) == want
        device_table.drop()
    finally:
        native.close()


# --- errors and stats -------------------------------------------------------------------------------------------------
def scan_status(device, device_table, left, condition, right, right_in_left=None) -> int:
    struct = capi.ColumnScanPredicate()
    struct.left_column_id, struct.condition, struct.right_column_id = left, condition, right
    keep = None
    if right_in_left is not None:
        keep = np.ascontiguousarray(right_in_left, dtype=np.uint32)
        struct.right_in_left = keep.ctypes.data
    handle = C.c_uint64()
    status = device.lib.hyb_table_scan_columns(device.ptr, device_table.handle, C.byref(struct), 0, C.byref(handle))
    if status == P.HYB_OK:
        device.lib.hyb_pos_list_free(device.ptr, handle.value)
    del keep
    return status


def test_error_codes(device):
    table, _ = string_table(np.random.default_rng(2), "partial", chunk_sizes=(7, 9))
    device_table = device.upload(table)
    translation = table.string_column_translation(0, 1)
    assert scan_status(device, device_table, 0, P.PRED_EQUALS, 2, translation) == P.HYB_ERR_INVALID  # string x int
    assert scan_status(device, device_table, 2, P.PRED_EQUALS, 0) == P.HYB_ERR_INVALID
    for like in capi.LIKE_CONDITIONS:
        assert scan_status(device, device_table, 0, like, 1, translation) == P.HYB_ERR_UNSUPPORTED
    for other in (P.PRED_BETWEEN_INCLUSIVE, P.PRED_IN, P.PRED_IS_NULL, 99):
        assert scan_status(device, device_table, 0, other, 1, translation) == P.HYB_ERR_INVALID
    assert scan_status(device, device_table, 0, P.PRED_LESS_THAN, 1) == P.HYB_ERR_INVALID  # no right_in_left
    assert scan_status(device, device_table, 0, P.PRED_LESS_THAN, 3, translation) == P.HYB_ERR_INVALID  # out of range
    assert scan_status(device, device_table, 3, P.PRED_LESS_THAN, 2) == P.HYB_ERR_INVALID
    assert scan_status(device, device_table, 0, P.PRED_LESS_THAN, 1, translation) == P.HYB_OK
    struct, _ = build_column_scan_predicate(table, ColumnComparison(0, P.PRED_EQUALS, 1))
    assert struct.right_in_left
    device_table.drop()


def test_stats_count_both_columns_and_the_translation(device):
    table, _ = string_table(np.random.default_rng(4), "partial", chunk_sizes=(100, 50))
    device_table = device.upload(table)
    result = device.table_scan_columns(device_table, ColumnComparison(0, P.PRED_NOT_EQUALS, 1))
    stats = device.last_stats()
    column_bytes = sum(chunk.segments[c].attribute_vector.nbytes for chunk in table.chunks for c in (0, 1))
    words = sum(len(chunk.segments[1].string_dictionary) for chunk in table.chunks)
    matches = result.info()[0]
    assert stats.algorithmic_bytes == column_bytes + 4 * words + 8 * matches  # + the RowIDs written
    assert stats.input_rows == table.row_count and stats.output_rows == matches
    result.free()
    device_table.drop()


def test_cpp_mirror_column_scan():
    build = subprocess.run(["make", "-C", REPO, "build/column_scan_check"], capture_output=True, text=True)
    assert build.returncode == 0, build.stdout + build.stderr
    run = subprocess.run([os.path.join(REPO, "build", "column_scan_check")], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0 and run.stdout.strip() == "OK", run.stdout + run.stderr
