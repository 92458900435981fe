"""LIKE / NOT LIKE [INSENSITIVE] scans on the device: PosLists and per-chunk offsets bit-exact against the row-by-row
oracle (like_oracle.py), under both unfiltered scan pipelines and with the cp.async.bulk staged kernel on and off;
TPC-H sf-0.01 text against SQLite; LIKE fused into AggregateHash."""
import os
import sqlite3

import numpy as np
import pytest

import like_oracle as lo
import oracle_lib as orc
from conftest import GOLDEN
from helpers import assert_aggregate_outputs_exact, assert_pos_lists_equal, row_ids_equal, tbl
from hyrise_b200 import capi
from hyrise_b200.device import ROW_ID_DTYPE, Aggregate, Expression, Predicate
from hyrise_b200.storage import ColumnDefinition, Table
from test_oracle_like import SCAN_CASES

pytestmark = pytest.mark.gpu
P = capi
LIKES = list(capi.LIKE_CONDITIONS)


@pytest.fixture(autouse=True, params=["single-pass/bulk", "single-pass/no-bulk", "two-pass"])
def scan_variant(device, request):
    """Every case runs under the single-pass look-back pipeline (with and without the TMA-staged kernel, where the column
    qualifies for it) and the two-pass mask / expand pipeline."""
    device.set_option("scan_two_pass", "1" if request.param == "two-pass" else "0")
    device.set_option("scan_bulk", "0" if request.param == "single-pass/no-bulk" else "1")
    yield request.param
    device.set_option("scan_two_pass", "1")  # the context's defaults
    device.set_option("scan_bulk", "0")


def check_like(device, table, device_table, column, pattern, condition, device_filter=None, oracle_filter=None,
               ascending=True):
    expected = lo.table_scan(table, column, pattern, condition, oracle_filter, ascending)
    result = device.table_scan(device_table, Predicate(column, condition, pattern), device_filter)
    try:
        assert_pos_lists_equal(result.to_host(), result.chunk_offsets(), expected)
    except AssertionError as error:
        raise AssertionError(f"{pattern!r} condition {condition}: {error}") from error
    return result, expected


def chunk_classes(table, column, pattern, condition) -> set:
    """The per-chunk test prepare_chunk_tests derives from the bitmap: none / run (range) / set."""
    classes = set()
    for chunk in table.chunks:
        segment = chunk.segments[column]
        matcher = lo.Matcher(pattern, condition)
        bits = np.array([matcher(bytes(e)) for e in segment.string_dictionary], dtype=bool)
        if segment.row_count == 0 or not bits.any():
            classes.add("none")
        else:
            set_ids = np.flatnonzero(bits)
            classes.add("all" if len(set_ids) == len(bits) else
                        "run" if set_ids[-1] - set_ids[0] + 1 == len(set_ids) else "set")
    return classes


@pytest.mark.parametrize("bitpacking", [False, True])
@pytest.mark.parametrize("chunk_size", [2, 5])
def test_reference_fixtures(device, bitpacking, chunk_size):
    # table_scan_string_test.cpp: every LIKE case on dictionary segments (FixedWidth / BitPacking vectors), plus the
    # ...OnReferencedDictSegment form: the LIKE on the output of `a > 0`
    for source in sorted({case[1] for case in SCAN_CASES}):
        table = tbl(source, chunk_size).encode("Dictionary", bitpacking=bitpacking)
        device_table = device.upload(table)
        first = device.table_scan(device_table, Predicate(0, P.PRED_GREATER_THAN, 0))
        first_expected = orc.table_scan(table, Predicate(0, P.PRED_GREATER_THAN, 0))
        for _, case_source, condition, pattern, _ in SCAN_CASES:
            if case_source != source:
                continue
            for variant in LIKES:  # the case's condition and the other three
                check_like(device, table, device_table, 1, pattern, variant)
                check_like(device, table, device_table, 1, pattern, variant, first, first_expected)
        first.free()
        device_table.drop()


def seeded_column(rng, bitpacking=False):
    """One string column over ragged chunks: dictionaries of 1, 200 (1-byte ids), 3 000 and 65 535 entries (2-byte ids),
    one chunk with 70 000 distinct values (4-byte ids), an all-NULL chunk (no dictionary entry) and NULLs elsewhere."""
    colours = [b"almond", b"blue", b"Blush", b"forest", b"green", b"lace", b"PROMO", b"red", b"x\ny"]
    sizes = [(40_000, 1), (9_001, 200), (70_000, 70_000), (1_000, 0), (65_535 * 2 - 7, 65_535), (33_333, 3_000)]
    values, nulls, chunk_sizes = [], [], []
    serial = 0
    for rows, distinct in sizes:
        if distinct == 0:
            values.append(np.full(rows, b"", dtype="S24"))
            nulls.append(np.ones(rows, dtype=bool))
        else:
            pool = np.array([colours[(serial + i) % len(colours)] + b"-%06d" % (serial + i) for i in range(distinct)],
                            dtype="S24")
            serial += distinct
            # every pool entry occurs (the dictionary has exactly `distinct` entries), the rest drawn at random
            column = np.concatenate([pool, pool[rng.integers(0, distinct, max(rows - distinct, 0))]])[:rows]
            rng.shuffle(column)
            values.append(column)
            null = rng.random(rows) < 0.05
            if distinct >= 65_535:
                null[:] = False  # keep every entry present: the id width is the point of these chunks
            nulls.append(null)
        chunk_sizes.append(rows)
    # Table.from_columns cuts fixed-size chunks; build one chunk per entry of `sizes` instead
    table = Table.from_columns([ColumnDefinition("k", capi.TYPE_INT32), ColumnDefinition("s", capi.TYPE_STRING, True)],
                               [np.zeros(0, dtype=np.int32), np.zeros(0, dtype="S24")], [None, np.zeros(0, dtype=bool)])
    table._raw = []
    for column, null in zip(values, nulls):
        keys = rng.integers(0, 1000, len(column)).astype(np.int32)
        table._raw.append([(keys, None), (column, null)])
    table.encode("Dictionary", bitpacking=bitpacking)
    return table


SEEDED_PATTERNS = [b"%", b"%zzz%", b"blue%", b"%green%", b"%-0000%", b"%1", b"%e%-%9%", b"b_u%", b"x%y%", b"%x\ny%",
                   b"%N-%", b"PROMO%"]


@pytest.mark.parametrize("bitpacking", [False, True])
def test_seeded_multi_chunk_column(device, bitpacking):
    table = seeded_column(np.random.default_rng(11), bitpacking)
    widths = [chunk.segments[1].vector_type for chunk in table.chunks]
    if not bitpacking:
        assert {capi.VEC_FIXED_1B, capi.VEC_FIXED_2B, capi.VEC_FIXED_4B} <= set(widths)
    assert [chunk.segments[1].dictionary_size for chunk in table.chunks] == [1, 200, 70_000, 0, 65_535, 3_000]
    device_table = device.upload(table)
    classes = set()
    for pattern in SEEDED_PATTERNS:
        for condition in LIKES:
            classes |= chunk_classes(table, 1, pattern, condition)
            check_like(device, table, device_table, 1, pattern, condition)[0].free()
    assert classes == {"none", "all", "run", "set"}
    device_table.drop()


def test_filtered_inputs(device):
    rng = np.random.default_rng(12)
    table = seeded_column(rng)
    device_table = device.upload(table)
    # a scan's PosList
    first = device.table_scan(device_table, Predicate(0, P.PRED_LESS_THAN, 300))
    first_expected = orc.table_scan(table, Predicate(0, P.PRED_LESS_THAN, 300))
    for pattern in (b"%e%-%9%", b"blue%", b"%"):
        for condition in LIKES:
            check_like(device, table, device_table, 1, pattern, condition, first, first_expected)[0].free()
    first.free()
    # the build side of a Left join: unmatched probe rows carry NULL_ROW_ID, which never matches LIKE (or NOT LIKE)
    probe_keys = rng.integers(-200, 1200, 5_000).astype(np.int32)
    probe = Table.from_columns([ColumnDefinition("p", capi.TYPE_INT32)], [probe_keys], chunk_size=1_000).encode("Dictionary")
    probe_device = device.upload(probe)
    join = device.join_hash(device_table, 0, probe_device, 0, capi.JOIN_LEFT, -1)
    build_rows, _ = join.to_host()
    assert (build_rows["chunk_id"] == 0xFFFFFFFF).any()
    side = join.pos_list(0)
    host_side = lo.HostPosList(build_rows, np.array([0, len(build_rows)], dtype=np.uint64))
    for pattern in (b"%e%-%9%", b"%"):
        for condition in LIKES:
            check_like(device, table, device_table, 1, pattern, condition, side, host_side, ascending=False)[0].free()
    side.free()
    join.free()
    probe_device.drop()
    device_table.drop()


def test_bitmap_contract(device):
    """Padding bits set by the caller and all-NULL chunks (no dictionary entry, no bitmap word) give the clean result."""
    import ctypes as C

    table = seeded_column(np.random.default_rng(13))
    device_table = device.upload(table)
    for pattern, condition in [(b"%e%-%9%", P.PRED_LIKE), (b"%", P.PRED_NOT_LIKE), (b"blue%", P.PRED_NOT_LIKE)]:
        clean = check_like(device, table, device_table, 1, pattern, condition)[0]
        words = table.string_like_bitmaps(Predicate(1, condition, pattern)).copy()
        at = 0
        for chunk in table.chunks:
            size = chunk.segments[1].dictionary_size
            at += (size + 31) // 32
            if size % 32:
                words[at - 1] |= np.uint32(~((1 << (size % 32)) - 1) & 0xFFFFFFFF)
        assert at == len(words)
        struct = capi.ScanPredicate()
        struct.column_id, struct.condition, struct.value_id_bounds = 1, condition, words.ctypes.data
        handle = C.c_uint64()
        capi.check(device.lib.hyb_table_scan(device.ptr, device_table.handle, C.byref(struct), 0, C.byref(handle)))
        from hyrise_b200.device import DevicePosList
        padded = DevicePosList(device, handle.value)
        assert row_ids_equal(padded.to_host(), clean.to_host())
        assert np.array_equal(padded.chunk_offsets(), clean.chunk_offsets())
        padded.free()
        clean.free()
    # a missing bitmap is an error, not a CPU fallback
    struct = capi.ScanPredicate()
    struct.column_id, struct.condition = 1, P.PRED_LIKE
    handle = C.c_uint64()
    assert device.lib.hyb_table_scan(device.ptr, device_table.handle, C.byref(struct), 0, C.byref(handle)) == \
        capi.HYB_ERR_INVALID
    struct.column_id = 0  # int column
    assert device.lib.hyb_table_scan(device.ptr, device_table.handle, C.byref(struct), 0, C.byref(handle)) == \
        capi.HYB_ERR_INVALID
    device_table.drop()


def tpch_table(name, columns):
    data = np.load(os.path.join(GOLDEN, "tpch", f"sf-0.01_{name}.npz"))
    types = {"int": capi.TYPE_INT32, "string": capi.TYPE_STRING}
    definitions = [ColumnDefinition(c, types[str(data["type__" + c])]) for c in columns]
    table = Table.from_columns(definitions, [data[c] for c in columns], chunk_size=1_000).encode("Dictionary")
    return table, {c: [bytes(v) if isinstance(v, bytes) else v for v in data[c].tolist()] for c in columns}


TPCH_CASES = [
    ("orders_comment", "o_comment", P.PRED_NOT_LIKE, b"%special%requests%"),  # Q13
    ("part", "p_name", P.PRED_LIKE, b"%green%"),                             # Q9
    ("part", "p_name", P.PRED_LIKE, b"forest%"),                             # Q20
    ("part", "p_type", P.PRED_LIKE, b"%BRASS"),                              # Q2
    ("part", "p_type", P.PRED_LIKE, b"PROMO%"),
    ("part", "p_type", P.PRED_NOT_LIKE, b"MEDIUM POLISHED%"),                # Q16
    ("part", "p_container", P.PRED_LIKE, b"MED%"),
    ("part", "p_type", P.PRED_LIKE_INSENSITIVE, b"%medium%brass"),
    ("orders_comment", "o_comment", P.PRED_NOT_LIKE_INSENSITIVE, b"%SPECIAL%_equests%"),
]


@pytest.mark.parametrize("case", TPCH_CASES, ids=[f"{c[1]}-{c[2]}-{c[3].decode()}" for c in TPCH_CASES])
def test_tpch_against_sqlite(device, case):
    name, column, condition, pattern = case
    columns = ["o_orderkey", "o_comment"] if name == "orders_comment" else ["p_partkey", "p_name", "p_type", "p_container"]
    table, raw = tpch_table(name, columns)
    assert all(value.isascii() for value in raw[column])  # SQLite's `_` (a character) and the byte-wise `.` agree
    device_table = device.upload(table)
    result, _ = check_like(device, table, device_table, columns.index(column), pattern, condition)
    positions = [int(r["chunk_id"]) * 1_000 + int(r["chunk_offset"]) for r in result.to_host()]
    device_keys = sorted(raw[columns[0]][p] for p in positions)
    connection = sqlite3.connect(":memory:")
    connection.execute("CREATE TABLE t (key INTEGER, value TEXT)")
    connection.executemany("INSERT INTO t VALUES (?, ?)", zip(raw[columns[0]], [v.decode() for v in raw[column]]))
    sensitive = condition in (P.PRED_LIKE, P.PRED_NOT_LIKE)
    connection.execute(f"PRAGMA case_sensitive_like={'ON' if sensitive else 'OFF'}")
    negation = "NOT " if condition in (P.PRED_NOT_LIKE, P.PRED_NOT_LIKE_INSENSITIVE) else ""
    sqlite_keys = sorted(key for (key,) in connection.execute(f"SELECT key FROM t WHERE value {negation}LIKE ?",
                                                              (pattern.decode(),)))
    connection.close()
    assert device_keys == sqlite_keys and len(sqlite_keys) > 0
    result.free()
    device_table.drop()


def aggregate_table(rng):
    """s: LIKE column (ragged dictionaries, NULLs); g: 4-value string group key; v: int64 values; k: int range column;
    m: 1 where `s LIKE '%e%-%9%'` holds (the oracle's stand-in for the LIKE predicate)."""
    rows = 150_000
    words = np.array([b"%s-%05d" % (c, i) for i, c in enumerate([b"green", b"blue", b"red", b"lace"] * 900)], dtype="S16")
    s = words[rng.integers(0, len(words), rows)]
    s_nulls = rng.random(rows) < 0.03
    g = np.array([b"AIR", b"MAIL", b"SHIP", b"TRUCK"], dtype="S8")[rng.integers(0, 4, rows)]
    v = rng.integers(-10 ** 9, 10 ** 9, rows).astype(np.int64)
    k = rng.integers(0, 1000, rows).astype(np.int32)
    matcher = lo.Matcher(b"%e%-%9%", P.PRED_LIKE)
    m = np.array([0 if null else int(matcher(bytes(x))) for x, null in zip(s, s_nulls)], dtype=np.int32)
    definitions = [ColumnDefinition("s", capi.TYPE_STRING, True), ColumnDefinition("g", capi.TYPE_STRING),
                   ColumnDefinition("v", capi.TYPE_INT64), ColumnDefinition("k", capi.TYPE_INT32),
                   ColumnDefinition("m", capi.TYPE_INT32)]
    table = Table.from_columns(definitions, [s, g, v, k, m], [s_nulls, None, None, None, None], chunk_size=20_000)
    return table.encode("Dictionary")


@pytest.mark.parametrize("kernel", ["register-tile", "general"])
def test_fused_like_in_aggregate(device, scan_variant, kernel):
    if scan_variant != "two-pass":
        pytest.skip("the aggregate does not use the scan pipelines")
    table = aggregate_table(np.random.default_rng(14))
    device_table = device.upload(table)
    column = Expression.column
    aggregates = [Aggregate(P.AGG_SUM, column(2)), Aggregate(P.AGG_COUNT, column(2)), Aggregate(P.AGG_COUNT_STAR)]
    if kernel == "general":
        aggregates.append(Aggregate(P.AGG_MIN, column(2)))  # MIN is not on the fast paths
    device.set_option("aggregate_stream", "1")
    for condition in (P.PRED_LIKE, P.PRED_NOT_LIKE):
        predicates = [Predicate(0, condition, b"%e%-%9%"), Predicate(3, P.PRED_LESS_THAN, 700)]
        stand_in = [Predicate(4, P.PRED_EQUALS if condition == P.PRED_LIKE else P.PRED_NOT_EQUALS, 1),
                    Predicate(0, P.PRED_IS_NOT_NULL), Predicate(3, P.PRED_LESS_THAN, 700)]
        got = device.aggregate_hash(device_table, [1], aggregates, predicates=predicates)
        path = device.last_stats().path
        expected = orc.aggregate_hash(table, [1], aggregates, predicates=stand_in)
        assert_aggregate_outputs_exact(got, expected)
        assert path not in (P.AGG_PATH_STREAM_STATIC, P.AGG_PATH_STREAM_GENERIC)
        if kernel == "general":
            assert path == P.AGG_PATH_GENERAL, path
        else:
            assert path in (P.AGG_PATH_TILE_G4, P.AGG_PATH_TILE_G8), path
    device_table.drop()


def test_fused_like_never_streams(device, scan_variant):
    """A plan the streaming aggregate accepts with a range predicate on the string column: float values in 1-byte
    dictionaries, a 1-byte string group key, a NULL-free LIKE column with 2-byte value-IDs. The streaming row loop reads a
    dictionary predicate as a value-ID range, so with LIKE the same plan must fall to the register-tile kernel; both
    results are bit-exact (sums of sixteenths are exact in any order)."""
    if scan_variant != "two-pass":
        pytest.skip("the aggregate does not use the scan pipelines")
    import aggregate_layouts as layouts

    rng = np.random.default_rng(15)
    sizes = [20_000, 20_000, 20_000]
    rows = sum(sizes)
    words = np.array([b"%s-%05d" % (c, i) for i, c in enumerate([b"green", b"blue", b"red", b"lace"] * 750)], dtype="S16")
    s = layouts.with_distinct(rng, rows, words)
    matcher = lo.Matcher(b"%e%-%9%", P.PRED_LIKE)
    m = np.array([int(matcher(bytes(x))) for x in s], dtype=np.int32)
    columns = [s, layouts.strings(rng.integers(0, 4, rows)), layouts.sixteenths(rng, rows), rng.integers(0, 1000, rows)
               .astype(np.int32), m]
    definitions = [ColumnDefinition("s", capi.TYPE_STRING), ColumnDefinition("g", capi.TYPE_STRING),
                   ColumnDefinition("v", capi.TYPE_FLOAT32), ColumnDefinition("k", capi.TYPE_INT32),
                   ColumnDefinition("m", capi.TYPE_INT32)]
    table = layouts.table_from_chunks(definitions, columns, sizes, "Dictionary")
    for chunk in table.chunks:
        assert chunk.segments[0].vector_type == capi.VEC_FIXED_2B and chunk.segments[0].nulls is None
        assert chunk.segments[1].vector_type == capi.VEC_FIXED_1B and chunk.segments[1].dictionary_codes is not None
        assert chunk.segments[2].vector_type == capi.VEC_FIXED_1B
    assert chunk_classes(table, 0, b"%e%-%9%", P.PRED_LIKE) == {"set"}  # a range test would drop or add rows
    device_table = device.upload(table)
    column = Expression.column
    aggregates = [Aggregate(P.AGG_SUM, column(2)), Aggregate(P.AGG_COUNT, column(2)), Aggregate(P.AGG_COUNT_STAR)]
    device.set_option("aggregate_stream", "1")

    # control: with a range predicate on `s` the plan streams
    control = [Predicate(0, P.PRED_LESS_THAN, bytes(np.sort(words)[1_500])), Predicate(3, P.PRED_LESS_THAN, 700)]
    got = device.aggregate_hash(device_table, [1], aggregates, predicates=control)
    assert device.last_stats().path in (P.AGG_PATH_STREAM_STATIC, P.AGG_PATH_STREAM_GENERIC), device.last_stats().path
    assert_aggregate_outputs_exact(got, orc.aggregate_hash(table, [1], aggregates, predicates=control))

    for condition in (P.PRED_LIKE, P.PRED_NOT_LIKE):
        predicates = [Predicate(0, condition, b"%e%-%9%"), Predicate(3, P.PRED_LESS_THAN, 700)]
        stand_in = [Predicate(4, P.PRED_EQUALS if condition == P.PRED_LIKE else P.PRED_NOT_EQUALS, 1),
                    Predicate(3, P.PRED_LESS_THAN, 700)]
        got = device.aggregate_hash(device_table, [1], aggregates, predicates=predicates)
        path = device.last_stats().path
        assert path in (P.AGG_PATH_TILE_G4, P.AGG_PATH_TILE_G8), path
        assert_aggregate_outputs_exact(got, orc.aggregate_hash(table, [1], aggregates, predicates=stand_in))
    device_table.drop()
