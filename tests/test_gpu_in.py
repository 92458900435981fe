"""`<column> [NOT] IN (<literal>, ...)` TableScans on the device (hyb_table_scan_in): PosLists and per-chunk offsets
bit-exact against the row-by-row restatement (in_scan_oracle.py) for every column type x encoding x condition x list
shape, chunks of mixed encodings, empty chunks and partial tiles, position-filtered inputs (a previous scan's output and
a left join's PosList with NULL_ROW_IDs); TPC-H sf-0.01 Q12 / Q16 / Q19 predicates against SQLite; the scan's PosList as
an aggregate's filter; the error codes, the stats and the C++ mirror."""
import ctypes as C
import os
import sqlite3
import subprocess

import numpy as np
import pytest

import in_scan_oracle as ino
import oracle_lib as orc
from conftest import GOLDEN, REPO
from helpers import assert_aggregate_outputs_equal, assert_pos_lists_equal
from hyrise_b200 import capi
from hyrise_b200.binary_table import NativeBinaryTable, write_binary_table
from hyrise_b200.device import Aggregate, Expression, InList, build_in_predicate
from hyrise_b200.storage import ColumnDefinition, Table

pytestmark = pytest.mark.gpu
P = capi
CONDITIONS = [P.PRED_IN, P.PRED_NOT_IN]
NUMPY = {P.TYPE_INT32: np.int32, P.TYPE_INT64: np.int64, P.TYPE_FLOAT32: np.float32, P.TYPE_FLOAT64: np.float64}
CHUNKS = [2, 5, 16_383, 16_384, 0, 16_385, 700]  # a tile never straddles chunks; chunk 4 has no rows


def check(device, table, device_table, in_list, device_filter=None, oracle_filter=None, ascending=True,
          dictionary_matches=None):
    expected = ino.table_scan_in(table, in_list, oracle_filter, ascending)
    result = device.table_scan_in(device_table, in_list, device_filter, dictionary_matches)
    try:
        assert_pos_lists_equal(result.to_host(), result.chunk_offsets(), expected)
    except AssertionError as error:
        raise AssertionError(f"{in_list}: {error}") from error
    return result, expected


def ragged_table(definitions, chunks, spec, bitpacking=False) -> Table:
    table = Table.from_columns(definitions, [np.zeros(0, dtype=NUMPY.get(d.data_type, "S8")) for d in definitions],
                               [np.zeros(0, dtype=bool) if d.nullable else None for d in definitions])
    table._raw = chunks
    return table.encode(spec, bitpacking=bitpacking)


SPECIALS = {
    P.TYPE_INT32: [16777216, 16777217, 2**31 - 1, -2**31, 0],
    P.TYPE_INT64: [2**53, 2**53 + 1, 2**63 - 1, -2**63, 0],
    P.TYPE_FLOAT32: [np.nan, -0.0, 0.0, np.inf, float(np.float32(0.05)), 16777216.0],
    P.TYPE_FLOAT64: [np.nan, -0.0, 0.0, -np.inf, 0.05, 2.0**53],
}


def column_values(rng, data_type, rows, wide):
    values = rng.integers(-3000, 3000, rows) if wide else rng.integers(-40, 40, rows)
    if data_type in (P.TYPE_FLOAT32, P.TYPE_FLOAT64):
        values = values.astype(np.float64) + np.where(rng.random(rows) < 0.25, 0.5, 0.0)
    special = rng.random(rows) < 0.03
    specials = np.array(SPECIALS[data_type], dtype=object)
    out = values.astype(object)
    out[special] = specials[rng.integers(0, len(specials), int(special.sum()))]
    return np.array(list(out), dtype=NUMPY[data_type])


# Numeric columns: every type Unencoded (NULL-free and nullable) and Dictionary (nullable; narrow: 1-byte value-IDs,
# wide: 2-byte value-IDs), int32 also FrameOfReference; the bitpacking table packs the dictionary / FoR vectors.
def numeric_layout():
    layout = []
    for data_type in NUMPY:
        layout += [(data_type, "Unencoded", False, False), (data_type, "Unencoded", True, False),
                   (data_type, "Dictionary", True, False), (data_type, "Dictionary", False, True)]
        if data_type == P.TYPE_INT32:
            layout += [(data_type, "FrameOfReference", True, False), (data_type, "FrameOfReference", False, True)]
    return layout


def numeric_table(rng, bitpacking=False):
    layout = numeric_layout()
    definitions = [ColumnDefinition(f"c{i}", t, nullable) for i, (t, _, nullable, _) in enumerate(layout)]
    chunks = []
    for rows in CHUNKS:
        chunks.append([(column_values(rng, t, rows, wide), (rng.random(rows) < 0.1) if nullable else None)
                       for t, _, nullable, wide in layout])
    return ragged_table(definitions, chunks, [encoding for _, encoding, _, _ in layout], bitpacking), layout


@pytest.fixture(scope="module")
def numeric_tables():
    rng = np.random.default_rng(21)
    return {"fixed-width": numeric_table(rng), "bitpacking": numeric_table(rng, bitpacking=True)}


EDGES = [np.int32(-2**31), np.int32(2**31 - 1), np.int32(16777217), np.int64(2**53 + 1), np.int64(-2**63),
         np.int64(2**63 - 1), 9007199254740992.0, np.float32(16777216.0), 0.05, np.float32(0.05), -0.0, 0.0, float("nan"),
         float("inf"), np.float32(-np.inf), 5e-324, np.float32(1e-45), np.float32(3.4028235e38), 16777217.0, 2.5]


def numeric_lists(rng, data_type, values):
    present = [v for v in values.tolist() if v == v][:200] or [1]

    def pick(count):
        return [NUMPY[data_type](present[int(i)]) if data_type != P.TYPE_FLOAT64 else float(present[int(i)])
                for i in rng.integers(0, len(present), count)]

    one = pick(1)
    return {
        "empty": [],
        "one": one,
        "duplicates": one + pick(2) + one + one,
        "null": pick(3) + [None],
        "only-null": [None],
        "incompatible": ["x", b"y"],
        "mixed": [int(present[0]) if data_type in (P.TYPE_INT32, P.TYPE_INT64) else 3, float(pick(1)[0]) + 0.5,
                  np.float32(pick(1)[0]), "z", int(2**40), *pick(2)],
        "edges": EDGES + pick(2),
        "thousand": pick(1000),
        "eight": pick(8),
    }


@pytest.mark.parametrize("variant", ["fixed-width", "bitpacking"])
def test_numeric_matrix(device, numeric_tables, variant):
    table, layout = numeric_tables[variant]
    kinds = {(segment.encoding, segment.vector_type) for chunk in table.chunks for segment in chunk.segments}
    if variant == "fixed-width":
        assert {(P.ENC_DICTIONARY, P.VEC_FIXED_1B), (P.ENC_DICTIONARY, P.VEC_FIXED_2B),
                (P.ENC_FRAME_OF_REFERENCE, P.VEC_FIXED_1B), (P.ENC_FRAME_OF_REFERENCE, P.VEC_FIXED_2B)} <= kinds
    else:
        assert {(P.ENC_DICTIONARY, P.VEC_BITPACKED), (P.ENC_FRAME_OF_REFERENCE, P.VEC_BITPACKED)} <= kinds
    rng = np.random.default_rng(5)
    device_table = device.upload(table)
    for column, (data_type, _, _, _) in enumerate(layout):
        values = np.concatenate([chunk.segments[column].decode() for chunk in table.chunks])
        for name, elements in numeric_lists(rng, data_type, values).items():
            for condition in CONDITIONS:
                check(device, table, device_table, InList(column, condition, elements))[0].free()
    device_table.drop()


def test_four_byte_value_ids_and_mixed_encodings(device):
    # a 70 000-distinct-value chunk (4-byte value-IDs); the same column Unencoded, Dictionary and FoR in other chunks
    rng = np.random.default_rng(8)
    definitions = [ColumnDefinition("a", P.TYPE_INT32, True), ColumnDefinition("b", P.TYPE_FLOAT64, True)]
    sizes = [70_000, 3, 0, 20_000, 9_000, 16_384]
    chunks = []
    for rows in sizes:
        a = rng.permutation(max(rows, 1))[:rows].astype(np.int32) - 100
        b = rng.permutation(max(rows, 1))[:rows].astype(np.float64) / 2
        chunks.append([(a, rng.random(rows) < 0.05), (b, rng.random(rows) < 0.05)])
    table = ragged_table(definitions, chunks, "Dictionary")
    table.encode("Unencoded", chunk_ids=[1, 3])
    table.encode(["FrameOfReference", "Unencoded"], chunk_ids=[4])
    encodings = {chunk.segments[0].encoding for chunk in table.chunks}
    assert encodings == {P.ENC_DICTIONARY, P.ENC_UNENCODED, P.ENC_FRAME_OF_REFERENCE}
    assert table.chunks[0].segments[0].vector_type == P.VEC_FIXED_4B
    device_table = device.upload(table)
    lists = [[5], list(range(0, 2000, 3)), [-100, -99, -98, 5000, 69_899], [1.5, 2.0, None], [0.5, 7.0, 10_000.5],
             list(rng.integers(-100, 70_000, 1000)), []]
    for elements in lists:
        for column in (0, 1):
            for condition in CONDITIONS:
                check(device, table, device_table, InList(column, condition, elements))[0].free()
    device_table.drop()


def string_table(rng, chunk_sizes=(2, 5, 16_385, 0, 3_000), bitpacking=False):
    alphabet = [b"a", b"b", b"\x80", b"\xff", b"ab", b"MAIL", b"SHIP"]
    pool = sorted({b"".join(alphabet[int(i)] for i in rng.integers(0, len(alphabet), int(rng.integers(0, 4))))
                   for _ in range(300)})
    pool = np.array(pool, dtype="S")
    definitions = [ColumnDefinition("s", P.TYPE_STRING, True), ColumnDefinition("t", P.TYPE_STRING)]
    chunks = []
    for index, rows in enumerate(chunk_sizes):
        s = pool[rng.integers(0, len(pool), rows)]
        t = pool[rng.integers(0, 3 if index == 2 else len(pool), rows)]  # chunk 2 of t: a 3-entry dictionary
        chunks.append([(s, rng.random(rows) < 0.1), (t, None)])
    return ragged_table(definitions, chunks, "Dictionary", bitpacking), [bytes(v) for v in pool]


@pytest.mark.parametrize("bitpacking", [False, True])
def test_string_matrix(device, bitpacking):
    rng = np.random.default_rng(13)
    table, pool = string_table(rng, bitpacking=bitpacking)
    device_table = device.upload(table)
    picks = lambda count: [pool[int(i)] for i in rng.integers(0, len(pool), count)]  # noqa: E731
    one = picks(1)
    lists = {
        "empty": [], "one": one, "duplicates": one + one + picks(2), "null": picks(2) + [None],
        "incompatible": [1, 2.5, None], "mixed": ["ab", 1, None, 2.5] + picks(2),
        "edges": [b"", b"a", b"ab", b"\xff", b"\x80\x80", b"absent"], "thousand": picks(1000),
        "all": list(pool), "run": pool[:40], "eight": picks(8),
    }
    for elements in lists.values():
        for column in (0, 1):
            for condition in CONDITIONS:
                check(device, table, device_table, InList(column, condition, elements))[0].free()
    device_table.drop()


# --- filtered inputs --------------------------------------------------------------------------------------------------
def test_filtered_inputs(device, numeric_tables):
    table, layout = numeric_tables["fixed-width"]
    device_table = device.upload(table)
    column = [i for i, c in enumerate(layout) if c == (P.TYPE_INT32, "Unencoded", True, False)][0]
    dictionary = [i for i, c in enumerate(layout) if c == (P.TYPE_FLOAT64, "Dictionary", True, False)][0]
    first, first_expected = check(device, table, device_table, InList(column, P.PRED_NOT_IN, [3, 4, 5]))
    for elements in ([1.5, -2.0, 0.5, 7.0], [], ["only strings"], [None, 2.5]):
        for condition in CONDITIONS:
            check(device, table, device_table, InList(dictionary, condition, elements), first, first_expected)[0].free()
    first.free()

    # a left join's build-side PosList holds NULL_ROW_IDs: they read as NULL (`m2.a NOT IN ('a', 'b')` shape)
    rng = np.random.default_rng(4)
    key = [i for i, c in enumerate(layout) if c == (P.TYPE_INT32, "Unencoded", False, False)][0]
    probe = Table.from_columns([ColumnDefinition("p", P.TYPE_INT32)], [rng.integers(-60, 60, 3_000).astype(np.int32)],
                               chunk_size=1_000).encode("Dictionary")
    probe_device = device.upload(probe)
    join = device.join_hash(device_table, key, probe_device, 0, P.JOIN_LEFT, -1)
    build_rows, _ = join.to_host()
    assert (build_rows["chunk_id"] == 0xFFFFFFFF).any()
    side = join.pos_list(0)
    host_side = orc.HostPosList(build_rows, np.array([0, len(build_rows)], dtype=np.uint64))
    null_row_matches = 0
    for elements in ([1.5, -2.0, 0.5], [None, 0.5], [], ["a", "b"], [float("nan")]):
        for condition in CONDITIONS:
            result, expected = check(device, table, device_table, InList(dictionary, condition, elements), side,
                                     host_side, ascending=False)
            null_row_matches += int((expected.row_ids["chunk_id"] == 0xFFFFFFFF).sum() > 0)
            result.free()
    assert null_row_matches == 2  # the degenerate NOT IN lists ([] and strings only) select the NULL_ROW_IDs
    side.free()
    join.free()
    probe_device.drop()
    device_table.drop()


def test_string_filtered_and_binary_bitmaps(device, tmp_path):
    rng = np.random.default_rng(17)
    table, pool = string_table(rng, chunk_sizes=(50, 9_000, 1))
    device_table = device.upload(table)
    first, first_expected = check(device, table, device_table, InList(1, P.PRED_IN, pool[::3]))
    for elements in (pool[:50], ["x", None], [], [pool[0], None]):
        for condition in CONDITIONS:
            check(device, table, device_table, InList(0, condition, elements), first, first_expected)[0].free()
    first.free()
    path = os.path.join(tmp_path, "strings.bin")
    write_binary_table(table, path)
    native = NativeBinaryTable(path)
    try:
        native_device = native.upload(device)
        for condition in CONDITIONS:
            elements = pool[5:30] + [b"absent"]
            bitmaps = native.in_bitmaps(0, condition, elements)
            check(device, native.table, native_device, InList(0, condition, elements), dictionary_matches=bitmaps)[0].free()
        native_device.drop()
    finally:
        native.close()
    device_table.drop()


def test_two_pass_option_does_not_matter(device, numeric_tables):
    table, layout = numeric_tables["fixed-width"]
    device_table = device.upload(table)
    in_list = InList(0, P.PRED_IN, [1, 2, 3, 5, 8, 13, 21, 34])
    for two_pass in ("1", "0"):
        device.set_option("scan_two_pass", two_pass)
        check(device, table, device_table, in_list)[0].free()
    device.set_option("scan_two_pass", "1")
    device_table.drop()


# --- TPC-H sf-0.01 against SQLite ------------------------------------------------------------------------------------
def npz_table(name, columns, chunk_size=10_000):
    data = np.load(os.path.join(GOLDEN, "tpch", name))
    types = {"int": P.TYPE_INT32, "string": P.TYPE_STRING}
    definitions = [ColumnDefinition(c, types[str(data["type__" + c])]) for c in columns]
    table = Table.from_columns(definitions, [data[c] for c in columns], chunk_size=chunk_size)
    raw = {c: [bytes(v) if isinstance(v, bytes) else int(v) for v in data[c].tolist()] for c in columns}
    return table, raw


def sqlite_rows(columns, raw, where, parameters):
    connection = sqlite3.connect(":memory:")
    connection.execute(f"CREATE TABLE t ({', '.join(c + ' BLOB' for c in columns)})")  # BLOBs compare with memcmp
    connection.executemany(f"INSERT INTO t VALUES ({', '.join('?' * len(columns))})", zip(*[raw[c] for c in columns]))
    rows = [r[0] - 1 for r in connection.execute(f"SELECT rowid FROM t WHERE {where} ORDER BY rowid", parameters)]
    connection.close()
    return rows


def flat_rows(result, chunk_size):
    rows = result.to_host()
    return (rows["chunk_id"].astype(np.int64) * chunk_size + rows["chunk_offset"]).tolist()


@pytest.mark.parametrize("encoding", ["Dictionary", "Unencoded"])
def test_tpch_in_lists_against_sqlite(device, encoding):
    cases = [
        ("sf-0.01_lineitem_dates.npz", ["l_orderkey", "l_shipmode"], "l_shipmode", P.PRED_IN, [b"MAIL", b"SHIP"]),
        ("sf-0.01_part.npz", ["p_partkey", "p_container"], "p_container", P.PRED_IN,
         [b"SM CASE", b"SM BOX", b"SM PACK", b"SM PKG"]),
        ("sf-0.01_part.npz", ["p_partkey", "p_container"], "p_container", P.PRED_IN,
         [b"MED BAG", b"MED BOX", b"MED PKG", b"MED PACK"]),
        ("sf-0.01_part_in.npz", ["p_partkey", "p_brand", "p_size"], "p_size", P.PRED_IN, [49, 14, 23, 45, 19, 3, 36, 9]),
        ("sf-0.01_part_in.npz", ["p_partkey", "p_brand", "p_size"], "p_brand", P.PRED_NOT_IN, [b"Brand#45"]),
        ("sf-0.01_part_in.npz", ["p_partkey", "p_brand", "p_size"], "p_size", P.PRED_NOT_IN, [1, 2, 3, 50]),
    ]
    chunk_size = 10_000
    for name, columns, column, condition, elements in cases:
        table, raw = npz_table(name, columns, chunk_size)
        table.encode(encoding)
        device_table = device.upload(table)
        in_list = InList(columns.index(column), condition, elements)
        result, _ = check(device, table, device_table, in_list)
        where = f"{column} {'NOT IN' if condition == P.PRED_NOT_IN else 'IN'} ({', '.join('?' * len(elements))})"
        expected = sqlite_rows(columns, raw, where, elements)
        assert flat_rows(result, chunk_size) == expected, (name, column)
        assert len(expected) > 0
        result.free()
        device_table.drop()


def test_in_scan_feeds_an_aggregate(device):
    table, raw = npz_table("sf-0.01_part_in.npz", ["p_partkey", "p_brand", "p_size"])
    table.encode(["FrameOfReference", "Dictionary", "Unencoded"])
    device_table = device.upload(table)
    in_list = InList(2, P.PRED_IN, [49, 14, 23, 45, 19, 3, 36, 9])
    scan, expected_scan = check(device, table, device_table, in_list)
    aggregates = [Aggregate(P.AGG_COUNT_STAR), Aggregate(P.AGG_SUM, Expression.column(0)),
                  Aggregate(P.AGG_MAX, Expression.column(2))]
    output = device.aggregate_hash(device_table, [1], aggregates, input_filter=scan)
    expected = orc.aggregate_hash(table, [1], aggregates, input_filter=expected_scan)
    assert_aggregate_outputs_equal(output, expected)
    scan.free()
    device_table.drop()


# --- errors, stats, mirror -------------------------------------------------------------------------------------------
def raw_scan(device, device_table, struct):
    handle = C.c_uint64()
    return device.lib.hyb_table_scan_in(device.ptr, device_table.handle, C.byref(struct), 0, C.byref(handle))


def test_error_codes(device):
    rng = np.random.default_rng(2)
    table, _ = string_table(rng, chunk_sizes=(7, 9))
    numeric = Table.from_columns([ColumnDefinition("i", P.TYPE_INT32)], [np.arange(20, dtype=np.int32)], chunk_size=8)
    device_table, numeric_device = device.upload(table), device.upload(numeric)
    struct, keep = build_in_predicate(table, InList(0, P.PRED_IN, ["a"]))
    for condition in (P.PRED_EQUALS, P.PRED_LIKE, P.PRED_IS_NULL):
        struct.condition = condition
        assert raw_scan(device, device_table, struct) == P.HYB_ERR_INVALID
    struct.condition = P.PRED_IN
    struct.column_id = 2
    assert raw_scan(device, device_table, struct) == P.HYB_ERR_INVALID
    numeric_struct, numeric_keep = build_in_predicate(numeric, InList(0, P.PRED_IN, [1, 2]))
    numeric_struct.dictionary_matches = keep.ctypes.data  # bitmaps on a numeric column
    assert raw_scan(device, numeric_device, numeric_struct) == P.HYB_ERR_INVALID
    numeric_struct.dictionary_matches = None
    numeric_keep[0].data_type = P.TYPE_STRING  # a non-numeric literal
    assert raw_scan(device, numeric_device, numeric_struct) == P.HYB_ERR_INVALID
    # IN / NOT IN inside hyb_scan_predicate stay unsupported, in scans and in fused aggregate predicates
    from hyrise_b200.device import Predicate
    for condition in CONDITIONS:
        with pytest.raises(capi.UnsupportedOnDevice):
            device.table_scan(numeric_device, Predicate(0, condition, 1))
        with pytest.raises(capi.UnsupportedOnDevice):
            device.aggregate_hash(numeric_device, [], [Aggregate(P.AGG_COUNT_STAR)], predicates=[Predicate(0, condition, 1)])
    device_table.drop()
    numeric_device.drop()


def test_stats_count_column_list_and_matches(device):
    rng = np.random.default_rng(6)
    values = rng.integers(0, 100, 30_000).astype(np.int32)
    table = Table.from_columns([ColumnDefinition("i", P.TYPE_INT32)], [values], chunk_size=10_000)
    device_table = device.upload(table)
    result = device.table_scan_in(device_table, InList(0, P.PRED_IN, [5, 7, 9, 10, 11]))
    stats = device.last_stats()
    matches = result.info()[0]
    assert matches == int(np.isin(values, [5, 7, 9, 10, 11]).sum())
    # column bytes + the uploaded intervals ([5, 5], [7, 7], [9, 11] as int32 pairs) + the RowIDs written
    assert stats.algorithmic_bytes == 4 * 30_000 + 3 * 8 + 8 * matches
    assert stats.input_rows == 30_000 and stats.output_rows == matches
    result.free()
    device_table.drop()


def test_cpp_mirror_in_scan():
    build = subprocess.run(["make", "-C", REPO, "build/in_scan_check"], capture_output=True, text=True)
    assert build.returncode == 0, build.stdout + build.stderr
    run = subprocess.run([os.path.join(REPO, "build", "in_scan_check")], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0, run.stdout + run.stderr
    assert "in_scan_check: ok" in run.stdout
