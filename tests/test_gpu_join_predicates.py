"""JoinHash with secondary predicates on the device (hyb_join_hash_predicates): pairs, partition offsets and order
bit-exact against join_predicates_oracle.ordered, the hyb_join_path of every run asserted under every join_table
setting, the error codes, and TPC-H sf-0.01 joins against SQLite."""
import dataclasses
import os
import sqlite3
import subprocess

import numpy as np
import pytest

import join_predicates_oracle as jpo
import oracle_lib as orc
import join_layouts
import test_gpu_join
from helpers import TPCH, row_ids_equal, tbl
from hyrise_b200 import capi
from hyrise_b200.device import ColumnComparison, Predicate
from hyrise_b200.storage import ColumnDefinition, Table

pytestmark = pytest.mark.gpu

MODES = [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_SEMI, capi.JOIN_ANTI_NULL_AS_FALSE]
KINDS = list(test_gpu_join.TABLE_KINDS)  # auto, hash, direct, direct on the tile kernels, rank
CONDITIONS = [capi.PRED_EQUALS, capi.PRED_NOT_EQUALS, capi.PRED_LESS_THAN, capi.PRED_LESS_THAN_EQUALS,
              capi.PRED_GREATER_THAN, capi.PRED_GREATER_THAN_EQUALS]
TYPES = [capi.TYPE_INT32, capi.TYPE_INT64, capi.TYPE_FLOAT32, capi.TYPE_FLOAT64]
NUMPY = {capi.TYPE_INT32: np.int32, capi.TYPE_INT64: np.int64, capi.TYPE_FLOAT32: np.float32,
         capi.TYPE_FLOAT64: np.float64}


@pytest.fixture(autouse=True)
def restore_table_kind(device):
    yield
    test_gpu_join.select_table_kind(device, "auto")


def predicted_path(build, build_column, build_filter, probe, probe_column, probe_filter, kind) -> int:
    """hyb_join_path of a join with secondary predicates, predicted from the inputs: plan_join_table's table (as
    join_layouts predicts it for every join), the tile kernels' generic loop when there are probe rows, the rerun for a
    duplicated build key (Semi / Anti joins included), and SECONDARY."""
    # a scan's list is in table order; a join's list (one slice over many chunks) is not
    ascending = build_filter is not None and not build_filter.multiple_chunks
    build_facts = join_layouts.side_facts(build, build_column, build_filter, ascending)
    probe_facts = join_layouts.side_facts(probe, probe_column, probe_filter, False)
    # a table without chunks has no column types on the device: its keys count as int32 (prepare_side)
    if not build.chunks:
        build_facts = dataclasses.replace(build_facts, data_type=capi.TYPE_INT32)
    if not probe.chunks:
        probe_facts = dataclasses.replace(probe_facts, data_type=capi.TYPE_INT32)
    path = join_layouts.predict_table(build_facts, probe_facts, kind)[0] | capi.JOIN_PATH_SECONDARY
    if probe_facts.positions:
        path |= capi.JOIN_PATH_PROBE_TILE | (capi.JOIN_PATH_RERUN if build_facts.duplicates else 0)
    return path


def check_join(device, build, build_dev, build_column, probe, probe_dev, probe_column, mode, radix_bits, predicates,
               build_filter=None, probe_filter=None, kinds=KINDS, expected=None):
    """Runs the join under every table setting; asserts result, order, offsets and path. Returns the expected result."""
    host_build = build_filter[0] if build_filter else None
    host_probe = probe_filter[0] if probe_filter else None
    dev_build = build_filter[1] if build_filter else None
    dev_probe = probe_filter[1] if probe_filter else None
    if expected is None:
        expected = jpo.ordered(build, build_column, probe, probe_column, mode, radix_bits, predicates,
                               build_filter=host_build, probe_filter=host_probe)
    for kind in kinds:
        test_gpu_join.select_table_kind(device, kind)
        plain = device.join_hash(build_dev, build_column, probe_dev, probe_column, mode, radix_bits,
                                 build_filter=dev_build, probe_filter=dev_probe)
        plain_path = device.last_stats().path
        plain.free()
        result = device.join_hash(build_dev, build_column, probe_dev, probe_column, mode, radix_bits,
                                  build_filter=dev_build, probe_filter=dev_probe, secondary=predicates)
        path = device.last_stats().path
        context = (kind, mode, radix_bits, predicates, hex(path), hex(plain_path))
        try:
            if predicates:
                assert path == predicted_path(build, build_column, host_build, probe, probe_column, host_probe, kind), \
                    context
            else:
                assert path == plain_path, context
            pairs, _, bits = result.info()
            assert pairs == expected.pair_count, context
            assert bits == expected.radix_bits, context
            assert np.array_equal(result.partition_offsets(), expected.partition_offsets), context
            got_build, got_probe = result.to_host()
            assert row_ids_equal(got_probe, expected.probe), context
            if expected.build is not None:
                assert row_ids_equal(got_build, expected.build), context
        finally:
            result.free()
    return expected


# ---- join_test_runner inputs (the CPU module's cases) --------------------------------------------------------------
PREDICATE_SETS = {
    "none": [],
    "lt": [(0, 0, capi.PRED_LESS_THAN)],
    "ge": [(0, 0, capi.PRED_GREATER_THAN_EQUALS)],
    "ne": [(0, 0, capi.PRED_NOT_EQUALS)],
    "int_long": [(1, 6, capi.PRED_LESS_THAN_EQUALS), (7, 0, capi.PRED_NOT_EQUALS)],
    "float_double": [(2, 4, capi.PRED_GREATER_THAN), (3, 1, capi.PRED_NOT_EQUALS)],
}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("predicate_set", list(PREDICATE_SETS))
def test_join_test_runner_inputs(device, mode, predicate_set):
    predicates = PREDICATE_SETS[predicate_set]
    for sizes in [(10, 15), (15, 10), (0, 10), (10, 0), (15, 15)]:
        for chunk_size in (10, 3, 1):
            left = tbl(f"join_test_runner/input_table_left_{sizes[0]}.tbl", chunk_size)
            right = tbl(f"join_test_runner/input_table_right_{sizes[1]}.tbl", chunk_size)
            left_dev, right_dev = device.upload(left), device.upload(right)
            for left_column, right_column in [(0, 0), (1, 1), (7, 7), (0, 6)]:
                orders = [(right, right_dev, right_column, left, left_dev, left_column, jpo.flip(predicates))]
                if mode == capi.JOIN_INNER:  # both side orders (join_test_runner.cpp:464-479)
                    orders.append((left, left_dev, left_column, right, right_dev, right_column, predicates))
                for build, build_dev, build_column, probe, probe_dev, probe_column, oriented in orders:
                    for radix_bits in (0, 1, 2, 5):
                        # every table setting on one chunk size; the others under "auto"
                        kinds = KINDS if chunk_size == 3 else ["auto"]
                        check_join(device, build, build_dev, build_column, probe, probe_dev, probe_column, mode,
                                   radix_bits, oriented, kinds=kinds)
            left_dev.drop()
            right_dev.drop()


# ---- every numeric type pairing, special values, encodings and NULLs ------------------------------------------------
SPECIAL = {
    capi.TYPE_INT32: [np.iinfo(np.int32).min, np.iinfo(np.int32).max, 0, -1, 1, 16777217, -16777217, 7],
    capi.TYPE_INT64: [np.iinfo(np.int64).min, np.iinfo(np.int64).max, 0, -1, 1, 2 ** 53 + 1, 2 ** 24 + 1, 7],
    capi.TYPE_FLOAT32: [np.nan, np.inf, -np.inf, -0.0, 0.0, 1.0, 16777216.0, 7.0],
    capi.TYPE_FLOAT64: [np.nan, np.inf, -np.inf, -0.0, 0.0, 1.0, 9007199254740992.0, 7.0],
}


def typed_table(rng, rows, keys, chunk_size, encodings, nullable, bitpacking):
    """Key column (int32) + one column per numeric type, values drawn from SPECIAL and a small range; encodings mixed
    across chunks (`encodings` cycles over the chunks)."""
    definitions = [ColumnDefinition("k", capi.TYPE_INT32)] + [
        ColumnDefinition(f"c{t}", t, nullable) for t in TYPES]
    columns = [keys.astype(np.int32)]
    nulls = [None]
    for data_type in TYPES:
        pool = np.array(SPECIAL[data_type], dtype=NUMPY[data_type])
        small = rng.integers(-3, 8, rows).astype(NUMPY[data_type])
        special = pool[rng.integers(0, len(pool), rows)]
        columns.append(np.where(rng.random(rows) < 0.5, special, small).astype(NUMPY[data_type]))
        nulls.append(rng.random(rows) < 0.15 if nullable else None)
    table = Table.from_columns(definitions, columns, nulls, chunk_size)
    for chunk_id in range(table.chunk_count):
        table.encode(encodings[chunk_id % len(encodings)], chunk_ids=[chunk_id], bitpacking=bitpacking)
    return table


@pytest.mark.parametrize("layout", ["unencoded", "mixed", "mixed_bitpacked", "nullable"])
def test_type_pairings(device, layout):
    rng = np.random.default_rng(7)
    encodings = {"unencoded": ["Unencoded"], "mixed": ["Dictionary", "Unencoded", "FrameOfReference"],
                 "mixed_bitpacked": ["FrameOfReference", "Dictionary"], "nullable": ["Dictionary", "Unencoded"]}[layout]
    bitpacking = layout == "mixed_bitpacked"
    nullable = layout == "nullable"
    build = typed_table(rng, 3000, rng.integers(0, 700, 3000), 1000, encodings, nullable, bitpacking)
    probe = typed_table(rng, 5000, rng.integers(-50, 750, 5000), 1024, encodings[::-1], nullable, bitpacking)
    build_dev, probe_dev = device.upload(build), device.upload(probe)
    for build_type in TYPES:
        for probe_type in TYPES:
            for condition in CONDITIONS:
                predicates = [(1 + TYPES.index(build_type), 1 + TYPES.index(probe_type), condition)]
                for mode in (capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_SEMI, capi.JOIN_ANTI_NULL_AS_FALSE):
                    check_join(device, build, build_dev, 0, probe, probe_dev, 0, mode, 3, predicates, kinds=["auto"])
    # four predicates at once, under every table setting
    predicates = [(1, 2, capi.PRED_LESS_THAN_EQUALS), (2, 3, capi.PRED_NOT_EQUALS), (3, 4, capi.PRED_GREATER_THAN_EQUALS),
                  (4, 1, capi.PRED_NOT_EQUALS)]
    for mode in MODES:
        check_join(device, build, build_dev, 0, probe, probe_dev, 0, mode, 5, predicates)
    build_dev.drop()
    probe_dev.drop()


def key_table(keys, extra, chunk_size, encoding="Unencoded"):
    table = Table.from_columns([ColumnDefinition("k", capi.TYPE_INT32), ColumnDefinition("x", capi.TYPE_INT64)],
                               [np.asarray(keys, dtype=np.int32), np.asarray(extra, dtype=np.int64)], None, chunk_size)
    return table.encode(encoding)


def test_unique_and_heavily_duplicated_build_keys(device):
    rng = np.random.default_rng(11)
    # unique, increasing build keys (rank table under auto), and a key repeated 50 000 times
    unique = key_table(np.arange(20_000) * 3, rng.integers(0, 100, 20_000), 4096)
    hot = key_table(np.concatenate([np.full(50_000, 5), np.arange(10, 1000)]),
                    rng.integers(0, 100, 50_990), 8192)
    probe = key_table(np.concatenate([np.full(40, 5), rng.integers(0, 60_000, 9_960)]), rng.integers(0, 100, 10_000), 2048,
                      "FrameOfReference")
    probe_dev = device.upload(probe)
    for build in (unique, hot):
        build_dev = device.upload(build)
        for condition in (capi.PRED_LESS_THAN, capi.PRED_NOT_EQUALS, capi.PRED_EQUALS):
            for mode in MODES:
                check_join(device, build, build_dev, 0, probe, probe_dev, 0, mode, 2, [(1, 1, condition)])
        build_dev.drop()
    probe_dev.drop()


def test_every_candidate_fails_or_passes(device):
    rng = np.random.default_rng(3)
    build = key_table(rng.integers(0, 300, 4000), np.full(4000, 10), 1000)
    probe = key_table(rng.integers(0, 320, 6000), np.full(6000, 10), 1000)
    build_dev, probe_dev = device.upload(build), device.upload(probe)
    for condition, all_pass in ((capi.PRED_NOT_EQUALS, False), (capi.PRED_LESS_THAN, False),
                                (capi.PRED_EQUALS, True), (capi.PRED_GREATER_THAN_EQUALS, True)):
        for mode in MODES:
            expected = check_join(device, build, build_dev, 0, probe, probe_dev, 0, mode, 4, [(1, 1, condition)])
            plain = jpo.ordered(build, 0, probe, 0, mode, 4, [])
            if all_pass:
                assert row_ids_equal(expected.probe, plain.probe)
            elif mode in (capi.JOIN_INNER, capi.JOIN_SEMI):
                assert expected.pair_count == 0
    build_dev.drop()
    probe_dev.drop()


def test_empty_and_one_row_sides(device):
    empty = key_table([], [], 10)
    one = key_table([4], [2], 10)
    other = key_table([4, 4, 5, 4], [1, 2, 3, 2], 3)
    tables = [(t, device.upload(t)) for t in (empty, one, other)]
    for build, build_dev in tables:
        for probe, probe_dev in tables:
            for mode in MODES:
                for condition in (capi.PRED_LESS_THAN, capi.PRED_EQUALS):
                    check_join(device, build, build_dev, 0, probe, probe_dev, 0, mode, 1, [(1, 1, condition)])
    for _, table_dev in tables:
        table_dev.drop()


def test_filters_from_scans_and_left_joins(device):
    rng = np.random.default_rng(5)
    build = typed_table(rng, 3000, rng.integers(0, 400, 3000), 700, ["Dictionary", "Unencoded"], True, False)
    probe = typed_table(rng, 4000, rng.integers(0, 500, 4000), 900, ["FrameOfReference", "Dictionary"], True, False)
    other = key_table(rng.integers(0, 1200, 500), rng.integers(0, 5, 500), 128)  # keys the tables lack: NULL partners
    build_dev, probe_dev, other_dev = device.upload(build), device.upload(probe), device.upload(other)
    predicate = Predicate(2, capi.PRED_GREATER_THAN, 0)
    scans = {}
    for name, table, table_dev in (("build", build, build_dev), ("probe", probe, probe_dev)):
        scan = device.table_scan(table_dev, predicate)
        host = scan.to_host()
        scans[name] = (orc_pos_list(host, scan.chunk_offsets()), scan)
    # a LEFT join's side holding NULL_ROW_IDs: `other` LEFT JOIN table on the key; its table-side list
    lefts = {}
    for name, table, table_dev in (("build", build, build_dev), ("probe", probe, probe_dev)):
        join = device.join_hash(table_dev, 0, other_dev, 0, capi.JOIN_LEFT, 0)
        pos_list = join.pos_list(0)
        host = pos_list.to_host()
        assert (host["chunk_id"] == jpo.INVALID_CHUNK_ID).any()
        lefts[name] = (joined_list(host, table), pos_list, join)
    predicates = [(3, 3, capi.PRED_LESS_THAN), (1, 4, capi.PRED_NOT_EQUALS)]
    for build_filter in (None, scans["build"], lefts["build"]):
        for probe_filter in (None, scans["probe"], lefts["probe"]):
            for mode in MODES:
                check_join(device, build, build_dev, 0, probe, probe_dev, 0, mode, 3, predicates,
                           build_filter=build_filter[:2] if build_filter else None,
                           probe_filter=probe_filter[:2] if probe_filter else None, kinds=["auto", "hash"])
    for _, pos_list, join in lefts.values():
        pos_list.free()
        join.free()
    for _, scan in scans.values():
        scan.free()
    for table_dev in (build_dev, probe_dev, other_dev):
        table_dev.drop()


def orc_pos_list(row_ids, chunk_offsets):
    return orc.HostPosList(row_ids, np.asarray(chunk_offsets, dtype=np.uint64))


def joined_list(row_ids, table):
    """The oracle's form of a join result's side: one slice holding the whole list, read as one PosList over many
    chunks (join_layouts.JoinFilter.host)."""
    return orc.HostPosList(row_ids, np.array([0] + [len(row_ids)] * table.chunk_count, dtype=np.uint64),
                           multiple_chunks=True)


# ---- errors -----------------------------------------------------------------------------------------------------------
def test_errors(device):
    strings = tbl("join_test_runner/input_table_left_10.tbl", 3)  # column 8: string, 0: int
    other = tbl("join_test_runner/input_table_right_10.tbl", 3)
    left_dev, right_dev = device.upload(strings), device.upload(other)
    cases = [
        (capi.JOIN_INNER, [(8, 8, capi.PRED_EQUALS)], capi.HYB_ERR_UNSUPPORTED),         # string x string
        (capi.JOIN_INNER, [(0, 0, capi.PRED_LESS_THAN)] * 5, capi.HYB_ERR_UNSUPPORTED),  # more than 4
        (capi.JOIN_ANTI_NULL_AS_TRUE, [(0, 0, capi.PRED_LESS_THAN)], capi.HYB_ERR_UNSUPPORTED),
        (capi.JOIN_INNER, [(8, 0, capi.PRED_EQUALS)], capi.HYB_ERR_INVALID),             # string x numeric
        (capi.JOIN_INNER, [(0, 8, capi.PRED_EQUALS)], capi.HYB_ERR_INVALID),
        (capi.JOIN_INNER, [(10, 0, capi.PRED_EQUALS)], capi.HYB_ERR_INVALID),            # column out of range
        (capi.JOIN_INNER, [(0, 10, capi.PRED_EQUALS)], capi.HYB_ERR_INVALID),
        (capi.JOIN_INNER, [(0, 0, capi.PRED_LIKE)], capi.HYB_ERR_INVALID),               # unknown condition
        (capi.JOIN_INNER, [(0, 0, capi.PRED_BETWEEN_INCLUSIVE)], capi.HYB_ERR_INVALID),
    ]
    for mode, predicates, status in cases:
        with pytest.raises(capi.HyriseB200Error) as error:
            device.join_hash(left_dev, 0, right_dev, 0, mode, 0, secondary=predicates)
        assert error.value.status == status, (mode, predicates)
    # reserved must be 0
    import ctypes as C
    build_side = capi.JoinSide(left_dev.handle, 0, 0)
    probe_side = capi.JoinSide(right_dev.handle, 0, 0)
    predicate = capi.JoinPredicate(0, 0, capi.PRED_LESS_THAN, 1)
    handle = C.c_uint64()
    assert device.lib.hyb_join_hash_predicates(device.ptr, C.byref(build_side), C.byref(probe_side), capi.JOIN_INNER, 0,
                                               C.byref(predicate), 1, C.byref(handle)) == capi.HYB_ERR_INVALID
    # output chunks are the plain join's only
    result = device.join_hash(left_dev, 0, right_dev, 0, capi.JOIN_INNER, 0, secondary=[(0, 0, capi.PRED_EQUALS)])
    with pytest.raises(capi.UnsupportedOnDevice):
        result.output_chunks()
    result.free()
    # the context still joins correctly afterwards
    check_join(device, other, right_dev, 0, strings, left_dev, 0, capi.JOIN_LEFT, 1, [(0, 0, capi.PRED_LESS_THAN)])
    left_dev.drop()
    right_dev.drop()


def test_algorithmic_bytes(device):
    build = key_table(np.arange(1000), np.arange(1000), 300)
    probe = key_table(np.arange(2000) % 1000, np.arange(2000), 300)
    build_dev, probe_dev = device.upload(build), device.upload(probe)
    device.join_hash(build_dev, 0, probe_dev, 0, capi.JOIN_INNER, 0).free()
    plain = device.last_stats().algorithmic_bytes
    result = device.join_hash(build_dev, 0, probe_dev, 0, capi.JOIN_INNER, 0,
                              secondary=[(1, 1, capi.PRED_LESS_THAN), (1, 1, capi.PRED_NOT_EQUALS)])
    pairs = result.info()[0]
    result.free()
    assert pairs == 1000  # the probe row with x = k + 1000 of every key
    # the int64 column of both sides once each; the written pairs (16 bytes each) as before
    assert device.last_stats().algorithmic_bytes == plain + 8 * (1000 + 2000) - 16 * (2000 - pairs)
    build_dev.drop()
    probe_dev.drop()


# ---- TPC-H sf-0.01 against SQLite -------------------------------------------------------------------------------------
def lineitem_table():
    keys = np.load(os.path.join(TPCH, "sf-0.01_lineitem_keys.npz"))
    dates = np.load(os.path.join(TPCH, "sf-0.01_lineitem_dates.npz"))
    assert np.array_equal(keys["l_orderkey"], dates["l_orderkey"])
    assert np.array_equal(keys["l_linenumber"], dates["l_linenumber"])

    def day(column):
        return np.array([int(value.replace(b"-", b"")) for value in dates[column]], dtype=np.int32)

    columns = [keys["l_orderkey"], keys["l_partkey"], keys["l_suppkey"], day("l_commitdate"), day("l_receiptdate")]
    names = ["l_orderkey", "l_partkey", "l_suppkey", "l_commitdate", "l_receiptdate"]
    table = Table.from_columns([ColumnDefinition(n, capi.TYPE_INT32) for n in names], columns, None, 10_000)
    return table.encode("Automatic"), columns


def test_tpch_q21_exists_core(device):
    table, columns = lineitem_table()
    orderkey, _, suppkey, commit, receipt = columns
    table_dev = device.upload(table)
    late = device.table_scan_columns(table_dev, ColumnComparison(4, capi.PRED_GREATER_THAN, 3))
    late_host = orc_pos_list(late.to_host(), late.chunk_offsets())
    # orderkey self-join: candidates per probe row
    self_join = device.join_hash(table_dev, 0, table_dev, 0, capi.JOIN_INNER, -1)
    assert self_join.info()[0] == 301_389
    self_join.free()
    # EXISTS (l2: same order, other supplier) over the late lines l1: Semi join, probe = l1
    suppkey_differs = [(2, 2, capi.PRED_NOT_EQUALS)]
    semi = check_join(device, table, table_dev, 0, table, table_dev, 0, capi.JOIN_SEMI, -1, suppkey_differs,
                      probe_filter=(late_host, late), kinds=["auto"])
    semi_dev = device.join_hash(table_dev, 0, table_dev, 0, capi.JOIN_SEMI, -1, probe_filter=late,
                                secondary=suppkey_differs)
    exists = semi_dev.pos_list(1)
    exists_host = joined_list(exists.to_host(), table)
    # NOT EXISTS (l3: same order, other supplier, late): AntiNullAsFalse, build = the late lines
    anti = check_join(device, table, table_dev, 0, table, table_dev, 0, capi.JOIN_ANTI_NULL_AS_FALSE, -1, suppkey_differs,
                      build_filter=(late_host, late), probe_filter=(exists_host, exists), kinds=["auto"])
    connection = sqlite3.connect(":memory:")
    connection.execute("CREATE TABLE l (id INTEGER, o INTEGER, s INTEGER, c INTEGER, r INTEGER)")
    connection.executemany("INSERT INTO l VALUES (?, ?, ?, ?, ?)",
                           zip(range(len(orderkey)), orderkey.tolist(), suppkey.tolist(), commit.tolist(), receipt.tolist()))
    connection.execute("CREATE INDEX l_o ON l (o)")
    exists_ids = [row[0] for row in connection.execute(
        "SELECT l1.id FROM l l1 WHERE l1.r > l1.c AND EXISTS (SELECT 1 FROM l l2 WHERE l2.o = l1.o AND l2.s <> l1.s)")]
    final_ids = [row[0] for row in connection.execute(
        "SELECT l1.id FROM l l1 WHERE l1.r > l1.c AND EXISTS (SELECT 1 FROM l l2 WHERE l2.o = l1.o AND l2.s <> l1.s) "
        "AND NOT EXISTS (SELECT 1 FROM l l3 WHERE l3.o = l1.o AND l3.s <> l1.s AND l3.r > l3.c)")]

    def ids(rows):
        return sorted((rows["chunk_id"].astype(np.int64) * 10_000 + rows["chunk_offset"]).tolist())

    assert semi.pair_count == len(exists_ids) and ids(semi.probe) == sorted(exists_ids)
    assert anti.pair_count == len(final_ids) and ids(anti.probe) == sorted(final_ids)
    exists.free()
    semi_dev.free()
    late.free()
    table_dev.drop()


def test_tpch_two_key_self_join(device):
    table, columns = lineitem_table()
    _, partkey, suppkey, _, _ = columns
    table_dev = device.upload(table)
    expected = check_join(device, table, table_dev, 1, table, table_dev, 1, capi.JOIN_INNER, -1,
                          [(2, 2, capi.PRED_EQUALS)], kinds=["auto", "hash"])
    assert expected.pair_count == 511_733
    connection = sqlite3.connect(":memory:")
    connection.execute("CREATE TABLE l (p INTEGER, s INTEGER)")
    connection.executemany("INSERT INTO l VALUES (?, ?)", zip(partkey.tolist(), suppkey.tolist()))
    (count,) = connection.execute("SELECT COUNT(*) FROM l a JOIN l b ON a.p = b.p AND a.s = b.s").fetchone()
    assert count == expected.pair_count
    table_dev.drop()


def test_cpp_mirror_join_predicates():
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    build = subprocess.run(["make", "-C", repo, "build/join_predicates_check"], capture_output=True, text=True)
    assert build.returncode == 0, build.stdout + build.stderr
    run = subprocess.run([os.path.join(repo, "build", "join_predicates_check")], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0 and run.stdout.strip() == "OK", run.stdout + run.stderr
