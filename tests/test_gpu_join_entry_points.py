"""JoinHash's entry points (hyb_join_hash, _partition, _partition_push, _materialize, _side_positions, _hash_distributed).
This pins what hyb_join_hash reports on every table kind, probe family and the rerun (hyb_operator_stats: path,
kernel_launches, input_rows, output_rows, algorithmic_bytes), what the partitioning calls report and write, and the status
of every rejection, each followed by a join on the same context that still matches the oracle."""
import ctypes as C

import numpy as np
import pytest

import join_layouts as layouts
import oracle_lib as orc
import test_gpu_join
from helpers import random_table, row_ids_equal, rows_with_keys
from hyrise_b200 import capi as P
from hyrise_b200.device import Predicate
from hyrise_b200.storage import ColumnDefinition, Table
from test_gpu_join_paths import device_filter

pytestmark = pytest.mark.gpu
BUILDERS = {builder.__name__: builder for builder in layouts.GPU_BUILDERS}
SEMI_ANTI = (P.JOIN_SEMI, P.JOIN_ANTI_NULL_AS_TRUE, P.JOIN_ANTI_NULL_AS_FALSE)


@pytest.fixture(autouse=True)
def restore_table_kind(device):
    yield
    test_gpu_join.select_table_kind(device, "auto")


def key_bytes(table, column, pos_list):
    """What a join reads of one side's keys: a PosList's RowIDs and keys, or the key column once (values, or the
    attribute vector plus FrameOfReference block minima; no dictionary, no NULL flags)."""
    type_size = 4 if table.column_definitions[column].data_type == P.TYPE_INT32 else 8
    if pos_list is not None:
        return len(pos_list.row_ids) * (8 + type_size)
    total = 0
    for chunk in table.chunks:
        segment = chunk.segments[column]
        if segment.encoding == P.ENC_UNENCODED:
            total += type_size * segment.row_count
        else:
            total += segment.attribute_vector.nbytes
            if segment.encoding == P.ENC_FRAME_OF_REFERENCE:
                total += 4 * ((segment.row_count + P.FOR_BLOCK_SIZE - 1) // P.FOR_BLOCK_SIZE)
    return total


def expected_launches(first_call, build_table, build_facts, probe_facts, path):
    """Key bounds (first join over a build (table, key column) whose table has rows, whatever its filter) + int64 hash
    table keys + build + count, scan, write and offsets of the probe + the rerun: position lists (count, scan, fill, sort),
    the exact count and its scan, and a second probe."""
    launches = int(first_call and build_table.row_count > 0)
    if build_facts.positions:
        launches += 1 + int(path & P.JOIN_PATH_TABLE_MASK == P.JOIN_PATH_TABLE_HASH_WIDE)
    if probe_facts.positions:
        launches += 4
    if path & P.JOIN_PATH_RERUN:
        launches += 10
    return launches


def check_stats(device, bounds_seen, sides, column, mode, radix_bits, facts, kinds=tuple(layouts.TABLE_KINDS)):
    """sides: (host table, DeviceTable, HostPosList or None, DevicePosList or None) of the build and the probe side.
    bounds_seen: the (table handle, column) pairs whose key bounds the library has cached."""
    (build, build_dev, build_list, build_dev_list), (probe, probe_dev, probe_list, probe_dev_list) = sides
    expected = orc.join_hash(build, column, probe, column, mode, radix_bits, build_filter=build_list,
                             probe_filter=probe_list)
    read = key_bytes(build, column, build_list) + key_bytes(probe, column, probe_list)
    for kind in kinds:
        test_gpu_join.select_table_kind(device, kind)
        first_call = (build_dev.handle, column) not in bounds_seen
        result = device.join_hash(build_dev, column, probe_dev, column, mode, radix_bits, build_filter=build_dev_list,
                                  probe_filter=probe_dev_list)
        bounds_seen.add((build_dev.handle, column))
        stats = device.last_stats()
        try:
            path = layouts.predict_path(*facts, kind, mode)
            pairs = result.info()[0]
            want = (path, expected_launches(first_call, build, *facts, path), facts[1].positions, pairs,
                    read + pairs * (8 if mode in SEMI_ANTI else 16))
            got = (stats.path, stats.kernel_launches, stats.input_rows, stats.output_rows, stats.algorithmic_bytes)
            assert got == want, (kind, mode, hex(path))
            assert pairs == expected.pair_count, (kind, mode)
            assert np.array_equal(result.partition_offsets(), expected.partition_offsets), (kind, mode)
            got_build, got_probe = result.to_host()
            assert row_ids_equal(got_probe, expected.probe), (kind, mode)
            if expected.build is not None:
                assert row_ids_equal(got_build, expected.build), (kind, mode)
        finally:
            result.free()


# table kind x probe family x rerun, int32 and int64 keys, a filtered build side (ascending scan) and a filtered probe
# side (a LEFT join's build side, NULL_ROW_IDs included), an empty probe side and a build side of NULLs only
STATS_LAYOUTS = ["span_for2", "span_plain64", "span_shifted_int64", "int64_collisions_duplicated", "chunks_empty_middle",
                 "shifted_duplicates", "poslist_ascending_scan", "poslist_left_probe", "empty_probe_int64", "all_null_build"]


@pytest.mark.parametrize("name", STATS_LAYOUTS)
def test_stats_on_each_path(device, name):
    layout = BUILDERS[name]()
    column = layout.column
    build_dev, probe_dev = device.upload(layout.build), device.upload(layout.probe)
    owners, bounds_seen, lists = [], set(), {}
    for side, spec, table, this_dev in (("build", layout.build_filter, layout.build, build_dev),
                                        ("probe", layout.probe_filter, layout.probe, probe_dev)):
        lists[side] = (None, None)
        if spec is None:
            continue
        other_dev = device.upload(spec.table) if spec.table is not None else None
        pos_list, owner = device_filter(device, spec, this_dev, other_dev, column)
        if spec.source == "left-join":   # that join cached the key bounds of its build side
            bounds_seen.add(((this_dev if spec.side == 0 else other_dev).handle, column))
        lists[side] = (spec.host(table, column), pos_list)
        owners += [owner, pos_list] + ([other_dev] if other_dev else [])
    facts = layouts.layout_facts(layout, lists["build"][0], lists["probe"][0])
    sides = ((layout.build, build_dev) + lists["build"], (layout.probe, probe_dev) + lists["probe"])
    try:
        for mode in (P.JOIN_INNER, P.JOIN_LEFT, P.JOIN_SEMI):
            check_stats(device, bounds_seen, sides, column, mode, 3, facts)
        assert (build_dev.handle, column) in bounds_seen
    finally:
        for owner in reversed(owners):
            owner.drop() if hasattr(owner, "drop") else owner.free()
        build_dev.drop()
        probe_dev.drop()


def small_tables(rng):
    """A dense int32 / int64 build with duplicate keys (FrameOfReference and Dictionary chunks) and a probe table."""
    build = random_table(rng, 9_000, 2_500).encode("FrameOfReference")
    build.encode("Dictionary", [1])
    probe = random_table(rng, 20_000, 6_000).encode("Unencoded")
    probe.encode("FrameOfReference", [2])
    return build, probe


@pytest.mark.parametrize("column", [0, 1, 4])
def test_stats_filtered_and_empty_sides(device, column):
    """Scan-filtered build and probe sides, each also filtered to nothing: no build or probe kernel then, but the key
    bounds of a build table with rows are still computed once."""
    build, probe = small_tables(np.random.default_rng(90 + column))
    build_dev, probe_dev = device.upload(build), device.upload(probe)
    bounds_seen = set()
    some = Predicate(4, P.PRED_LESS_THAN, 120)
    nothing = Predicate(4, P.PRED_GREATER_THAN, 10 ** 6)
    scans = []
    try:
        filters = {}
        for side, table, table_dev in (("build", build, build_dev), ("probe", probe, probe_dev)):
            for label, predicate in (("some", some), ("nothing", nothing)):
                scans.append(device.table_scan(table_dev, predicate))
                filters[side, label] = (orc.table_scan(table, predicate), scans[-1])
        for build_label, probe_label in ((None, None), ("some", None), (None, "some"), ("some", "some"),
                                         ("nothing", "some"), (None, "nothing"), ("nothing", "nothing")):
            build_list = filters["build", build_label] if build_label else (None, None)
            probe_list = filters["probe", probe_label] if probe_label else (None, None)
            facts = (layouts.side_facts(build, column, build_list[0], True),
                     layouts.side_facts(probe, column, probe_list[0], True))
            sides = ((build, build_dev) + build_list, (probe, probe_dev) + probe_list)
            for mode in (P.JOIN_INNER, P.JOIN_ANTI_NULL_AS_TRUE):
                check_stats(device, bounds_seen, sides, column, mode, 2, facts, kinds=("auto", "hash", "direct-tiles"))
    finally:
        for scan in scans:
            scan.free()
        build_dev.drop()
        probe_dev.drop()


# ---- the partitioning entry points -----------------------------------------------------------------------------------
def side_positions(device, side):
    positions = C.c_uint64()
    P.check(device.lib.hyb_join_side_positions(device.ptr, C.byref(side), C.byref(positions)))
    return positions.value


def expected_tuples(table, column, host_filter, chunk_id_base):
    rows = rows_with_keys(table, column, host_filter)
    keys = np.array([key for _, key in rows if key is not None], dtype=np.int64)
    row_ids = np.array([(chunk_id + chunk_id_base) | (offset << 32) for (chunk_id, offset), key in rows
                        if key is not None], dtype=np.int64)
    return rows, keys, row_ids


def check_partition_stats(device, launches, positions):
    stats = device.last_stats()
    assert (stats.kernel_launches, stats.input_rows, stats.output_rows, stats.algorithmic_bytes) == \
        (launches, positions, 0, 16 * positions)


@pytest.mark.parametrize("predicate", [None, Predicate(4, P.PRED_LESS_THAN, 150),
                                       Predicate(4, P.PRED_GREATER_THAN, 10 ** 6)], ids=["table", "scan", "empty"])
def test_partition_materialize_and_push(device, predicate):
    import torch

    rng = np.random.default_rng(14)
    table = random_table(rng, 25_000, 7_000).encode("Automatic")
    table_dev = device.upload(table)
    scan = device.table_scan(table_dev, predicate) if predicate else None
    host_filter = orc.table_scan(table, predicate) if predicate else None
    cuda = torch.device("cuda", 0)
    try:
        for column in (0, 1):
            side = P.JoinSide(table_dev.handle, column, scan.handle if scan else 0)
            positions = side_positions(device, side)
            rows, want_keys, want_rows = expected_tuples(table, column, host_filter, 500)
            assert positions == len(rows)
            # hyb_join_materialize: {key, global RowID} per position, RowID -1 for a NULL key
            keys = torch.zeros(positions + 1, dtype=torch.int64, device=cuda)
            row_ids = torch.zeros(positions + 1, dtype=torch.int64, device=cuda)
            torch.cuda.synchronize()
            P.check(device.lib.hyb_join_materialize(device.ptr, C.byref(side), 500, keys.data_ptr(), row_ids.data_ptr()))
            stats = device.last_stats()
            assert (stats.kernel_launches, stats.input_rows, stats.output_rows, stats.algorithmic_bytes) == \
                (1, positions, positions, 16 * positions)
            got_keys, got_rows = keys[:positions].cpu().numpy(), row_ids[:positions].cpu().numpy()
            not_null = np.array([key is not None for _, key in rows], dtype=bool)
            assert np.array_equal(got_rows[~not_null], np.full((~not_null).sum(), -1))
            assert np.array_equal(got_rows[not_null], want_rows) and np.array_equal(got_keys[not_null], want_keys)
            for partition_count in (1, 4):
                # hyb_join_partition: the non-NULL tuples split stably by key & (partition_count - 1)
                offsets = (C.c_uint64 * (partition_count + 1))()
                P.check(device.lib.hyb_join_partition(device.ptr, C.byref(side), partition_count, 500, keys.data_ptr(),
                                                      row_ids.data_ptr(), offsets))
                check_partition_stats(device, 4 if positions else 0, positions)
                offsets = np.array(offsets[:], dtype=np.int64)
                owner = want_keys & (partition_count - 1)
                order = np.argsort(owner, kind="stable")
                assert np.array_equal(np.diff(offsets), np.bincount(owner, minlength=partition_count))
                assert np.array_equal(keys[:offsets[-1]].cpu().numpy(), want_keys[order])
                assert np.array_equal(row_ids[:offsets[-1]].cpu().numpy(), want_rows[order])
                # hyb_join_partition_push: the same groups, at the destinations the exchange callback names
                received = {}

                def exchange(_user, counts, dest_keys, dest_rows):
                    for p in range(partition_count):
                        received[p] = (torch.full((int(counts[p]) + 1,), -7, dtype=torch.int64, device=cuda),
                                       torch.full((int(counts[p]) + 1,), -7, dtype=torch.int64, device=cuda))
                        dest_keys[p], dest_rows[p] = received[p][0].data_ptr(), received[p][1].data_ptr()
                    torch.cuda.synchronize()
                    return 0

                callback = P.EXCHANGE_FN(exchange)
                P.check(device.lib.hyb_join_partition_push(device.ptr, C.byref(side), partition_count, 500, callback, None))
                check_partition_stats(device, 4 if positions else 0, positions)
                for p in range(partition_count):
                    begin, end = int(offsets[p]), int(offsets[p + 1])
                    assert np.array_equal(received[p][0][:end - begin].cpu().numpy(), want_keys[order][begin:end])
                    assert np.array_equal(received[p][1][:end - begin].cpu().numpy(), want_rows[order][begin:end])
                    assert int(received[p][0][end - begin]) == -7
    finally:
        if scan:
            scan.free()
        table_dev.drop()


# ---- rejections ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def reject_tables(device):
    rng = np.random.default_rng(15)
    build, probe = small_tables(rng)
    words = np.array([b"w%02d" % i for i in rng.integers(0, 40, 3_000)], dtype="S")
    strings = Table.from_columns([ColumnDefinition("s", P.TYPE_STRING)], [words], chunk_size=1_000).encode("Dictionary")
    devices = [device.upload(table) for table in (build, probe, strings)]
    yield (build, probe), devices
    for table_dev in devices:
        table_dev.drop()


def good_join(device, reject_tables):
    """A join on the same context after a rejection: still bit-exact against the oracle."""
    (build, probe), (build_dev, probe_dev, _) = reject_tables
    expected = orc.join_hash(build, 0, probe, 0, P.JOIN_INNER, 2)
    result = device.join_hash(build_dev, 0, probe_dev, 0, P.JOIN_INNER, 2)
    try:
        got_build, got_probe = result.to_host()
        assert row_ids_equal(got_probe, expected.probe) and row_ids_equal(got_build, expected.build)
        assert np.array_equal(result.partition_offsets(), expected.partition_offsets)
    finally:
        result.free()


def join_status(device, build_side, probe_side, mode=P.JOIN_INNER, radix_bits=2):
    out = C.c_uint64()
    return device.lib.hyb_join_hash(device.ptr, build_side and C.byref(build_side), probe_side and C.byref(probe_side),
                                    mode, radix_bits, C.byref(out))


def test_join_hash_rejections(device, reject_tables):
    (build, _), (build_dev, probe_dev, strings_dev) = reject_tables
    side = lambda table, column=0, pos_list=0: P.JoinSide(table.handle, column, pos_list)   # noqa: E731
    scan = device.table_scan(build_dev, Predicate(4, P.PRED_LESS_THAN, 100))
    try:
        cases = [
            ((None, side(probe_dev)), P.HYB_ERR_INVALID),                             # NULL argument
            ((side(build_dev), None), P.HYB_ERR_INVALID),
            ((P.JoinSide(987_654, 0, 0), side(probe_dev)), P.HYB_ERR_NOT_FOUND),      # unknown table
            ((side(build_dev), P.JoinSide(987_654, 0, 0)), P.HYB_ERR_NOT_FOUND),
            ((side(build_dev, 5), side(probe_dev)), P.HYB_ERR_INVALID),               # key column out of range
            ((side(build_dev), side(probe_dev, 9)), P.HYB_ERR_INVALID),
            ((side(build_dev, 2), side(probe_dev, 2)), P.HYB_ERR_UNSUPPORTED),        # float keys
            ((side(build_dev, 3), side(probe_dev)), P.HYB_ERR_UNSUPPORTED),
            ((side(strings_dev), side(probe_dev)), P.HYB_ERR_UNSUPPORTED),            # string key
            ((side(build_dev), side(probe_dev, 0, 987_654)), P.HYB_ERR_NOT_FOUND),    # unknown filter
            ((side(build_dev), side(probe_dev, 0, scan.handle)), P.HYB_ERR_INVALID),  # filter of another table
        ]
        for (build_side, probe_side), status in cases:
            assert join_status(device, build_side, probe_side) == status, (build_side, probe_side)
            good_join(device, reject_tables)
        assert join_status(device, side(build_dev), side(probe_dev), radix_bits=9) == P.HYB_ERR_INVALID
        good_join(device, reject_tables)
        assert join_status(device, side(build_dev), side(probe_dev), mode=99) == P.HYB_ERR_UNSUPPORTED
        good_join(device, reject_tables)
        out = C.c_uint64()
        assert device.lib.hyb_join_hash(None, C.byref(side(build_dev)), C.byref(side(probe_dev)), P.JOIN_INNER, 2,
                                        C.byref(out)) == P.HYB_ERR_INVALID
        assert device.lib.hyb_join_hash(device.ptr, C.byref(side(build_dev)), C.byref(side(probe_dev)), P.JOIN_INNER, 2,
                                        None) == P.HYB_ERR_INVALID
        good_join(device, reject_tables)
    finally:
        scan.free()


def test_partition_rejections(device, reject_tables):
    import torch

    _, (build_dev, _, strings_dev) = reject_tables
    side = P.JoinSide(build_dev.handle, 0, 0)
    positions = side_positions(device, side)
    keys = torch.zeros(positions, dtype=torch.int64, device="cuda")
    row_ids = torch.zeros(positions, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    lib = device.lib
    for partition_count in (3, 512, 0):
        offsets = (C.c_uint64 * 513)()
        assert lib.hyb_join_partition(device.ptr, C.byref(side), partition_count, 0, keys.data_ptr(), row_ids.data_ptr(),
                                      offsets) == P.HYB_ERR_INVALID
        good_join(device, reject_tables)
    offsets = (C.c_uint64 * 3)()
    assert lib.hyb_join_partition(device.ptr, C.byref(side), 2, 0, None, None, offsets) == P.HYB_ERR_INVALID
    assert lib.hyb_join_partition(device.ptr, C.byref(side), 2, 0, keys.data_ptr(), row_ids.data_ptr(),
                                  None) == P.HYB_ERR_INVALID
    strings_side = P.JoinSide(strings_dev.handle, 0, 0)
    assert lib.hyb_join_partition(device.ptr, C.byref(strings_side), 2, 0, keys.data_ptr(), row_ids.data_ptr(),
                                  offsets) == P.HYB_ERR_UNSUPPORTED
    good_join(device, reject_tables)

    destinations = {}

    def exchange_with(result, leave_null):
        def exchange(_user, counts, dest_keys, dest_rows):
            for p in range(2):
                destinations[p] = (torch.zeros(int(counts[p]) + 1, dtype=torch.int64, device="cuda"),
                                   torch.zeros(int(counts[p]) + 1, dtype=torch.int64, device="cuda"))
                dest_keys[p], dest_rows[p] = destinations[p][0].data_ptr(), destinations[p][1].data_ptr()
            if leave_null:
                dest_rows[1] = None
            torch.cuda.synchronize()
            return result
        return P.EXCHANGE_FN(exchange)

    never_called = exchange_with(0, False)
    assert lib.hyb_join_partition_push(device.ptr, C.byref(side), 32, 0, never_called, None) == P.HYB_ERR_INVALID
    assert lib.hyb_join_partition_push(device.ptr, C.byref(side), 2, 0, None, None) == P.HYB_ERR_INVALID
    good_join(device, reject_tables)
    # the exchange callback fails, or leaves the destination of a non-empty group NULL: the call's scratch is released
    for callback in (exchange_with(1, False), exchange_with(0, True)):
        for _ in range(3):
            assert lib.hyb_join_partition_push(device.ptr, C.byref(side), 2, 0, callback, None) == P.HYB_ERR_INVALID
            good_join(device, reject_tables)
    good = exchange_with(0, False)
    P.check(lib.hyb_join_partition_push(device.ptr, C.byref(side), 2, 0, good, None))
    assert sum(len(destinations[p][0]) - 1 for p in range(2)) == len(
        [key for _, key in rows_with_keys(reject_tables[0][0], 0) if key is not None])


# ---- distributed, world of one ---------------------------------------------------------------------------------------
def test_distributed_default_radix_bits(device, reject_tables):
    """radix_bits = -1 on both distributed paths (the exchange and the co-located shortcut) takes JoinHash's rule."""
    from hyrise_b200 import distributed as hd

    (build, probe), (build_dev, probe_dev, _) = reject_tables
    status = device.lib.hyb_join_hash_distributed(device.ptr, 987_654, C.byref(P.JoinSide(build_dev.handle, 4, 0)),
                                                  C.byref(P.JoinSide(probe_dev.handle, 4, 0)), 0, 0, -1,
                                                  C.byref(C.c_uint64()))
    assert status == P.HYB_ERR_NOT_FOUND
    good_join(device, reject_tables)
    group = hd.connect_peer_group(device, 4 * (build.row_count + probe.row_count) + 4096)
    try:
        expected = orc.join_hash(build, 4, probe, 4, P.JOIN_INNER, -1)
        for colocated in ("0", "1"):
            device.set_option("join_colocated", colocated)
            result = group.join_hash(build_dev, 4, probe_dev, 4, 0, 0, -1)
            try:
                assert result.info()[2] == expected.radix_bits
                assert np.array_equal(result.partition_offsets(), expected.partition_offsets)
                got_build, got_probe = result.to_host()
                assert row_ids_equal(got_probe, expected.probe) and row_ids_equal(got_build, expected.build)
            finally:
                result.free()
            assert group.stats().colocated == int(colocated)
    finally:
        device.set_option("join_colocated", "1")
        group.destroy()
    good_join(device, reject_tables)
