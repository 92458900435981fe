"""The five TableScan entry points (hyb_table_scan, _columns, _in, _expression, _expression_tests) end in one host driver.
For each of them: the operator stats under every unfiltered pipeline and every kind of input filter, empty tables and the
empty lists they produce fed back into every operator, and the codes for unknown and foreign input filters."""
import numpy as np
import pytest

from hyrise_b200 import capi
from hyrise_b200.device import Aggregate, ColumnComparison, DevicePosList, InList, Predicate, ScanExpression
from hyrise_b200.storage import ColumnDefinition, Table
from test_oracle_expression_scan import col, lit

pytestmark = pytest.mark.gpu
P = capi
leaf, scan, in_list = ScanExpression.leaf, ScanExpression.scan, ScanExpression.in_list

DEFINITIONS = [ColumnDefinition("a", P.TYPE_INT32, nullable=True), ColumnDefinition("b", P.TYPE_INT32),
               ColumnDefinition("c", P.TYPE_FLOAT64, nullable=True)]
CHUNK_ENCODINGS = [["Unencoded", "Dictionary", "Dictionary"], ["FrameOfReference", "Unencoded", "Unencoded"],
                   ["Dictionary", "Dictionary", "Unencoded"], ["Unencoded", "Unencoded", "Dictionary"]]
TEST_LEAF_LAUNCHES = 2  # the tree below: one scan_prepare_kernel and one in_prepare_kernel

# name -> (call, kernel launches before the scan's own, stats.path)
ENTRY_POINTS = {
    "scan": (lambda device, table, source: device.table_scan(table, Predicate(1, P.PRED_LESS_THAN, 300), source), 1, 0),
    "columns": (lambda device, table, source: device.table_scan_columns(table, ColumnComparison(0, P.PRED_LESS_THAN, 1),
                                                                       source), 1, 0),
    "in": (lambda device, table, source: device.table_scan_in(table, InList(0, P.PRED_NOT_IN, [3, 17, 250]), source), 1, 0),
    "expression": (lambda device, table, source: device.table_scan_expression(
        table, leaf(P.PRED_GREATER_THAN, col(0) + col(2) + ["+"], lit(400.5)) | leaf(P.PRED_IS_NULL, col(0)), source), 1, 0),
    "expression_tests": (lambda device, table, source: device.table_scan_expression_tests(
        table, (scan(Predicate(1, P.PRED_LESS_THAN, 600)) & in_list(InList(0, P.PRED_IN, [5, 9, 700])))
        | leaf(P.PRED_LESS_THAN, col(2), lit(-50.0)), source), TEST_LEAF_LAUNCHES, 2),
}
# the uploaded lists and programs count in algorithmic_bytes; hyb_table_scan and a numeric column pair upload none
UPLOADS = {"scan": False, "columns": False, "in": True, "expression": True, "expression_tests": True}
COLUMNS_READ = {"scan": [1], "columns": [0, 1], "in": [0], "expression": [0, 2], "expression_tests": [0, 1, 2]}
PIPELINES = {"two-pass": ("1", "0"), "single-pass": ("0", "0"), "bulk": ("0", "1")}


def mixed_table(rng, chunk_rows):
    """Columns a (int32, NULLs), b (int32, no NULLs: the bulk kernel applies) and c (float64, NULLs); every chunk its own
    encodings. A chunk of 0 rows is an empty chunk."""
    table = Table(list(DEFINITIONS))
    table._raw = []
    for rows in chunk_rows:
        a = rng.integers(0, 1000, rows).astype(np.int32)
        b = rng.integers(0, 1000, rows).astype(np.int32)
        c = rng.uniform(-100.0, 1000.0, rows)
        table._raw.append([(a, rng.random(rows) < 0.1), (b, None), (c, rng.random(rows) < 0.1)])
    table.encode("Unencoded")
    for chunk_id in range(len(chunk_rows)):
        table.encode(CHUNK_ENCODINGS[chunk_id % len(CHUNK_ENCODINGS)], [chunk_id])
    return table


def column_bytes(table, column_id):
    """What one unfiltered pass reads of a column: values or value-IDs, FrameOfReference block minima, NULL flags."""
    total = 0
    for chunk in table.chunks:
        segment = chunk.segments[column_id]
        if segment.encoding == P.ENC_UNENCODED:
            total += segment.values.itemsize * segment.row_count
        else:
            total += segment.attribute_vector.nbytes
            if segment.encoding == P.ENC_FRAME_OF_REFERENCE:
                total += 4 * ((segment.row_count + P.FOR_BLOCK_SIZE - 1) // P.FOR_BLOCK_SIZE)
        if segment.nulls is not None:
            total += segment.row_count
    return total


@pytest.fixture(scope="module")
def tables(device):
    rng = np.random.default_rng(71)
    table = mixed_table(rng, [3000, 1, 0, 17_000, 2048, 999])
    other = Table.from_columns([ColumnDefinition("k", P.TYPE_INT32)], [np.arange(0, 1400, 2, dtype=np.int32)],
                               chunk_size=300).encode("Dictionary")
    device_table, device_other = device.upload(table), device.upload(other)
    yield table, device_table, other, device_other
    device_table.drop()
    device_other.drop()
    device.set_option("scan_two_pass", "1")
    device.set_option("scan_bulk", "0")


def check_stats(device, name, result, launches, input_rows, column_read_bytes, prepared):
    """kernel_launches, path, input_rows and output_rows as given; algorithmic_bytes = the uploads (`prepared`, None: not
    known here, returned for the caller to compare) + the input read + one RowID per output row."""
    stats = device.last_stats()
    output_rows = result.info()[0]
    assert (stats.kernel_launches, stats.path, stats.input_rows, stats.output_rows) == \
        (launches, ENTRY_POINTS[name][2], input_rows, output_rows)
    uploaded = stats.algorithmic_bytes - column_read_bytes - 8 * output_rows
    if prepared is not None:
        assert uploaded == prepared
    assert (uploaded > 0) == UPLOADS[name]
    return uploaded


@pytest.mark.parametrize("name", list(ENTRY_POINTS))
def test_stats(device, tables, name):
    table, device_table, other, device_other = tables
    call, prepare_launches, _ = ENTRY_POINTS[name]
    read = sum(column_bytes(table, column_id) for column_id in COLUMNS_READ[name])
    prepared = None
    for pipeline, (two_pass, bulk) in PIPELINES.items():
        device.set_option("scan_two_pass", two_pass)
        device.set_option("scan_bulk", bulk)
        result = call(device, device_table, None)
        own = 3 if name != "scan" or pipeline == "two-pass" else 1
        prepared = check_stats(device, name, result, prepare_launches + own, table.row_count, read, prepared)
        result.free()
    device.set_option("scan_two_pass", "1")
    device.set_option("scan_bulk", "0")

    ascending = device.table_scan(device_table, Predicate(0, P.PRED_IS_NOT_NULL))
    inner = device.join_hash(device_table, 1, device_other, 0, P.JOIN_INNER, -1)
    left = device.join_hash(device_table, 1, device_other, 0, P.JOIN_LEFT, -1)
    unordered, with_null_rows = inner.pos_list(0), left.pos_list(0)
    assert (left.to_host()[0]["chunk_id"] == 0xFFFFFFFF).any()
    for source in (ascending, unordered, with_null_rows):
        rows = source.info()[0]
        result = call(device, device_table, source)
        check_stats(device, name, result, prepare_launches + 2 + (name == "expression_tests"), rows, 8 * rows, prepared)
        result.free()
    for handle in (ascending, unordered, with_null_rows, inner, left):
        handle.free()


EMPTY_TABLES = {"no chunks": [], "empty chunks": [0, 0, 0]}
# a table without chunks has no segment to type an IN list's elements by: those calls answer HYB_ERR_INVALID
TYPES_IN_LISTS = {"in", "expression_tests"}


@pytest.fixture(params=list(EMPTY_TABLES))
def empty_table(device, request):
    table = mixed_table(np.random.default_rng(72), EMPTY_TABLES[request.param])
    device_table = device.upload(table)
    yield table, device_table
    device_table.drop()


def accepts(table, name):
    return table.chunk_count > 0 or name not in TYPES_IN_LISTS


@pytest.mark.parametrize("name", list(ENTRY_POINTS))
def test_empty_tables(device, tables, empty_table, name):
    device_other = tables[3]
    table, device_table = empty_table
    if not accepts(table, name):
        pytest.skip("IN lists are typed by the column's segments")
    call, prepare_launches, _ = ENTRY_POINTS[name]
    listed = call(device, device_table, None)
    assert listed.info() == (0, table.chunk_count)
    check_stats(device, name, listed, prepare_launches, 0, 0, None)
    for other_name, (other_call, _, _) in ENTRY_POINTS.items():
        if not accepts(table, other_name):
            continue
        again = other_call(device, device_table, listed)
        assert again.info()[0] == 0
        again.free()
    assert device.aggregate_hash(device_table, [1], [Aggregate(P.AGG_COUNT_STAR)], input_filter=listed).group_count == 0
    join = device.join_hash(device_other, 0, device_table, 1, P.JOIN_INNER, -1, probe_filter=listed)
    assert join.info()[0] == 0
    join.free()
    listed.free()


@pytest.mark.parametrize("name", list(ENTRY_POINTS))
def test_sort_of_an_empty_scan(device, empty_table, name):
    # an unfiltered scan of a table without rows launches no tile: the list's total is the "unset" fill, which is 0 rows
    table, device_table = empty_table
    if not accepts(table, name):
        pytest.skip("IN lists are typed by the column's segments")
    listed = ENTRY_POINTS[name][0](device, device_table, None)
    ordered = device.sort(device_table, [(1, False)], listed)
    assert ordered.info() == (0, 1)
    assert device.last_stats().input_rows == 0
    ordered.free()
    listed.free()


@pytest.mark.parametrize("name", list(ENTRY_POINTS))
def test_unknown_and_foreign_filters(device, tables, name):
    _, device_table, _, device_other = tables
    call = ENTRY_POINTS[name][0]
    with pytest.raises(capi.HyriseB200Error) as error:
        call(device, device_table, DevicePosList(device, 0x7FFF_FFFF))
    assert error.value.status == capi.HYB_ERR_NOT_FOUND
    foreign = device.table_scan(device_other, Predicate(0, P.PRED_LESS_THAN, 100))
    with pytest.raises(capi.HyriseB200Error) as error:
        call(device, device_table, foreign)
    assert error.value.status == capi.HYB_ERR_INVALID
    foreign.free()
