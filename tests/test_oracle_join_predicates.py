"""Pins orc_join_hash_predicates (the C++ restatement of JoinHash with secondary predicates, join_predicates_oracle.ordered)
to JoinVerification semantics with predicates (join_predicates_oracle.nested_loop, numpy comparisons) on the
join_test_runner inputs and on every numeric type pairing with special values. CPU only."""
import ctypes as C

import numpy as np
import pytest

import join_predicates_oracle as jpo
import oracle_lib as orc
from helpers import row_ids_equal, tbl
from hyrise_b200 import capi
from hyrise_b200.storage import NUMPY_TYPES, ColumnDefinition, Table

MODES = [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_SEMI, capi.JOIN_ANTI_NULL_AS_FALSE]

# join_test_runner.cpp:207-211: secondary predicates on column 0 vs column 0 (l_int / r_int); l_int, l_int_null, l_long,
# l_long_null are columns 0, 1, 6, 7 and l_float, l_double 2, 4
PREDICATE_SETS = {
    "none": [],
    "lt": [(0, 0, capi.PRED_LESS_THAN)],
    "ge": [(0, 0, capi.PRED_GREATER_THAN_EQUALS)],
    "ne": [(0, 0, capi.PRED_NOT_EQUALS)],
    "int_long": [(1, 6, capi.PRED_LESS_THAN_EQUALS), (7, 0, capi.PRED_NOT_EQUALS)],
    "float_double": [(2, 4, capi.PRED_GREATER_THAN), (3, 1, capi.PRED_NOT_EQUALS)],
}
KEY_COLUMN_PAIRS = [(0, 0), (1, 1), (0, 1), (6, 6), (7, 7), (0, 6), (7, 1)]  # test_oracle_join.int_column_pairs


def sides(left, right, mode, left_column, right_column, predicates, swap):
    """(build, build column, probe, probe column, predicates): JoinHash::_on_execute's choice (join_hash.cpp:139-165) —
    the smaller side builds an Inner join — or, with `swap`, the other order, the predicates flipped."""
    left_builds = mode == capi.JOIN_INNER and left.row_count <= right.row_count
    if swap:
        left_builds = not left_builds
    if left_builds:
        return left, left_column, right, right_column, predicates
    return right, right_column, left, left_column, jpo.flip(predicates)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("radix_bits", [0, 1, 2, 5])
@pytest.mark.parametrize("sizes", [(10, 15), (15, 10), (0, 10), (10, 0), (0, 0), (15, 15)])
@pytest.mark.parametrize("chunk_size", [10, 3, 1])
def test_join_test_runner_inputs(mode, radix_bits, sizes, chunk_size):
    left = tbl(f"join_test_runner/input_table_left_{sizes[0]}.tbl", chunk_size)
    right = tbl(f"join_test_runner/input_table_right_{sizes[1]}.tbl", chunk_size)
    for left_column, right_column in KEY_COLUMN_PAIRS:
        for swap in (False, True):
            if swap and mode != capi.JOIN_INNER:
                continue  # the probe side is the preserved / filtered side of every other mode
            for predicate_set, predicates in PREDICATE_SETS.items():
                build, build_column, probe, probe_column, oriented = sides(left, right, mode, left_column, right_column,
                                                                           predicates, swap)
                result = jpo.ordered(build, build_column, probe, probe_column, mode, radix_bits, oriented)
                want = jpo.nested_loop(build, build_column, probe, probe_column, mode, oriented)
                got = jpo.result_rows(result)
                context = (mode, radix_bits, sizes, chunk_size, predicate_set, left_column, right_column, swap)
                assert sorted(got) == sorted(want), context
                assert result.partition_offsets[-1] == len(got), context
                assert len(result.partition_offsets) == (1 << radix_bits) + 1, context


@pytest.mark.parametrize("predicate_set", ["lt", "ge", "ne", "int_long", "float_double"])
def test_flip_rule(predicate_set):
    # an Inner join and its swap with flipped predicates (join_hash.cpp:158-165) emit the same pairs
    left = tbl("join_test_runner/input_table_left_15.tbl", 3)
    right = tbl("join_test_runner/input_table_right_15.tbl", 3)
    predicates = PREDICATE_SETS[predicate_set]
    for left_column, right_column in KEY_COLUMN_PAIRS:
        one = jpo.ordered(left, left_column, right, right_column, capi.JOIN_INNER, 2, predicates)
        other = jpo.ordered(right, right_column, left, left_column, capi.JOIN_INNER, 2, jpo.flip(predicates))
        assert sorted(jpo.result_rows(one)) == sorted((p, b) for b, p in jpo.result_rows(other))
        assert len(jpo.result_rows(one)) == len(jpo.nested_loop(left, left_column, right, right_column,
                                                                 capi.JOIN_INNER, predicates))


def test_flip_matches_the_library():
    # the restatement flips conditions as hyb_flip_predicate_condition (flip_predicate_condition, types.cpp:51-82) does
    out = C.c_int32()
    for condition, flipped in jpo.FLIPPED.items():
        capi.check(capi.load_library().hyb_flip_predicate_condition(condition, C.byref(out)))
        assert out.value == flipped


@pytest.mark.parametrize("mode", MODES)
def test_always_true_predicate_keeps_the_plain_join(mode):
    # `k = k` on the key columns themselves holds for every candidate: the result is hyb_join_hash's, in its order
    left = tbl("join_test_runner/input_table_left_15.tbl", 3)
    right = tbl("join_test_runner/input_table_right_15.tbl", 1)
    for radix_bits in (0, 1, 5):
        plain = orc.join_hash(right, 6, left, 0, mode, radix_bits)
        derived = jpo.ordered(right, 6, left, 0, mode, radix_bits, [(6, 0, capi.PRED_EQUALS)])
        assert row_ids_equal(derived.probe, plain.probe)
        assert (derived.partition_offsets == plain.partition_offsets).all()
        if plain.build is not None:
            assert row_ids_equal(derived.build, plain.build)


SPECIAL = {
    capi.TYPE_INT32: [np.iinfo(np.int32).min, np.iinfo(np.int32).max, 0, -1, 16777217, 7],
    capi.TYPE_INT64: [np.iinfo(np.int64).min, np.iinfo(np.int64).max, 0, -1, 2 ** 53 + 1, 7],
    capi.TYPE_FLOAT32: [np.nan, np.inf, -np.inf, -0.0, 0.0, 16777216.0],
    capi.TYPE_FLOAT64: [np.nan, np.inf, -np.inf, -0.0, 0.0, 9007199254740992.0],
}
TYPES = list(SPECIAL)


def typed_table(rng, rows, key_high, chunk_size):
    definitions = [ColumnDefinition("k", capi.TYPE_INT32)] + [ColumnDefinition(f"c{t}", t, True) for t in TYPES]
    columns = [rng.integers(0, key_high, rows).astype(np.int32)]
    nulls = [None]
    for data_type in TYPES:
        dtype = np.dtype(NUMPY_TYPES[data_type])
        pool = np.array(SPECIAL[data_type], dtype=dtype)
        columns.append(np.where(rng.random(rows) < 0.5, pool[rng.integers(0, len(pool), rows)],
                                rng.integers(-3, 8, rows).astype(dtype)).astype(dtype))
        nulls.append(rng.random(rows) < 0.1)
    return Table.from_columns(definitions, columns, nulls, chunk_size).encode(["Unencoded", "Dictionary", "Dictionary",
                                                                               "Unencoded", "Dictionary"])


@pytest.mark.parametrize("mode", MODES)
def test_type_pairings(mode):
    # the C++ evaluator's std functors on the columns' own types against numpy's casts to the common type
    rng = np.random.default_rng(mode)
    build, probe = typed_table(rng, 300, 60, 70), typed_table(rng, 400, 70, 90)
    for build_type in TYPES:
        for probe_type in TYPES:
            for condition in jpo.FLIPPED:
                predicates = [(1 + TYPES.index(build_type), 1 + TYPES.index(probe_type), condition)]
                result = jpo.ordered(build, 0, probe, 0, mode, 2, predicates)
                want = jpo.nested_loop(build, 0, probe, 0, mode, predicates)
                assert sorted(jpo.result_rows(result)) == sorted(want), (build_type, probe_type, condition)


def test_filters_with_null_row_ids():
    # a LEFT join's side as the filter of either side: NULL_ROW_IDs are NULL keys and never pass a predicate
    rng = np.random.default_rng(9)
    table, other = typed_table(rng, 300, 40, 64), typed_table(rng, 200, 120, 50)
    left = orc.join_hash(table, 0, other, 0, capi.JOIN_LEFT, 0)
    rows = left.build
    assert (rows["chunk_id"] == jpo.INVALID_CHUNK_ID).any()
    joined = orc.HostPosList(rows, np.array([0] + [len(rows)] * table.chunk_count, dtype=np.uint64), multiple_chunks=True)
    predicates = [(3, 4, capi.PRED_LESS_THAN), (1, 2, capi.PRED_NOT_EQUALS)]
    for mode in MODES:
        for build_filter, probe_filter in ((joined, None), (None, joined)):
            result = jpo.ordered(table, 0, table, 0, mode, 3, predicates, build_filter=build_filter,
                                 probe_filter=probe_filter)
            want = jpo.nested_loop(table, 0, table, 0, mode, predicates, build_filter=build_filter,
                                   probe_filter=probe_filter)
            assert sorted(jpo.result_rows(result)) == sorted(want), mode


def test_rejections():
    table = tbl("join_test_runner/input_table_left_10.tbl", 3)  # column 8: string
    for mode, predicates, status in ((capi.JOIN_ANTI_NULL_AS_TRUE, [(0, 0, capi.PRED_LESS_THAN)], capi.HYB_ERR_UNSUPPORTED),
                                     (capi.JOIN_INNER, [(8, 8, capi.PRED_EQUALS)], capi.HYB_ERR_UNSUPPORTED),
                                     (capi.JOIN_INNER, [(8, 0, capi.PRED_EQUALS)], capi.HYB_ERR_INVALID)):
        with pytest.raises(capi.HyriseB200Error) as error:
            jpo.ordered(table, 0, table, 0, mode, 0, predicates)
        assert error.value.status == status
