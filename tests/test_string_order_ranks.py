"""Order ranks of string columns (hyb_dictionary_order_ranks, hyb_binary_table_string_order_ranks and the Python
restatement storage.dictionary_order_ranks) against sorted(set(...)) of Python bytes, which compare unsigned and put a
proper prefix first, as char_traits<char>::compare does."""
import ctypes as C
import glob
import os
import random

import pytest

from hyrise_b200 import capi
from hyrise_b200.binary_table import NativeBinaryTable
from hyrise_b200.storage import dictionary_order_ranks

BIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bin")

# the StringVariations strings of the reference's binary writer tests, plus high bytes and prefixes
VARIATIONS = [b"", b"\0", b"\0\0", b"\0\0\0", b"\0\0\0\0", b"\0\0\0\0\0", b"a\0b", b"a", b"ab", b"abc", b"a\0", b"\xff",
              b"\xff\xff", b"\x7f", b"\x80", b"b", b"A", b"\xfe\xff"]


def expected_ranks(dictionaries):
    distinct = sorted({entry for dictionary in dictionaries for entry in dictionary})
    rank = {value: index for index, value in enumerate(distinct)}
    return [rank[entry] for dictionary in dictionaries for entry in dictionary], len(distinct)


def check(dictionaries):
    want, distinct = expected_ranks(dictionaries)
    got, got_distinct = capi.dictionary_order_ranks(dictionaries)
    assert got.tolist() == want and got_distinct == distinct
    assert dictionary_order_ranks(dictionaries).tolist() == want


def test_string_variations():
    everything = sorted(set(VARIATIONS))
    check([everything])
    check([everything[::2], everything[1::2], everything, []])
    check([[entry] for entry in reversed(everything)])


@pytest.mark.parametrize("seed", range(8))
def test_random_dictionaries(seed):
    rng = random.Random(seed)
    alphabet = [b"\0", b"a", b"b", b"\x80", b"\xff"]
    universe = sorted({b"".join(rng.choice(alphabet) for _ in range(rng.randrange(0, 5))) for _ in range(200)})
    dictionaries = []
    for chunk in range(rng.randrange(1, 12)):
        kind = rng.randrange(3)
        if kind == 0:  # disjoint slice
            begin = rng.randrange(len(universe))
            dictionaries.append(universe[begin:begin + rng.randrange(0, 20)])
        elif kind == 1:  # full overlap
            dictionaries.append(list(universe))
        else:  # random subset
            dictionaries.append(sorted(rng.sample(universe, rng.randrange(0, len(universe)))))
    check(dictionaries)


def test_no_dictionaries():
    check([])
    check([[], []])


def test_not_strictly_increasing():
    for bad in ([b"b", b"a"], [b"a", b"a"]):
        with pytest.raises(capi.HyriseB200Error) as error:
            capi.dictionary_order_ranks([[b"x"], bad])
        assert error.value.status == capi.HYB_ERR_INVALID


def raw_dictionary(table: NativeBinaryTable, chunk: int, column: int) -> list[bytes]:
    """The entries as stored (numpy's 'S' arrays would drop trailing NUL bytes)."""
    chars, offsets, count = C.c_void_p(), C.POINTER(C.c_uint64)(), C.c_uint32()
    capi.check(table.lib.hyb_binary_table_string_dictionary(table.ptr, chunk, column, C.byref(chars), C.byref(offsets),
                                                            C.byref(count)))
    blob = C.string_at(chars, offsets[count.value]) if count.value and chars.value else b""
    return [blob[offsets[i]:offsets[i + 1]] for i in range(count.value)]


def test_binary_fixtures():
    checked = 0
    for path in sorted(glob.glob(os.path.join(BIN, "**", "*.bin"), recursive=True)):
        try:
            table = NativeBinaryTable(path)
        except capi.HyriseB200Error:
            continue  # the invalid and LZ4 fixtures
        for column, definition in enumerate(table.table.column_definitions):
            if definition.data_type != capi.TYPE_STRING:
                continue
            dictionaries = [raw_dictionary(table, chunk, column) for chunk in range(table.table.chunk_count)]
            want, _ = expected_ranks(dictionaries)
            assert table.string_order_ranks(column).tolist() == want, (path, column)
            assert capi.dictionary_order_ranks(dictionaries)[0].tolist() == want
            checked += 1
    assert checked > 0
