"""Hyrise's binary table format (SURVEY.md §8 f4: the loading path) -> host segments in the layout the device pool uploads.

Follows `import_export/binary/binary_parser.cpp:40-330` / `binary_writer.cpp` (format tables in `binary_writer.hpp:25-230`;
note that the header stores the column TYPES as strings and every string length as a `size_t`, `binary_parser.cpp:106-111`):

    header   chunk size u32 | chunk count u32 | column count u16 | type names | nullable flags (1 byte each) | column names
    chunk    row count u32 | sorted-column count u32 | {column id u16, sort mode u8} ... | one segment per column
    segment  encoding type u8 (`storage/encoding_type.hpp:26`: Unencoded, Dictionary, RunLength, FixedStringDictionary,
             FrameOfReference, LZ4) + the encoding's payload

What is read stays in the reference's encoding wherever the device path reads that encoding (ValueSegment,
DictionarySegment, FrameOfReferenceSegment with FixedWidthInteger or BitPacking vectors): the buffers are copied once, into
256-byte aligned slots of a few large host blocks (pinned when a DeviceContext provides the memory), so that
`DeviceContext.upload_blocks` + `upload_from_blocks` move a table with one DMA per block. RunLengthSegments are expanded to
ValueSegments and FixedStringDictionarySegments become string DictionarySegments (both stay exact); LZ4 segments raise
UnsupportedOnDevice — the reference's default benchmark encoding does not produce them.
"""
from __future__ import annotations

import os
import struct
from dataclasses import dataclass, field

import numpy as np

from . import capi
from .storage import (NUMPY_TYPES, Chunk, ColumnDefinition, Segment, StringKeyRegistry, Table, compress_fixed_width,
                      make_value_segment)

ENCODING_UNENCODED, ENCODING_DICTIONARY, ENCODING_RUN_LENGTH, ENCODING_FIXED_STRING, ENCODING_FOR, ENCODING_LZ4 = range(6)
# storage/vector_compression/compressed_vector_type.hpp:28-33
VECTOR_BITPACKING, VECTOR_FIXED_1B, VECTOR_FIXED_2B, VECTOR_FIXED_4B = range(4)
TYPE_NAMES = {"int": capi.TYPE_INT32, "long": capi.TYPE_INT64, "float": capi.TYPE_FLOAT32, "double": capi.TYPE_FLOAT64,
              "string": capi.TYPE_STRING}
NAME_OF_TYPE = {value: key for key, value in TYPE_NAMES.items()}
BLOCK_BYTES = 64 << 20
ALIGN = 256
TAIL_PAD = 64   # kernels may read one 16-byte vector past the last element


class BinaryFormatError(ValueError):
    """What the reference reports with Fail() (std::logic_error): invalid encoding type, invalid vector type, truncated file."""


class HostArena:
    """Large host blocks with 256-byte aligned slots; `allocate` = hyb_host_alloc-backed numpy arrays when a context is given."""

    def __init__(self, context=None, block_bytes: int = BLOCK_BYTES):
        self.context = context
        self.block_bytes = block_bytes
        self.blocks: list[np.ndarray] = []
        self.used: list[int] = []

    def _new_block(self, size: int) -> None:
        size = max(size + ALIGN, self.block_bytes)
        block = self.context.pinned_empty(size, np.uint8) if self.context is not None else np.empty(size, dtype=np.uint8)
        self.blocks.append(block)
        self.used.append((-block.ctypes.data) % ALIGN)   # numpy's own allocations are not 256-byte aligned

    def place(self, array: np.ndarray) -> np.ndarray:
        """Copies `array` into the arena; returns the aligned view that replaces it."""
        array = np.ascontiguousarray(array)
        need = (array.nbytes + TAIL_PAD + ALIGN - 1) // ALIGN * ALIGN
        if not self.blocks or self.used[-1] + need > len(self.blocks[-1]):
            self._new_block(need)
        start = self.used[-1]
        self.used[-1] += need
        slot = self.blocks[-1][start:start + array.nbytes].view(array.dtype) if array.nbytes else np.zeros(0, dtype=array.dtype)
        if array.nbytes:
            slot[...] = array.reshape(-1)
        return slot

    def host_blocks(self) -> list:
        return [capi.HostBlock(block.ctypes.data, used) for block, used in zip(self.blocks, self.used) if used]


@dataclass
class BinaryTable:
    """A parsed file: the table plus what the format carries beyond segments."""
    table: Table
    arena: HostArena
    sorted_columns: list[list[tuple[int, int]]] = field(default_factory=list)   # per chunk: (column id, SortMode)

    def host_blocks(self) -> list:
        return self.arena.host_blocks()


class _Reader:
    def __init__(self, data: bytes):
        self.data = memoryview(data)
        self.position = 0

    def take(self, count: int) -> memoryview:
        if self.position + count > len(self.data):
            raise BinaryFormatError("unexpected end of file")
        view = self.data[self.position:self.position + count]
        self.position += count
        return view

    def value(self, fmt: str):
        return struct.unpack("<" + fmt, self.take(struct.calcsize("<" + fmt)))[0]

    def array(self, dtype, count: int) -> np.ndarray:
        dtype = np.dtype(dtype)
        return np.frombuffer(self.take(dtype.itemsize * count), dtype=dtype, count=count)

    def strings(self, count: int) -> list[bytes]:
        lengths = self.array(np.uint64, count)   # size_t per string, binary_parser.cpp:83-96
        buffer = bytes(self.take(int(lengths.sum())))
        out, start = [], 0
        for length in lengths:
            out.append(buffer[start:start + int(length)])
            start += int(length)
        return out

    def bools(self, count: int) -> np.ndarray:
        return self.array(np.uint8, count) != 0

    def compressed_vector(self, vector_type: int, count: int):
        """-> (raw vector as the reference stores it, hyb vector type, bit width)."""
        if vector_type == VECTOR_BITPACKING:
            bits = self.value("B")
            words = (count * bits + 63) // 64   # compact::vector::bytes(): whole 64-bit words
            return self.array(np.uint64, words), capi.VEC_BITPACKED, bits
        if vector_type == VECTOR_FIXED_1B:
            return self.array(np.uint8, count), capi.VEC_FIXED_1B, 0
        if vector_type == VECTOR_FIXED_2B:
            return self.array(np.uint16, count), capi.VEC_FIXED_2B, 0
        if vector_type == VECTOR_FIXED_4B:
            return self.array(np.uint32, count), capi.VEC_FIXED_4B, 0
        raise BinaryFormatError(f"cannot import attribute vector with compressed vector type id {vector_type}")


def _string_array(values: list[bytes]) -> np.ndarray:
    width = max((len(value) for value in values), default=1) or 1
    return np.array(values, dtype=f"S{width}")


def _read_segment(reader: _Reader, rows: int, definition: ColumnDefinition, arena: HostArena,
                  string_keys: StringKeyRegistry) -> Segment:
    data_type = definition.data_type
    is_string = data_type == capi.TYPE_STRING
    encoding = reader.value("B")
    if encoding == ENCODING_UNENCODED:
        nulls = None
        if definition.nullable and reader.value("B"):   # "segment nullable" is only written for nullable columns
            nulls = reader.bools(rows)
        if is_string:
            values = _string_array(reader.strings(rows))
            return _dictionary_from_values(values, nulls, data_type, arena, string_keys)   # strings reach the device as value-IDs
        values = reader.array(NUMPY_TYPES[data_type], rows)
        segment = make_value_segment(values, nulls if nulls is not None else (np.zeros(rows, bool) if definition.nullable else None),
                                     data_type)
        segment.values = arena.place(segment.values)
        if segment.nulls is not None:
            segment.nulls = arena.place(segment.nulls)
        return segment
    if encoding in (ENCODING_DICTIONARY, ENCODING_FIXED_STRING):
        vector_type = reader.value("B")
        dictionary_size = reader.value("I")
        segment = Segment(capi.ENC_DICTIONARY, data_type, rows, dictionary_size=dictionary_size)
        if encoding == ENCODING_FIXED_STRING:
            length = reader.value("I")   # FixedStringVector: string length (binary_parser.cpp:339-344), then size * length chars (NUL padded)
            chars = bytes(reader.take(dictionary_size * length))
            entries = [chars[i * length:(i + 1) * length].rstrip(b"\0") for i in range(dictionary_size)]
            segment.string_dictionary = _string_array(entries)
        elif is_string:
            segment.string_dictionary = _string_array(reader.strings(dictionary_size))
        else:
            segment.values = arena.place(reader.array(NUMPY_TYPES[data_type], dictionary_size))
        vector, segment.vector_type, segment.bit_width = reader.compressed_vector(vector_type, rows)
        segment.attribute_vector = arena.place(vector)
        if is_string:
            segment.dictionary_codes = arena.place(string_keys.codes(segment.string_dictionary))
        return segment
    if encoding == ENCODING_RUN_LENGTH:
        runs = reader.value("I")
        if is_string:
            run_values = _string_array(reader.strings(runs))
        else:
            run_values = reader.array(NUMPY_TYPES[data_type], runs)
        run_nulls = reader.bools(runs)
        ends = reader.array(np.uint32, runs).astype(np.int64)   # inclusive end position of every run
        lengths = np.diff(np.concatenate([[-1], ends]))
        values = np.repeat(run_values, lengths)
        nulls = np.repeat(run_nulls, lengths)
        if is_string:
            return _dictionary_from_values(values, nulls if nulls.any() or definition.nullable else None, data_type, arena, string_keys)
        segment = make_value_segment(values, nulls if (nulls.any() or definition.nullable) else None, data_type)
        segment.values = arena.place(segment.values)
        if segment.nulls is not None:
            segment.nulls = arena.place(segment.nulls)
        return segment
    if encoding == ENCODING_FOR:
        if data_type != capi.TYPE_INT32:
            raise BinaryFormatError("unsupported data type for FrameOfReference encoding")
        vector_type = reader.value("B")
        blocks = reader.value("I")
        minima = reader.array(np.int32, blocks)
        nulls = reader.bools(rows) if reader.value("B") else None
        vector, hyb_vector_type, bits = reader.compressed_vector(vector_type, rows)
        return Segment(capi.ENC_FRAME_OF_REFERENCE, data_type, rows, values=arena.place(minima),
                       nulls=None if nulls is None else arena.place(nulls.astype(np.uint8)),
                       attribute_vector=arena.place(vector), vector_type=hyb_vector_type, bit_width=bits)
    if encoding == ENCODING_LZ4:
        raise capi.UnsupportedOnDevice(capi.HYB_ERR_UNSUPPORTED, "LZ4 segments are not read by the device path")
    raise BinaryFormatError(f"invalid EncodingType {encoding}")


def _dictionary_from_values(values: np.ndarray, nulls, data_type: int, arena: HostArena, string_keys: StringKeyRegistry) -> Segment:
    """A string column that the file stores value by value: dictionary-encoded like DictionaryEncoder would
    (sorted unique dictionary, value-ID = rank, NULL = dictionary size, dictionary_encoder.hpp:33-110)."""
    null_mask = np.zeros(len(values), dtype=bool) if nulls is None else np.asarray(nulls, dtype=bool)
    dictionary, inverse = np.unique(values[~null_mask], return_inverse=True)
    ids = np.full(len(values), len(dictionary), dtype=np.uint32)
    ids[~null_mask] = inverse.astype(np.uint32)
    vector, vector_type = compress_fixed_width(ids, len(dictionary))
    segment = Segment(capi.ENC_DICTIONARY, data_type, len(values), attribute_vector=arena.place(vector), vector_type=vector_type,
                      dictionary_size=len(dictionary))
    segment.string_dictionary = dictionary if len(dictionary) else np.zeros(0, dtype="S1")
    segment.dictionary_codes = arena.place(string_keys.codes(segment.string_dictionary))
    return segment


def read_binary_table(path: str, context=None) -> BinaryTable:
    """BinaryParser::parse. `context` (a DeviceContext): segment buffers are placed in pinned host blocks."""
    with open(path, "rb") as file:
        reader = _Reader(file.read())
    chunk_size = reader.value("I")
    chunk_count = reader.value("I")
    column_count = reader.value("H")
    type_names = [name.decode() for name in reader.strings(column_count)]
    nullable = reader.bools(column_count)
    names = [name.decode() for name in reader.strings(column_count)]
    definitions = []
    for name, type_name, is_nullable in zip(names, type_names, nullable):
        if type_name not in TYPE_NAMES:
            raise BinaryFormatError(f"unknown column type {type_name!r}")
        definitions.append(ColumnDefinition(name, TYPE_NAMES[type_name], bool(is_nullable)))
    table = Table(definitions, target_chunk_size=chunk_size)
    table._string_keys = [StringKeyRegistry() for _ in definitions]
    arena = HostArena(context)
    parsed = BinaryTable(table, arena)
    for _ in range(chunk_count):
        rows = reader.value("I")
        sorted_count = reader.value("I")
        parsed.sorted_columns.append([(reader.value("H"), reader.value("B")) for _ in range(sorted_count)])
        segments = [_read_segment(reader, rows, definition, arena, table._string_keys[column_id])
                    for column_id, definition in enumerate(definitions)]
        table.chunks.append(Chunk(segments))
    return parsed


# ---------------------------------------------------------------------------------------------------------------------
# Writer (BinaryWriter::write): the encodings the device path holds; used to hand generated tables to a Hyrise instance and
# for round-trip tests.
# ---------------------------------------------------------------------------------------------------------------------
def _write_strings(out: list, values) -> None:
    values = [bytes(value) for value in values]
    out.append(np.array([len(value) for value in values], dtype=np.uint64).tobytes())
    out.append(b"".join(values))


def _write_vector(out: list, segment: Segment) -> None:
    if segment.vector_type == capi.VEC_BITPACKED:
        out.append(struct.pack("<B", segment.bit_width))
        words = (segment.row_count * segment.bit_width + 63) // 64
        out.append(np.ascontiguousarray(segment.attribute_vector).view(np.uint64)[:words].tobytes())
    else:
        out.append(np.ascontiguousarray(segment.attribute_vector).tobytes())


def write_binary_table(table: Table, path: str) -> None:
    out: list[bytes] = [struct.pack("<IIH", table.target_chunk_size, table.chunk_count, table.column_count)]
    _write_strings(out, [NAME_OF_TYPE[d.data_type].encode() for d in table.column_definitions])
    out.append(bytes(1 if d.nullable else 0 for d in table.column_definitions))
    _write_strings(out, [d.name.encode() for d in table.column_definitions])
    vector_ids = {capi.VEC_BITPACKED: VECTOR_BITPACKING, capi.VEC_FIXED_1B: VECTOR_FIXED_1B, capi.VEC_FIXED_2B: VECTOR_FIXED_2B,
                  capi.VEC_FIXED_4B: VECTOR_FIXED_4B}
    for chunk in table.chunks:
        out.append(struct.pack("<II", chunk.size, 0))   # no sort information
        for definition, segment in zip(table.column_definitions, chunk.segments):
            if segment.encoding == capi.ENC_UNENCODED:
                out.append(struct.pack("<B", ENCODING_UNENCODED))
                if definition.nullable:
                    out.append(struct.pack("<B", 1 if segment.nulls is not None else 0))
                    if segment.nulls is not None:
                        out.append(np.ascontiguousarray(segment.nulls, dtype=np.uint8).tobytes())
                out.append(np.ascontiguousarray(segment.values).tobytes())
            elif segment.encoding == capi.ENC_DICTIONARY:
                out.append(struct.pack("<BBI", ENCODING_DICTIONARY, vector_ids[segment.vector_type], segment.dictionary_size))
                if definition.data_type == capi.TYPE_STRING:
                    _write_strings(out, list(segment.string_dictionary))
                else:
                    out.append(np.ascontiguousarray(segment.values).tobytes())
                _write_vector(out, segment)
            elif segment.encoding == capi.ENC_FRAME_OF_REFERENCE:
                out.append(struct.pack("<BBI", ENCODING_FOR, vector_ids[segment.vector_type], len(segment.values)))
                out.append(np.ascontiguousarray(segment.values, dtype=np.int32).tobytes())
                out.append(struct.pack("<B", 1 if segment.nulls is not None else 0))
                if segment.nulls is not None:
                    out.append(np.ascontiguousarray(segment.nulls, dtype=np.uint8).tobytes())
                _write_vector(out, segment)
            else:
                raise ValueError(f"cannot write encoding {segment.encoding}")
    with open(path, "wb") as file:
        file.write(b"".join(out))


# ---------------------------------------------------------------------------------------------------------------------
# The native loader (hyrise_b200/csrc/binary_loader.cu, hyb_binary_table_*): the same parse inside the C-ABI library, into
# pinned host blocks, with a one-call upload. This wrapper exposes it as a storage.Table whose segment buffers are views
# into the library's host blocks.
# ---------------------------------------------------------------------------------------------------------------------
import ctypes as C  # noqa: E402


class NativeBinaryTable:
    """hyb_binary_table: parse in C++ (no GPU needed), `upload(context)` = hyb_table_upload_binary."""

    def __init__(self, path: str, pinned: bool = False):
        self.lib = capi.load_library()
        self.ptr = C.c_void_p()
        capi.check(self.lib.hyb_binary_table_open(os.fsencode(path), 1 if pinned else 0, C.byref(self.ptr)))
        chunk_size, chunk_count, column_count = C.c_uint32(), C.c_uint32(), C.c_uint32()
        capi.check(self.lib.hyb_binary_table_info(self.ptr, C.byref(chunk_size), C.byref(chunk_count), C.byref(column_count)))
        definitions = []
        for column in range(column_count.value):
            name, data_type, nullable = C.c_char_p(), C.c_int32(), C.c_int32()
            capi.check(self.lib.hyb_binary_table_column(self.ptr, column, C.byref(name), C.byref(data_type), C.byref(nullable)))
            definitions.append(ColumnDefinition(name.value.decode(), data_type.value, bool(nullable.value)))
        view = capi.TableView()
        capi.check(self.lib.hyb_binary_table_view(self.ptr, C.byref(view)))
        self.table = Table(definitions, target_chunk_size=chunk_size.value)
        self.sorted_columns = []
        for chunk in range(chunk_count.value):
            segments = [self._segment(view.segments[chunk * column_count.value + column], chunk, column, definitions[column])
                        for column in range(column_count.value)]
            self.table.chunks.append(Chunk(segments))
            ids, modes, count = (C.c_uint16 * 64)(), (C.c_uint8 * 64)(), C.c_uint32()
            capi.check(self.lib.hyb_binary_table_sorted_columns(self.ptr, chunk, ids, modes, C.byref(count)))
            self.sorted_columns.append([(ids[i], modes[i]) for i in range(count.value)])

    @staticmethod
    def _view(address, dtype, count) -> np.ndarray | None:
        if not address:
            return None
        dtype = np.dtype(dtype)
        if count == 0:
            return np.zeros(0, dtype=dtype)
        buffer = (C.c_uint8 * (count * dtype.itemsize)).from_address(address)
        return np.frombuffer(buffer, dtype=dtype, count=count)

    def _segment(self, desc, chunk: int, column: int, definition: ColumnDefinition) -> Segment:
        rows = desc.row_count
        segment = Segment(desc.encoding, desc.data_type, rows, vector_type=desc.vector_type, bit_width=desc.bit_width,
                          dictionary_size=desc.dictionary_size)
        if desc.encoding == capi.ENC_UNENCODED:
            segment.values = self._view(desc.values, NUMPY_TYPES[desc.data_type], rows)
        elif desc.encoding == capi.ENC_FRAME_OF_REFERENCE:
            segment.values = self._view(desc.values, np.int32, (rows + capi.FOR_BLOCK_SIZE - 1) // capi.FOR_BLOCK_SIZE)
        elif definition.data_type != capi.TYPE_STRING:
            segment.values = self._view(desc.values, NUMPY_TYPES[desc.data_type], desc.dictionary_size)
        segment.nulls = self._view(desc.nulls, np.uint8, rows)
        if desc.encoding != capi.ENC_UNENCODED:
            if desc.vector_type == capi.VEC_BITPACKED:
                segment.attribute_vector = self._view(desc.attribute_vector, np.uint64, (rows * desc.bit_width + 63) // 64)
            else:
                width = {capi.VEC_FIXED_1B: np.uint8, capi.VEC_FIXED_2B: np.uint16, capi.VEC_FIXED_4B: np.uint32}[desc.vector_type]
                segment.attribute_vector = self._view(desc.attribute_vector, width, rows)
        if definition.data_type == capi.TYPE_STRING:
            chars, offsets, count = C.c_void_p(), C.POINTER(C.c_uint64)(), C.c_uint32()
            capi.check(self.lib.hyb_binary_table_string_dictionary(self.ptr, chunk, column, C.byref(chars), C.byref(offsets), C.byref(count)))
            blob = C.string_at(chars, offsets[count.value]) if count.value else b""
            segment.string_dictionary = _string_array([blob[offsets[i]:offsets[i + 1]] for i in range(count.value)]) \
                if count.value else np.zeros(0, dtype="S1")
            segment.dictionary_codes = self._view(desc.dictionary_codes, np.uint64, desc.dictionary_size)
        return segment

    def value_id_bounds(self, column: int, value: bytes, value2: bytes | None = None) -> np.ndarray:
        width = 4 if value2 is not None else 2
        bounds = np.empty((self.table.chunk_count, width), dtype=np.uint32)
        capi.check(self.lib.hyb_binary_table_value_id_bounds(self.ptr, column, value, len(value), value2, len(value2) if value2 else 0,
                                                             bounds.ctypes.data_as(C.POINTER(C.c_uint32))))
        return bounds

    def like_bitmaps(self, column: int, pattern: bytes, condition: int) -> np.ndarray:
        """hyb_binary_table_like_bitmaps: value_id_bounds of a LIKE predicate, the per-chunk dictionary match bitmaps."""
        count = C.c_uint32()
        capi.check(self.lib.hyb_binary_table_like_bitmaps(self.ptr, column, pattern, len(pattern), condition, None,
                                                          C.byref(count)))
        words = np.zeros(max(count.value, 1), dtype=np.uint32)
        capi.check(self.lib.hyb_binary_table_like_bitmaps(self.ptr, column, pattern, len(pattern), condition,
                                                          words.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(count)))
        return words[: count.value]

    def in_bitmaps(self, column: int, condition: int, elements) -> np.ndarray:
        """hyb_binary_table_in_bitmaps: dictionary_matches of `<string column> [NOT] IN (elements)` (bytes)."""
        chars, offsets = capi._string_dictionary_arguments(elements)
        arguments = (self.ptr, column, condition, chars, offsets.ctypes.data_as(C.POINTER(C.c_uint64)), len(offsets) - 1)
        count = C.c_uint32()
        capi.check(self.lib.hyb_binary_table_in_bitmaps(*arguments, None, C.byref(count)))
        words = np.zeros(max(count.value, 1), dtype=np.uint32)
        capi.check(self.lib.hyb_binary_table_in_bitmaps(*arguments, words.ctypes.data_as(C.POINTER(C.c_uint32)),
                                                        C.byref(count)))
        return words[: count.value]

    def column_translation(self, left_column: int, right_column: int) -> np.ndarray:
        """hyb_binary_table_column_translation: right_in_left of a column-vs-column scan on two string columns."""
        count = C.c_uint32()
        capi.check(self.lib.hyb_binary_table_column_translation(self.ptr, left_column, right_column, None, C.byref(count)))
        words = np.zeros(max(count.value, 1), dtype=np.uint32)
        capi.check(self.lib.hyb_binary_table_column_translation(self.ptr, left_column, right_column,
                                                                words.ctypes.data_as(C.POINTER(C.c_uint32)),
                                                                C.byref(count)))
        return words[: count.value]

    def string_order_ranks(self, column: int) -> np.ndarray:
        """hyb_binary_table_string_order_ranks: the order ranks of a string column (hyb_table_set_string_order's words)."""
        count = C.c_uint32()
        capi.check(self.lib.hyb_binary_table_string_order_ranks(self.ptr, column, None, C.byref(count)))
        ranks = np.zeros(max(count.value, 1), dtype=np.uint32)
        capi.check(self.lib.hyb_binary_table_string_order_ranks(self.ptr, column, ranks.ctypes.data_as(C.POINTER(C.c_uint32)),
                                                                C.byref(count)))
        return ranks[: count.value]

    def host_blocks(self) -> list:
        count = C.c_uint32()
        capi.check(self.lib.hyb_binary_table_blocks(self.ptr, None, C.byref(count)))
        blocks = (capi.HostBlock * max(count.value, 1))()
        capi.check(self.lib.hyb_binary_table_blocks(self.ptr, blocks, C.byref(count)))
        return list(blocks[: count.value])

    def upload(self, context):
        """hyb_table_upload_binary: one DMA per host block; returns a DeviceTable bound to this host table."""
        from .device import DeviceTable
        handle = C.c_uint64()
        capi.check(self.lib.hyb_table_upload_binary(context.ptr, self.ptr, C.byref(handle)))
        return DeviceTable(context, handle.value, self.table, self.table.view())

    def close(self) -> None:
        if self.ptr:
            self.lib.hyb_binary_table_close(self.ptr)
            self.ptr = None
