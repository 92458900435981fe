"""Host-side mirror of the reference's storage layer for the hot path (numpy-backed).

Mirrors, by name and meaning, ``Table`` / ``Chunk`` / ``ValueSegment`` / ``DictionarySegment`` /
``FrameOfReferenceSegment`` (src/lib/storage/) and the segment encoders
(``ChunkEncoder::encode_all_chunks``, storage/chunk_encoder.hpp) so tests read like the reference's. Encoders here are
numpy restatements of

  * DictionaryEncoder::on_encode            storage/dictionary_segment/dictionary_encoder.hpp:33-103
  * FrameOfReferenceEncoder::on_encode      storage/frame_of_reference_segment/frame_of_reference_encoder.hpp:25-122
  * FixedWidthIntegerCompressor             storage/vector_compression/fixed_width_integer/fixed_width_integer_compressor.cpp:33-44
  * BitPackingCompressor                    storage/vector_compression/bitpacking/bitpacking_compressor.cpp:21-53

and are cross-checked against the oracle's independent C++ restatement in tests/test_storage.py.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Iterable, Sequence

import numpy as np

from . import capi

NUMPY_TYPES = {
    capi.TYPE_INT32: np.int32,
    capi.TYPE_INT64: np.int64,
    capi.TYPE_FLOAT32: np.float32,
    capi.TYPE_FLOAT64: np.float64,
}
TYPE_NAMES = {"int": capi.TYPE_INT32, "long": capi.TYPE_INT64, "float": capi.TYPE_FLOAT32,
              "double": capi.TYPE_FLOAT64, "string": capi.TYPE_STRING}
TYPE_NAMES_INV = {v: k for k, v in TYPE_NAMES.items()}


def _ptr(array: np.ndarray | None) -> int | None:
    return None if array is None else array.ctypes.data


# ---------------------------------------------------------------------------------------------------------------------
# Vector compression
# ---------------------------------------------------------------------------------------------------------------------
def compress_fixed_width(values: np.ndarray, max_value: int) -> tuple[np.ndarray, int]:
    """FixedWidthIntegerCompressor::_compress_using_max_value."""
    if max_value <= 0xFF:
        return values.astype(np.uint8), capi.VEC_FIXED_1B
    if max_value <= 0xFFFF:
        return values.astype(np.uint16), capi.VEC_FIXED_2B
    return values.astype(np.uint32), capi.VEC_FIXED_4B


def compress_bitpacking(values: np.ndarray) -> tuple[np.ndarray, int]:
    """BitPackingCompressor::compress: b = ceil(log2(max + 1)) (min 1) bits per entry, LSB-first in uint64 words
    (third_party/compact_vector/include/compact_iterator.hpp:218-252)."""
    n = len(values)
    bits = 1
    if n:
        max_element = int(values.max())
        if max_element != 0:
            bits = int(np.ceil(np.log2(max_element + 1)))
    words = np.zeros((n * bits + 63) // 64 + 1, dtype=np.uint64)  # +1: spill word simplifies the vectorised writes
    if n:
        bit = np.arange(n, dtype=np.uint64) * np.uint64(bits)
        word = (bit >> np.uint64(6)).astype(np.int64)
        shift = bit & np.uint64(63)
        v = values.astype(np.uint64)
        np.bitwise_or.at(words, word, v << shift)
        spill = (shift + np.uint64(bits)) > np.uint64(64)
        if spill.any():
            np.bitwise_or.at(words, word[spill] + 1, v[spill] >> (np.uint64(64) - shift[spill]))
    return words[: (n * bits + 63) // 64].copy(), bits


def decompress_vector(data: np.ndarray, vector_type: int, bits: int, n: int) -> np.ndarray:
    if vector_type != capi.VEC_BITPACKED:
        return data.astype(np.uint32)[:n]
    words = np.concatenate([data.astype(np.uint64), np.zeros(1, dtype=np.uint64)])
    bit = np.arange(n, dtype=np.uint64) * np.uint64(bits)
    word = (bit >> np.uint64(6)).astype(np.int64)
    shift = bit & np.uint64(63)
    value = words[word] >> shift
    spill = (shift + np.uint64(bits)) > np.uint64(64)
    value[spill] |= words[word[spill] + 1] << (np.uint64(64) - shift[spill])
    return (value & np.uint64((1 << bits) - 1)).astype(np.uint32)


# ---------------------------------------------------------------------------------------------------------------------
# Segments
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class Segment:
    """One column of one chunk, in the layout the device pool uploads (hyb_segment_desc)."""

    encoding: int
    data_type: int
    row_count: int
    values: np.ndarray | None = None          # unencoded values | numeric dictionary | FoR block minima
    nulls: np.ndarray | None = None           # uint8 per row (value / FoR segments)
    attribute_vector: np.ndarray | None = None
    vector_type: int = capi.VEC_NONE
    bit_width: int = 0
    dictionary_size: int = 0
    string_dictionary: np.ndarray | None = None   # host-only sorted dictionary of a string column (dtype 'S')
    dictionary_codes: np.ndarray | None = None    # uint64 group-by code per dictionary entry

    def desc(self) -> capi.SegmentDesc:
        d = capi.SegmentDesc()
        d.encoding = self.encoding
        d.data_type = self.data_type
        d.vector_type = self.vector_type
        d.bit_width = self.bit_width
        d.row_count = self.row_count
        d.dictionary_size = self.dictionary_size
        d.values = _ptr(self.values)
        d.nulls = _ptr(self.nulls)
        d.attribute_vector = _ptr(self.attribute_vector)
        d.dictionary_codes = _ptr(self.dictionary_codes)
        return d

    # Decoding (host side; used by tests and by the Python operator mirror to materialise results) -----------------
    def value_ids(self) -> np.ndarray:
        return decompress_vector(self.attribute_vector, self.vector_type, self.bit_width, self.row_count)

    def null_mask(self) -> np.ndarray:
        if self.encoding == capi.ENC_DICTIONARY:
            return self.value_ids() == self.dictionary_size
        if self.nulls is None:
            return np.zeros(self.row_count, dtype=bool)
        return self.nulls.astype(bool)

    def decode(self) -> np.ndarray:
        """Values per row (NULL rows hold an arbitrary value; combine with null_mask())."""
        if self.encoding == capi.ENC_UNENCODED:
            return self.values
        if self.encoding == capi.ENC_DICTIONARY:
            dictionary = self.string_dictionary if self.data_type == capi.TYPE_STRING else self.values
            ids = self.value_ids()
            if len(dictionary) == 0:
                return np.zeros(self.row_count, dtype=dictionary.dtype)
            return dictionary[np.minimum(ids, len(dictionary) - 1)]
        offsets = self.value_ids()
        minima = np.repeat(self.values, capi.FOR_BLOCK_SIZE)[: self.row_count]
        return (minima.astype(np.int64) + offsets.astype(np.int64)).astype(np.int32)


def short_string_code(value: bytes) -> int | None:
    """AggregateHash's immediate key for strings shorter than five characters (aggregate_hash.cpp:852-900)."""
    size = len(value)
    if size >= 5:
        return None
    base = [1, 2, 258, 65_794, 16_843_010][size]
    return base + sum(b << (8 * i) for i, b in enumerate(value))


class StringKeyRegistry:
    """Chunk-independent group-by codes for string dictionary entries, following _partition_by_groupby_keys
    (aggregate_hash.cpp:818-925): short strings are packed, longer ones get ids starting at 5 000 000 000 in order of
    first appearance. The reference assigns those ids while walking rows; walking dictionaries instead changes only the
    numeric value of the ids, never which rows share a group."""

    def __init__(self) -> None:
        self._ids: dict[bytes, int] = {}
        self._next = 5_000_000_000

    def codes(self, dictionary: np.ndarray) -> np.ndarray:
        out = np.empty(len(dictionary), dtype=np.uint64)
        for index, entry in enumerate(dictionary):
            entry = bytes(entry)
            code = short_string_code(entry)
            if code is None:
                code = self._ids.get(entry)
                if code is None:
                    code = self._next
                    self._ids[entry] = code
                    self._next += 1
            out[index] = code
        return out


def dictionary_order_ranks(dictionaries) -> np.ndarray:
    """Restatement of hyb_dictionary_order_ranks: the dense rank of every entry of every dictionary (sequences of bytes)
    among the distinct strings of all of them, as Python orders bytes (unsigned, a proper prefix first), dictionary
    after dictionary."""
    dictionaries = [[bytes(entry) for entry in dictionary] for dictionary in dictionaries]
    rank = {value: index for index, value in enumerate(sorted({entry for dictionary in dictionaries for entry in dictionary}))}
    return np.array([rank[entry] for dictionary in dictionaries for entry in dictionary], dtype=np.uint32)


def make_value_segment(values: np.ndarray, nulls: np.ndarray | None, data_type: int) -> Segment:
    if data_type == capi.TYPE_STRING:
        raise capi.UnsupportedOnDevice(capi.HYB_ERR_UNSUPPORTED, "unencoded string segments stay on the CPU")
    values = np.ascontiguousarray(values, dtype=NUMPY_TYPES[data_type])
    null_bytes = None if nulls is None or not nulls.any() else np.ascontiguousarray(nulls, dtype=np.uint8)
    if nulls is not None and null_bytes is None:
        null_bytes = np.zeros(len(values), dtype=np.uint8)  # nullable column, no NULL in this chunk
    return Segment(capi.ENC_UNENCODED, data_type, len(values), values=values, nulls=null_bytes)


def encode_dictionary(values: np.ndarray, nulls: np.ndarray | None, data_type: int, bitpacking: bool = False,
                      string_keys: StringKeyRegistry | None = None) -> Segment:
    """DictionaryEncoder::on_encode: sorted unique dictionary, value-ID = lower_bound, NULL = dictionary size."""
    n = len(values)
    null_mask = np.zeros(n, dtype=bool) if nulls is None else np.asarray(nulls, dtype=bool)
    dense = values[~null_mask]
    dictionary, inverse = np.unique(dense, return_inverse=True)
    ids = np.full(n, len(dictionary), dtype=np.uint32)
    ids[~null_mask] = inverse.astype(np.uint32)
    max_value_id = len(dictionary)  # the NULL value-ID is the largest id that can occur (dictionary_encoder.hpp:78-82)
    if bitpacking:
        attribute_vector, bits = compress_bitpacking(ids)
        vector_type = capi.VEC_BITPACKED
    else:
        attribute_vector, vector_type = compress_fixed_width(ids, max_value_id)
        bits = 0
    segment = Segment(capi.ENC_DICTIONARY, data_type, n, attribute_vector=np.ascontiguousarray(attribute_vector),
                      vector_type=vector_type, bit_width=bits, dictionary_size=len(dictionary))
    if data_type == capi.TYPE_STRING:
        segment.string_dictionary = dictionary
        if string_keys is not None:
            segment.dictionary_codes = string_keys.codes(dictionary)
    else:
        segment.values = np.ascontiguousarray(dictionary, dtype=NUMPY_TYPES[data_type])
    return segment


def encode_frame_of_reference(values: np.ndarray, nulls: np.ndarray | None, bitpacking: bool = False) -> Segment:
    """FrameOfReferenceEncoder::on_encode (int32 only): per 2048-row block the minimum of the non-NULL values
    (INT32_MAX for an all-NULL block); NULL rows get offset 0."""
    n = len(values)
    values = np.asarray(values, dtype=np.int32)
    null_mask = np.zeros(n, dtype=bool) if nulls is None else np.asarray(nulls, dtype=bool)
    blocks = (n + capi.FOR_BLOCK_SIZE - 1) // capi.FOR_BLOCK_SIZE
    padded = np.full(blocks * capi.FOR_BLOCK_SIZE, np.iinfo(np.int32).max, dtype=np.int64)
    padded[:n] = np.where(null_mask, np.iinfo(np.int32).max, values.astype(np.int64))
    minima = padded.reshape(blocks, capi.FOR_BLOCK_SIZE).min(axis=1) if blocks else np.zeros(0, dtype=np.int64)
    per_row_min = np.repeat(minima, capi.FOR_BLOCK_SIZE)[:n]
    offsets = np.where(null_mask, 0, values.astype(np.int64) - per_row_min).astype(np.uint32)
    max_offset = int(offsets.max()) if n else 0
    if bitpacking:
        compressed, bits = compress_bitpacking(offsets)
        vector_type = capi.VEC_BITPACKED
    else:
        compressed, vector_type = compress_fixed_width(offsets, max_offset)
        bits = 0
    null_bytes = np.ascontiguousarray(null_mask, dtype=np.uint8) if null_mask.any() else None
    return Segment(capi.ENC_FRAME_OF_REFERENCE, capi.TYPE_INT32, n, values=np.ascontiguousarray(minima, dtype=np.int32),
                   nulls=null_bytes, attribute_vector=np.ascontiguousarray(compressed), vector_type=vector_type,
                   bit_width=bits)


# ---------------------------------------------------------------------------------------------------------------------
# Table / Chunk
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class ColumnDefinition:
    name: str
    data_type: int
    nullable: bool = False


@dataclass
class Chunk:
    segments: list[Segment]

    @property
    def size(self) -> int:
        return self.segments[0].row_count if self.segments else 0


@dataclass
class Table:
    """Table(column_definitions, TableType::Data, chunk_size) — storage/table.hpp."""

    column_definitions: list[ColumnDefinition]
    chunks: list[Chunk] = field(default_factory=list)
    target_chunk_size: int = capi.DEFAULT_CHUNK_SIZE

    # construction ------------------------------------------------------------------------------------------------
    @classmethod
    def from_columns(cls, column_definitions: Sequence[ColumnDefinition], columns: Sequence[np.ndarray],
                     nulls: Sequence[np.ndarray | None] | None = None, chunk_size: int = capi.DEFAULT_CHUNK_SIZE,
                     ) -> "Table":
        """Unencoded table from whole-column arrays, split into chunks of `chunk_size` rows (Table::append)."""
        nulls = list(nulls) if nulls is not None else [None] * len(columns)
        table = cls(list(column_definitions), target_chunk_size=chunk_size)
        table._raw = []  # per chunk: list of (values, nulls) kept for (re-)encoding
        row_count = len(columns[0]) if columns else 0
        for begin in range(0, row_count, chunk_size):
            end = min(begin + chunk_size, row_count)
            raw = []
            for column, null in zip(columns, nulls):
                raw.append((column[begin:end], None if null is None else np.asarray(null[begin:end], dtype=bool)))
            table._raw.append(raw)
        table.encode("Unencoded")
        return table

    def encode(self, spec, chunk_ids: Iterable[int] | None = None, bitpacking: bool = False) -> "Table":
        """ChunkEncoder::encode_chunks: `spec` is one of "Unencoded" | "Dictionary" | "FrameOfReference" | "Automatic",
        or a list with one entry per column. "Automatic" follows segment_encoding_utils.cpp:105-115 (int32 ->
        FrameOfReference, everything else -> Dictionary). Strings are always dictionary encoded on this path."""
        specs = [spec] * len(self.column_definitions) if isinstance(spec, str) else list(spec)
        if not hasattr(self, "_string_keys"):
            self._string_keys = [StringKeyRegistry() for _ in self.column_definitions]
        while len(self.chunks) < len(self._raw):
            self.chunks.append(Chunk([None] * len(self.column_definitions)))
        chunk_ids = range(len(self._raw)) if chunk_ids is None else chunk_ids
        for chunk_id in chunk_ids:
            for column_id, definition in enumerate(self.column_definitions):
                values, nulls = self._raw[chunk_id][column_id]
                if definition.nullable and nulls is None:
                    nulls = np.zeros(len(values), dtype=bool)
                encoding = specs[column_id]
                if encoding == "Automatic":
                    encoding = "FrameOfReference" if definition.data_type == capi.TYPE_INT32 else "Dictionary"
                if definition.data_type == capi.TYPE_STRING:
                    encoding = "Dictionary"
                if encoding == "FrameOfReference" and definition.data_type != capi.TYPE_INT32:
                    encoding = "Dictionary"
                if encoding == "Unencoded":
                    segment = make_value_segment(values, nulls, definition.data_type)
                elif encoding == "Dictionary":
                    segment = encode_dictionary(values, nulls, definition.data_type, bitpacking,
                                                self._string_keys[column_id])
                elif encoding == "FrameOfReference":
                    segment = encode_frame_of_reference(values, nulls, bitpacking)
                else:
                    raise ValueError(f"unknown encoding {encoding!r}")
                self.chunks[chunk_id].segments[column_id] = segment
        return self

    # accessors ---------------------------------------------------------------------------------------------------
    @property
    def chunk_count(self) -> int:
        return len(self.chunks)

    @property
    def column_count(self) -> int:
        return len(self.column_definitions)

    @property
    def row_count(self) -> int:
        return sum(chunk.size for chunk in self.chunks)

    def column_id_by_name(self, name: str) -> int:
        for index, definition in enumerate(self.column_definitions):
            if definition.name == name:
                return index
        raise KeyError(name)

    def get_chunk(self, chunk_id: int) -> Chunk:
        return self.chunks[chunk_id]

    def view(self) -> "TableViewHolder":
        return TableViewHolder(self)

    def string_value_id_bounds(self, predicate) -> np.ndarray:
        """Per-chunk DictionarySegment::lower_bound / upper_bound (dictionary_segment.cpp:94-119) on the host-resident
        string dictionaries; INVALID_VALUE_ID when past the end. Layout: [chunk][lb, ub] or, for BETWEEN,
        [chunk][lb(lower), ub(lower), lb(upper), ub(upper)]."""
        between = capi.PRED_BETWEEN_INCLUSIVE <= predicate.condition <= capi.PRED_BETWEEN_EXCLUSIVE
        width = 4 if between else 2
        bounds = np.empty((self.chunk_count, width), dtype=np.uint32)
        values = [predicate.lower, predicate.upper] if between else [predicate.lower]
        for chunk_id, chunk in enumerate(self.chunks):
            dictionary = chunk.segments[predicate.column_id].string_dictionary
            for index, value in enumerate(values):
                needle = np.array([value if isinstance(value, bytes) else str(value).encode()], dtype="S")
                for offset, side in enumerate(("left", "right")):
                    position = int(np.searchsorted(dictionary, needle, side=side)[0]) if len(dictionary) else 0
                    bounds[chunk_id, 2 * index + offset] = capi.INVALID_VALUE_ID if position >= len(dictionary) \
                        else position
        return bounds

    def string_like_bitmaps(self, predicate) -> np.ndarray:
        """value_id_bounds of a LIKE predicate: per chunk, the dictionary match bitmap of ColumnLikeTableScanImpl
        (column_like_table_scan_impl.cpp:75-140) from hyb_like_dictionary_matches, ceil(dictionary size / 32) uint32 words
        per chunk in chunk order. The pattern is `predicate.lower` (bytes, or str encoded as UTF-8)."""
        pattern = predicate.lower if isinstance(predicate.lower, bytes) else str(predicate.lower).encode()
        words = [capi.like_dictionary_matches(pattern, predicate.condition,
                                              chunk.segments[predicate.column_id].string_dictionary)
                 for chunk in self.chunks]
        return np.concatenate(words) if words else np.zeros(0, dtype=np.uint32)

    def string_in_bitmaps(self, column_id: int, condition: int, elements) -> np.ndarray:
        """dictionary_matches of `<string column> [NOT] IN (elements)`: per chunk, hyb_in_dictionary_matches of the
        dictionary against the string elements (bytes), ceil(dictionary size / 32) uint32 words per chunk in chunk order;
        NOT IN is inverted."""
        words = [capi.in_dictionary_matches(condition, elements, chunk.segments[column_id].string_dictionary)
                 for chunk in self.chunks]
        return np.concatenate(words) if words else np.zeros(0, dtype=np.uint32)

    def string_column_translation(self, left_column_id: int, right_column_id: int) -> np.ndarray:
        """right_in_left of `left <condition> right` on two string columns: per chunk, hyb_dictionary_translate of the
        right dictionary into the left one's value-ID space, one uint32 word per right dictionary entry, in chunk order."""
        words = [capi.dictionary_translate(chunk.segments[left_column_id].string_dictionary,
                                           chunk.segments[right_column_id].string_dictionary)
                 for chunk in self.chunks]
        return np.concatenate(words) if words else np.zeros(0, dtype=np.uint32)

    def string_order_ranks(self, column_id: int) -> np.ndarray:
        """hyb_table_set_string_order's words for a string column: every dictionary entry's dense rank among the column's
        distinct strings, chunk after chunk (dictionary_order_ranks over the chunks' dictionaries)."""
        return dictionary_order_ranks([chunk.segments[column_id].string_dictionary for chunk in self.chunks])

    def column_values(self, column_id: int) -> tuple[np.ndarray, np.ndarray]:
        """Decoded values and null mask of a whole column (host side)."""
        if not self.chunks:
            dtype = NUMPY_TYPES.get(self.column_definitions[column_id].data_type, "S1")
            return np.zeros(0, dtype=dtype), np.zeros(0, dtype=bool)
        values = np.concatenate([chunk.segments[column_id].decode() for chunk in self.chunks])
        nulls = np.concatenate([chunk.segments[column_id].null_mask() for chunk in self.chunks])
        return values, nulls


class TableViewHolder:
    """Owns the ctypes descriptor array behind a hyb_table_view (keeps the numpy buffers alive)."""

    def __init__(self, table: Table):
        self.table = table
        count = table.chunk_count * table.column_count
        self._descs = (capi.SegmentDesc * max(count, 1))()
        for chunk_id, chunk in enumerate(table.chunks):
            for column_id, segment in enumerate(chunk.segments):
                self._descs[chunk_id * table.column_count + column_id] = segment.desc()
        self.view = capi.TableView(table.chunk_count, table.column_count,
                                   C.cast(self._descs, C.POINTER(capi.SegmentDesc)))

    def pointer(self):
        return C.byref(self.view)

    def chunk_descs(self, chunk_id: int):
        offset = chunk_id * self.table.column_count
        return C.cast(C.byref(self._descs, offset * C.sizeof(capi.SegmentDesc)), C.POINTER(capi.SegmentDesc))


# ---------------------------------------------------------------------------------------------------------------------
# .tbl loader — utils/load_table.cpp:22-94
# ---------------------------------------------------------------------------------------------------------------------
def load_table(path: str, chunk_size: int = capi.DEFAULT_CHUNK_SIZE) -> Table:
    with open(path, "r", encoding="utf-8") as handle:
        lines = handle.read().split("\n")
    if lines and lines[-1] == "":
        lines.pop()
    names = lines[0].split("|")
    definitions = []
    for name, type_spec in zip(names, lines[1].split("|")):
        parts = type_spec.split("_")
        definitions.append(ColumnDefinition(name, TYPE_NAMES[parts[0]], len(parts) > 1 and parts[1] == "null"))
    rows = [line.split("|") for line in lines[2:]]
    columns, nulls = [], []
    for column_id, definition in enumerate(definitions):
        raw = [row[column_id] for row in rows]
        null_mask = np.array([definition.nullable and value == "null" for value in raw], dtype=bool)
        if definition.data_type == capi.TYPE_STRING:
            data = np.array([b"" if is_null else value.encode() for value, is_null in zip(raw, null_mask)], dtype="S")
            if data.size == 0:
                data = np.zeros(0, dtype="S1")
        else:
            dtype = NUMPY_TYPES[definition.data_type]
            data = np.array([0 if is_null else value for value, is_null in zip(raw, null_mask)], dtype=np.float64
                            if dtype in (np.float32, np.float64) else np.int64).astype(dtype) if raw else \
                np.zeros(0, dtype=dtype)
        columns.append(data)
        nulls.append(null_mask if definition.nullable else None)
    return Table.from_columns(definitions, columns, nulls, chunk_size)
