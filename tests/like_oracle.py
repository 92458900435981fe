"""CPU oracle for LIKE scans (test infrastructure, never imported by hyrise_b200/).

An independent restatement of the reference's LikeMatcher (expression/evaluation/like_matcher.{hpp,cpp}) and of the
generic, row-by-row path of ColumnLikeTableScanImpl (operators/table_scan/column_like_table_scan_impl.cpp): every row's
string is matched on its own, a NULL never matches. It uses no dictionary bitmap, so it stays independent of the
library's dictionary path (hyb_like_dictionary_matches + the device's value-ID set test).

Matching rules restated from the reference:
  * tokens: `_` is one character, `%` any run, the rest literal (pattern_string_to_tokens); no escape character;
  * [str, %] starts-with, [%, str] ends-with, [%, str, %] contains; tokens alternating %, str, %, ... from the first on
    (the last may be a string) are an ordered multiple-contains; these match raw bytes;
  * anything else is the anchored ECMAScript regex of sql_like_to_regex (like_matcher.cpp:32-55): literals stay
    literal, `_` is `.` and `%` is `.*`, and ECMAScript's `.` matches neither '\\n' nor '\\r'. Patterns with `[` or `]`
    would open bracket expressions in that regex; they are not restated here;
  * the INSENSITIVE variants lower A-Z of pattern and input (std::tolower in the C locale), NOT inverts.
"""
from __future__ import annotations

import re

import numpy as np

from hyrise_b200 import capi
from hyrise_b200.device import ROW_ID_DTYPE
from oracle_lib import HostPosList

ANY, SINGLE = "%", "_"
NULL_CHUNK_ID = 0xFFFFFFFF  # NULL_ROW_ID of an outer join's result
_UPPER = bytes(range(ord("A"), ord("Z") + 1))
_LOWER_TABLE = bytes.maketrans(_UPPER, _UPPER.lower())


def lower(value: bytes) -> bytes:
    return value.translate(_LOWER_TABLE)


def tokens(pattern: bytes) -> list:
    """pattern_string_to_tokens: list of ANY / SINGLE / bytes."""
    out, literal = [], b""
    for byte in pattern:
        char = bytes([byte])
        if char in (b"%", b"_"):
            if literal:
                out.append(literal)
                literal = b""
            out.append(ANY if char == b"%" else SINGLE)
        else:
            literal += char
    if literal:
        out.append(literal)
    return out


def form(pattern: bytes):
    """(kind, payload): kind in starts_with / ends_with / contains / multiple_contains / regex."""
    t = tokens(pattern)
    if len(t) == 2 and isinstance(t[0], bytes) and t[1] == ANY:
        return "starts_with", t[0]
    if len(t) == 2 and t[0] == ANY and isinstance(t[1], bytes):
        return "ends_with", t[1]
    if len(t) == 3 and t[0] == ANY and isinstance(t[1], bytes) and t[2] == ANY:
        return "contains", t[1]
    if all((token == ANY) if index % 2 == 0 else isinstance(token, bytes) for index, token in enumerate(t)):
        return "multiple_contains", [token for token in t if isinstance(token, bytes)]
    if b"[" in pattern or b"]" in pattern:
        raise NotImplementedError("bracket expressions of the regex form are not restated")
    body = b"".join(b"[^\n\r]*" if token == ANY else b"[^\n\r]" if token == SINGLE else re.escape(token) for token in t)
    return "regex", re.compile(body)


class Matcher:
    def __init__(self, pattern: bytes, condition: int):
        assert condition in capi.LIKE_CONDITIONS
        self.insensitive = condition in (capi.PRED_LIKE_INSENSITIVE, capi.PRED_NOT_LIKE_INSENSITIVE)
        self.invert = condition in (capi.PRED_NOT_LIKE, capi.PRED_NOT_LIKE_INSENSITIVE)
        self.kind, self.payload = form(lower(pattern) if self.insensitive else pattern)

    def __call__(self, value: bytes) -> bool:
        value = lower(value) if self.insensitive else value
        if self.kind == "starts_with":
            match = value.startswith(self.payload)
        elif self.kind == "ends_with":
            match = value.endswith(self.payload)
        elif self.kind == "contains":
            match = self.payload in value
        elif self.kind == "multiple_contains":
            match, at = True, 0
            for needle in self.payload:
                found = value.find(needle, at)
                if found < 0:
                    match = False
                    break
                at = found + len(needle)
        else:
            match = self.payload.fullmatch(value) is not None
        return match != self.invert


def match(value: bytes, pattern: bytes, condition: int) -> bool:
    return Matcher(pattern, condition)(value)


def _row_matches(table, column_id: int, matcher: Matcher) -> list[np.ndarray]:
    """Per chunk: whether each row's decoded string satisfies the matcher (False for NULL). The matcher is a pure
    function of the string, so it runs once per distinct string of a chunk; the segment's value-IDs are not used."""
    out = []
    for chunk in table.chunks:
        segment = chunk.segments[column_id]
        values, nulls = segment.decode(), segment.null_mask()
        if len(values) == 0:
            out.append(np.zeros(0, dtype=bool))
            continue
        distinct, inverse = np.unique(values, return_inverse=True)
        verdicts = np.array([matcher(bytes(value)) for value in distinct], dtype=bool)
        out.append(verdicts[inverse.reshape(-1)] & ~nulls)
    return out


def table_scan(table, column_id: int, pattern: bytes, condition: int, input_filter: HostPosList | None = None,
               ascending: bool = True) -> HostPosList:
    """TableScan with a ColumnLikeTableScanImpl, row by row. With `input_filter` (a previous scan's output, or one side of
    a join result that may hold NULL_ROW_IDs) the matches keep the input order; an `ascending` input (a scan's output)
    keeps per-chunk boundaries, any other input forms one list, as hyb_table_scan reports it."""
    if table.column_definitions[column_id].data_type != capi.TYPE_STRING:
        raise ValueError("LIKE needs a string column")
    matches = _row_matches(table, column_id, Matcher(pattern, condition))
    if input_filter is None:
        parts, offsets = [], [0]
        for chunk_id, chunk_matches in enumerate(matches):
            chunk_rows = np.zeros(int(chunk_matches.sum()), dtype=ROW_ID_DTYPE)
            chunk_rows["chunk_id"] = chunk_id
            chunk_rows["chunk_offset"] = np.flatnonzero(chunk_matches)
            parts.append(chunk_rows)
            offsets.append(offsets[-1] + len(chunk_rows))
        rows = np.concatenate(parts) if parts else np.zeros(0, dtype=ROW_ID_DTYPE)
        return HostPosList(rows, np.array(offsets, dtype=np.uint64))
    keep = np.zeros(len(input_filter.row_ids), dtype=bool)
    for index, row in enumerate(input_filter.row_ids):
        chunk_id = int(row["chunk_id"])
        # NULL_ROW_ID (outer join): a NULL value, never LIKE anything
        keep[index] = chunk_id != NULL_CHUNK_ID and bool(matches[chunk_id][int(row["chunk_offset"])])
    rows = np.ascontiguousarray(input_filter.row_ids[keep])
    if ascending:
        ends = np.searchsorted(rows["chunk_id"], np.arange(table.chunk_count), side="right") if len(rows) else \
            np.zeros(table.chunk_count, dtype=np.int64)
        offsets = np.concatenate([[0], ends]).astype(np.uint64)
    else:
        offsets = np.array([0, len(rows)], dtype=np.uint64)
    return HostPosList(rows, offsets)


def dictionary_matches(entries, pattern: bytes, condition: int) -> np.ndarray:
    """The bitmap hyb_like_dictionary_matches must produce, from the row-wise matcher: ceil(n / 32) uint32 words."""
    bits = np.array([match(bytes(entry), pattern, condition) for entry in entries], dtype=bool)
    padded = np.zeros(((len(bits) + 31) // 32) * 32, dtype=bool)
    padded[: len(bits)] = bits
    weights = np.uint64(1) << np.arange(32, dtype=np.uint64)
    return (padded.reshape(-1, 32).astype(np.uint64) * weights).sum(axis=1).astype(np.uint32)
