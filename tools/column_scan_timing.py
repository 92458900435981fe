"""Kernel time of a column-vs-column scan of two string columns (hyb_table_scan_columns: two 2-byte value-ID vectors and
a gathered translation word per row) against a one-column value-ID range scan over a 4-byte value-ID column: the same
column bytes per row, the same selectivity (about 0.5). 60 M rows in 65 535-row chunks; every chunk's dictionaries hold
4 000 entries, different for the two columns of the pair. The scans alternate after a warm-up under the default two-pass
pipeline; the medians of hyb_operator_stats::dominant_kernel_ms, the achieved bytes/s on the algorithmic bytes
(w_left + w_right + 8 * selectivity per row plus the translation words; 4 + 8 * selectivity for the range scan) and the
card's name and power limit are printed as one JSON line (development aid)."""
import json
import subprocess
import sys

import numpy as np

sys.path.insert(0, ".")
from hyrise_b200 import capi  # noqa: E402
from hyrise_b200.device import ColumnComparison, DeviceContext, Predicate  # noqa: E402
from hyrise_b200.storage import Chunk, ColumnDefinition, Segment, Table  # noqa: E402

ROWS, ENTRIES, REPEATS = 60_000_000, 4_000, 15


def dictionary(suffix: bytes) -> np.ndarray:
    """ENTRIES sorted date-like strings. The right column's entries carry a suffix: its dictionary differs from the left
    one in every entry, and the left date sorts first against its own date (a proper prefix), so `l < r` holds for about
    half of the rows."""
    days = np.arange(ENTRIES)
    return np.array([b"%04d-%02d-%02d%s" % (1992 + d // 372, 1 + (d // 31) % 12, 1 + d % 31, suffix) for d in days],
                    dtype="S12")


def timing_table(rng) -> Table:
    left, right = dictionary(b""), dictionary(b"x")
    table = Table([ColumnDefinition("l", capi.TYPE_STRING), ColumnDefinition("r", capi.TYPE_STRING),
                   ColumnDefinition("w", capi.TYPE_STRING)])
    for begin in range(0, ROWS, capi.DEFAULT_CHUNK_SIZE):
        rows = min(capi.DEFAULT_CHUNK_SIZE, ROWS - begin)
        segments = []
        for values, vector_type, dtype in ((left, capi.VEC_FIXED_2B, np.uint16), (right, capi.VEC_FIXED_2B, np.uint16),
                                           (left, capi.VEC_FIXED_4B, np.uint32)):
            ids = rng.integers(0, ENTRIES, rows).astype(dtype)
            segments.append(Segment(capi.ENC_DICTIONARY, capi.TYPE_STRING, rows, attribute_vector=ids,
                                    vector_type=vector_type, dictionary_size=ENTRIES, string_dictionary=values))
        table.chunks.append(Chunk(segments))
    return table


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    table = timing_table(np.random.default_rng(1))
    pair = ColumnComparison(0, capi.PRED_LESS_THAN, 1)
    ranged = Predicate(2, capi.PRED_LESS_THAN, bytes(table.chunks[0].segments[2].string_dictionary[ENTRIES // 2]))
    translation = table.string_column_translation(0, 1)
    results = {"gpu": gpu, "rows": ROWS, "dictionary_entries": ENTRIES, "pipeline": "two_pass"}
    with DeviceContext(0) as device:
        device_table = device.upload(table)
        times = {"pair": [], "range": []}
        rates = {"pair": [], "range": []}
        counts = {}
        for repeat in range(REPEATS + 3):
            for label in ("pair", "range"):
                if label == "pair":
                    result = device.table_scan_columns(device_table, pair, right_in_left=translation)
                else:
                    result = device.table_scan(device_table, ranged)
                stats = device.last_stats()
                counts[label] = result.info()[0]
                result.free()
                if repeat >= 3:
                    times[label].append(stats.dominant_kernel_ms)
                    rates[label].append(stats.algorithmic_bytes / (stats.dominant_kernel_ms * 1e-3))
        device_table.drop()
    for label in ("pair", "range"):
        results[label] = {"dominant_kernel_ms": round(float(np.median(times[label])), 4),
                          "algorithmic_gb_per_s": round(float(np.median(rates[label])) / 1e9, 1),
                          "selectivity": round(counts[label] / ROWS, 4)}
    results["pair_over_range"] = round(results["pair"]["dominant_kernel_ms"] / results["range"]["dominant_kernel_ms"], 4)
    print(json.dumps(results))


if __name__ == "__main__":
    main()
