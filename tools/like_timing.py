"""Kernel time of a scattered-match LIKE (value-ID set test) against a value-ID range scan of the same selectivity on the
same column (development aid). The column is SF-10 sized: 60 M rows in 65 535-row chunks, 2-byte value-IDs, 4 000
entries in every chunk's dictionary. The two scans alternate after a warm-up, under the default two-pass pipeline and
the single-pass bulk pipeline; the medians of hyb_operator_stats::dominant_kernel_ms are printed as one JSON line with
the card's name and power limit."""
import json
import subprocess
import sys

import numpy as np

sys.path.insert(0, ".")
from hyrise_b200 import capi  # noqa: E402
from hyrise_b200.device import DeviceContext, Predicate  # noqa: E402
from hyrise_b200.storage import Chunk, ColumnDefinition, Segment, Table  # noqa: E402

ROWS, ENTRIES, REPEATS = 60_000_000, 4_000, 15


def column_table(rng) -> Table:
    dictionary = np.array([b"item %04d %s" % (i, [b"plain", b"green", b"brass"][i % 3]) for i in range(ENTRIES)], dtype="S24")
    dictionary.sort()
    table = Table([ColumnDefinition("s", capi.TYPE_STRING)])
    for begin in range(0, ROWS, capi.DEFAULT_CHUNK_SIZE):
        rows = min(capi.DEFAULT_CHUNK_SIZE, ROWS - begin)
        ids = rng.integers(0, ENTRIES, rows).astype(np.uint16)
        table.chunks.append(Chunk([Segment(capi.ENC_DICTIONARY, capi.TYPE_STRING, rows, attribute_vector=ids,
                                           vector_type=capi.VEC_FIXED_2B, dictionary_size=ENTRIES,
                                           string_dictionary=dictionary)]))
    return table


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    table = column_table(np.random.default_rng(1))
    dictionary = table.chunks[0].segments[0].string_dictionary
    like = Predicate(0, capi.PRED_LIKE, b"%green%")  # every third entry: a scattered set in every chunk
    matches = sum(b"green" in bytes(entry) for entry in dictionary)
    ranged = Predicate(0, capi.PRED_LESS_THAN, bytes(dictionary[matches]))  # the first `matches` entries
    results = {"gpu": gpu, "rows": ROWS, "dictionary_entries": ENTRIES, "selectivity": matches / ENTRIES}
    with DeviceContext(0) as device:
        device_table = device.upload(table)
        for pipeline, options in (("two_pass", {"scan_two_pass": "1", "scan_bulk": "0"}),
                                  ("bulk", {"scan_two_pass": "0", "scan_bulk": "1"})):
            for name, value in options.items():
                device.set_option(name, value)
            times = {"like_set": [], "range": []}
            counts = {}
            for repeat in range(REPEATS + 3):
                for label, predicate in (("like_set", like), ("range", ranged)):
                    result = device.table_scan(device_table, predicate)
                    kernel_ms = device.last_stats().dominant_kernel_ms
                    counts[label] = result.info()[0]
                    result.free()
                    if repeat >= 3:
                        times[label].append(kernel_ms)
            results[pipeline] = {label: round(float(np.median(values)), 4) for label, values in times.items()}
            results[pipeline]["matches"] = counts
            results[pipeline]["set_over_range"] = round(results[pipeline]["like_set"] / results[pipeline]["range"], 4)
        device_table.drop()
    print(json.dumps(results))


if __name__ == "__main__":
    main()
