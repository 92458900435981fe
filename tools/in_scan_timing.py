"""Kernel time of `<column> IN (<8 literals>)` scans (hyb_table_scan_in) against a BETWEEN of the same selectivity on the
same column. 60 M rows in 65 535-row chunks, values uniform in [0, 1000), so 8 list elements and an 8-value BETWEEN both
select 0.8 % of the rows:
  (a) an int32 ValueSegment column: the list's intervals are searched per row (evaluate8_in);
  (b) an int32 Dictionary column with 2-byte value-IDs: the list becomes a value-ID set per chunk (in_prepare_kernel);
  (c) a string Dictionary column with 2-byte value-IDs: the list's dictionary bitmaps, the LIKE path's kTestIdSet.
Each case alternates its IN scan with its BETWEEN scan, 15 timed repeats after 3 warm-ups, under the default two-pass
pipeline; the medians of hyb_operator_stats::dominant_kernel_ms, the achieved bytes/s on the algorithmic bytes and the
card's name and power limit are printed as one JSON line (development aid)."""
import json
import subprocess
import sys

import numpy as np

sys.path.insert(0, ".")
from hyrise_b200 import capi  # noqa: E402
from hyrise_b200.device import DeviceContext, InList, Predicate  # noqa: E402
from hyrise_b200.storage import Chunk, ColumnDefinition, Segment, Table  # noqa: E402

ROWS, DOMAIN, REPEATS, WARMUP = 60_000_000, 1000, 15, 3
LIST = [3, 97, 211, 350, 512, 640, 777, 901]
STRINGS = np.array([b"key-%04d" % v for v in range(DOMAIN)], dtype="S8")


def timing_table(rng) -> Table:
    table = Table([ColumnDefinition("v", capi.TYPE_INT32), ColumnDefinition("d", capi.TYPE_INT32),
                   ColumnDefinition("s", capi.TYPE_STRING)])
    dictionary = np.arange(DOMAIN, dtype=np.int32)
    for begin in range(0, ROWS, capi.DEFAULT_CHUNK_SIZE):
        rows = min(capi.DEFAULT_CHUNK_SIZE, ROWS - begin)
        values = rng.integers(0, DOMAIN, rows).astype(np.int32)
        table.chunks.append(Chunk([
            Segment(capi.ENC_UNENCODED, capi.TYPE_INT32, rows, values=values),
            Segment(capi.ENC_DICTIONARY, capi.TYPE_INT32, rows, values=dictionary, attribute_vector=values.astype(np.uint16),
                    vector_type=capi.VEC_FIXED_2B, dictionary_size=DOMAIN),
            Segment(capi.ENC_DICTIONARY, capi.TYPE_STRING, rows, attribute_vector=values.astype(np.uint16),
                    vector_type=capi.VEC_FIXED_2B, dictionary_size=DOMAIN, string_dictionary=STRINGS),
        ]))
    return table


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    table = timing_table(np.random.default_rng(1))
    cases = {
        "a_value_int32": (InList(0, capi.PRED_IN, LIST), Predicate(0, capi.PRED_BETWEEN_INCLUSIVE, 0, 7)),
        "b_dictionary_int32": (InList(1, capi.PRED_IN, LIST), Predicate(1, capi.PRED_BETWEEN_INCLUSIVE, 0, 7)),
        "c_dictionary_string": (InList(2, capi.PRED_IN, [bytes(STRINGS[v]) for v in LIST]),
                                Predicate(2, capi.PRED_BETWEEN_INCLUSIVE, bytes(STRINGS[0]), bytes(STRINGS[7]))),
    }
    results = {"gpu": gpu, "rows": ROWS, "list_elements": len(LIST), "pipeline": "two_pass"}
    with DeviceContext(0) as device:
        device_table = device.upload(table)
        for name, (in_list, between) in cases.items():
            times = {"in": [], "between": []}
            rates = {"in": [], "between": []}
            counts = {}
            for repeat in range(REPEATS + WARMUP):
                for label in ("in", "between"):
                    if label == "in":
                        result = device.table_scan_in(device_table, in_list)
                    else:
                        result = device.table_scan(device_table, between)
                    stats = device.last_stats()
                    counts[label] = result.info()[0]
                    result.free()
                    if repeat >= WARMUP:
                        times[label].append(stats.dominant_kernel_ms)
                        rates[label].append(stats.algorithmic_bytes / (stats.dominant_kernel_ms * 1e-3))
            case = {}
            for label in ("in", "between"):
                case[label] = {"dominant_kernel_ms": round(float(np.median(times[label])), 4),
                               "algorithmic_gb_per_s": round(float(np.median(rates[label])) / 1e9, 1),
                               "selectivity": round(counts[label] / ROWS, 5)}
            case["in_over_between"] = round(case["in"]["dominant_kernel_ms"] / case["between"]["dominant_kernel_ms"], 4)
            results[name] = case
        device_table.drop()
    print(json.dumps(results))


if __name__ == "__main__":
    main()
