"""Kernel and device time of MAX over a string column against MAX over an INT32 dictionary column with identical
attribute vectors and dictionary sizes: 60 M rows in 65 535-row chunks, 2-byte value-IDs, 4 000-entry dictionaries per
chunk (consecutive chunks share most of their strings), grouped by a 1-byte-value-ID column with 4 groups. Both run the
general kernel's row loop; the string MAX reads the column's order ranks as its dictionaries and adds the small kernel
that resolves each group's extreme rank. The two alternate; the medians of 15 calls after 3 warm-ups of
hyb_operator_stats::dominant_kernel_ms and device_ms, their ratio, the host time to build the order ranks of the
~3.7 M dictionary entries (hyb_dictionary_order_ranks) and the card's name and power limit are printed as one JSON
line (development aid)."""
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
from hyrise_b200 import capi  # noqa: E402
from hyrise_b200.device import Aggregate, DeviceContext, Expression  # noqa: E402
from hyrise_b200.storage import Chunk, ColumnDefinition, Segment, Table  # noqa: E402

ROWS, CHUNK, DICTIONARY, GROUPS = 60_000_000, 65_535, 4_000, 4
WARMUP, REPEATS = 3, 15


def build_table(rng):
    """Columns: g (INT32, 4-entry dictionary, 1-byte IDs), s (STRING), i (INT32): s and i share every attribute vector."""
    definitions = [ColumnDefinition("g", capi.TYPE_INT32), ColumnDefinition("s", capi.TYPE_STRING),
                   ColumnDefinition("i", capi.TYPE_INT32)]
    table = Table(definitions, target_chunk_size=CHUNK)
    group_dictionary = np.arange(GROUPS, dtype=np.int32) * 1000  # sparse keys: no immediate-key order
    for begin in range(0, ROWS, CHUNK):
        chunk_id, rows = begin // CHUNK, min(CHUNK, ROWS - begin)
        groups = Segment(capi.ENC_DICTIONARY, capi.TYPE_INT32, rows, values=group_dictionary,
                         attribute_vector=rng.integers(0, GROUPS, rows).astype(np.uint8), vector_type=capi.VEC_FIXED_1B,
                         dictionary_size=GROUPS)
        ids = rng.integers(0, DICTIONARY, rows).astype(np.uint16)
        first = chunk_id * (DICTIONARY // 4)  # a quarter of the entries is new in every chunk
        strings = np.array([b"s%09d" % (first + i) for i in range(DICTIONARY)], dtype="S")
        numbers = (np.arange(DICTIONARY, dtype=np.int32) + first).astype(np.int32)
        text = Segment(capi.ENC_DICTIONARY, capi.TYPE_STRING, rows, attribute_vector=ids, vector_type=capi.VEC_FIXED_2B,
                       dictionary_size=DICTIONARY, string_dictionary=strings)
        integers = Segment(capi.ENC_DICTIONARY, capi.TYPE_INT32, rows, values=numbers, attribute_vector=ids,
                           vector_type=capi.VEC_FIXED_2B, dictionary_size=DICTIONARY)
        table.chunks.append(Chunk([groups, text, integers]))
    return table


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    table = build_table(np.random.default_rng(42))
    dictionaries = [chunk.segments[1].string_dictionary for chunk in table.chunks]
    begin = time.perf_counter()
    ranks, distinct = capi.dictionary_order_ranks(dictionaries)
    rank_seconds = time.perf_counter() - begin
    queries = {"max_string": Aggregate(capi.AGG_MAX, Expression.column(1)),
               "max_int32": Aggregate(capi.AGG_MAX, Expression.column(2))}
    results = {"gpu": gpu, "rows": ROWS, "chunks": table.chunk_count, "dictionary_entries": int(len(ranks)),
               "distinct_strings": distinct, "rank_build_host_s": round(rank_seconds, 3)}
    with DeviceContext(0) as device:
        device_table = device.upload(table)
        device.set_string_order(device_table, 1, ranks)
        kernel = {label: [] for label in queries}
        total = {label: [] for label in queries}
        paths = {}
        for repeat in range(WARMUP + REPEATS):
            for label, aggregate in queries.items():
                device.aggregate_hash(device_table, [0], [aggregate])
                stats = device.last_stats()
                paths[label] = stats.path
                if repeat >= WARMUP:
                    kernel[label].append(stats.dominant_kernel_ms)
                    total[label].append(stats.device_ms)
        device_table.drop()
    for label in queries:
        results[label] = {"dominant_kernel_ms": round(float(np.median(kernel[label])), 4),
                          "device_ms": round(float(np.median(total[label])), 4), "path": paths[label]}
    results["string_over_int32_device"] = round(results["max_string"]["device_ms"] / results["max_int32"]["device_ms"], 3)
    results["string_over_int32_kernel"] = round(
        results["max_string"]["dominant_kernel_ms"] / results["max_int32"]["dominant_kernel_ms"], 3)
    print(json.dumps(results))


if __name__ == "__main__":
    main()
