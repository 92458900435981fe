"""Device time of a Semi join with a secondary predicate (Q21's `EXISTS (... l2.l_orderkey = l1.l_orderkey AND
l2.l_suppkey <> l1.l_suppkey)`) against the same Semi join on the key alone and the Inner join that emits every candidate.

A seeded 60 M-row table shaped like SF-10 lineitem: orders of 1-7 rows each (uniform, as dbgen draws them), rows grouped by
order in key order, `suppkey` drawn at random from 100 000 suppliers. Every join is the table with itself on the order key:
(a) Semi on the key, (b) Semi with `build.suppkey <> probe.suppkey`, (c) Inner on the key (every candidate pair). The three
alternate after warm-ups; per join the median and p95 of hyb_operator_stats::device_ms, achieved bytes/s from
algorithmic_bytes over the median, the path and the output rows are printed with the card's name and power limit as one
JSON line (development aid)."""
import json
import subprocess
import sys

import numpy as np

sys.path.insert(0, ".")
from hyrise_b200 import capi  # noqa: E402
from hyrise_b200.device import DeviceContext  # noqa: E402
from hyrise_b200.storage import ColumnDefinition, Table  # noqa: E402

ROWS, WARMUP, REPEATS, SEED = 60_000_000, 3, 20, 42
JOINS = {
    "semi_key": (capi.JOIN_SEMI, None),
    "semi_suppkey_differs": (capi.JOIN_SEMI, [(1, 1, capi.PRED_NOT_EQUALS)]),
    "inner_key": (capi.JOIN_INNER, None),
}


def lineitem_like(rows: int, seed: int) -> Table:
    rng = np.random.default_rng(seed)
    lines = rng.integers(1, 8, rows // 2 + 1)  # 4 rows per order on average: twice as many orders as needed
    lines = lines[: np.searchsorted(np.cumsum(lines), rows) + 1]
    orderkey = np.repeat(np.arange(1, len(lines) + 1, dtype=np.int32), lines)[:rows]  # the last order may be cut short
    suppkey = rng.integers(1, 100_001, rows, dtype=np.int32)
    table = Table.from_columns([ColumnDefinition("l_orderkey", capi.TYPE_INT32), ColumnDefinition("l_suppkey", capi.TYPE_INT32)],
                               [orderkey, suppkey], None, capi.DEFAULT_CHUNK_SIZE)
    return table.encode("Unencoded")


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    rows = int(sys.argv[1]) if len(sys.argv) > 1 else ROWS
    table = lineitem_like(rows, SEED)
    assert table.row_count == rows, (table.row_count, rows)
    results = {"gpu": gpu, "rows": table.row_count, "warmup": WARMUP, "repeats": REPEATS}
    times = {label: [] for label in JOINS}
    facts = {}
    with DeviceContext(0) as device:
        lineitem = device.upload(table)
        for repeat in range(WARMUP + REPEATS):
            for label, (mode, secondary) in JOINS.items():
                result = device.join_hash(lineitem, 0, lineitem, 0, mode, -1, secondary=secondary)
                stats = device.last_stats()
                facts[label] = {"path": hex(stats.path), "output_rows": result.info()[0],
                                "algorithmic_bytes": stats.algorithmic_bytes}
                result.free()
                if repeat >= WARMUP:
                    times[label].append(stats.device_ms)
        lineitem.drop()
    for label in JOINS:
        median = float(np.median(times[label]))
        results[label] = dict(facts[label], device_ms_median=round(median, 3),
                              device_ms_p95=round(float(np.percentile(times[label], 95)), 3),
                              achieved_gb_per_s=round(facts[label]["algorithmic_bytes"] / median / 1e6, 1))
    print(json.dumps(results))


if __name__ == "__main__":
    main()
