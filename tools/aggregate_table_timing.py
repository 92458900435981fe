"""Device time of TPC-H Q18's subquery shape on the generator's lineitem (SF 10 by default: about 60 M rows, 15 M orders):
  (a) the aggregate GROUP BY l_orderkey, SUM(l_quantity) (kept alive);
  (b) hyb_aggregate_result_table of it, columns (l_orderkey at the representative rows, the sum): device_ms, the gather
      kernel's ms (dominant_kernel_ms) and algorithmic_bytes;
  (c) the HAVING scan SUM(l_quantity) > 300 on that table;
  (d) the semi join of orders onto the HAVING rows (o_orderkey IN (...)).
Each is timed ITERATIONS times after WARMUP runs, in order; the median and p95 of hyb_operator_stats::device_ms (CUDA
events), the rows, and the card's name and power limit, read in the same run, are printed as one JSON line. The HAVING
rows are checked once against the aggregate's own sums (development aid)."""
import argparse
import json
import subprocess
import sys

import numpy as np

sys.path.insert(0, ".")
from hyrise_b200 import capi  # noqa: E402
from hyrise_b200.device import Aggregate, DeviceContext, Expression, Predicate  # noqa: E402
from hyrise_b200.tpch import L_ORDERKEY, L_QUANTITY, O_ORDERKEY, TpchTables  # noqa: E402

ITERATIONS, WARMUP, QUANTITY = 10, 2, 300


def log(message):
    print(f"aggregate_table_timing: {message}", file=sys.stderr, flush=True)


def summary(times, extra):
    return dict(extra, device_ms_median=round(float(np.median(times)), 3),
                device_ms_p95=round(float(np.percentile(times, 95)), 3))


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--sf", type=float, default=10)
    args = parser.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    log(f"generating SF {args.sf}")
    data = TpchTables(args.sf, pinned=True)
    log(f"lineitem {data.lineitem.row_count} rows, orders {data.orders.row_count} rows")
    columns = [(capi.SORT_KEY_COLUMN, L_ORDERKEY), (capi.SORT_KEY_AGGREGATE, 0)]
    times = {"aggregate": [], "result_table": [], "result_table_kernel": [], "having_scan": [], "semi_join": []}
    facts = {}
    with DeviceContext(0) as device:
        lineitem, orders = device.upload(data.lineitem), device.upload(data.orders)
        log("uploaded")
        for repeat in range(WARMUP + ITERATIONS):
            timed = repeat >= WARMUP
            log(f"run {repeat}")
            output = device.aggregate_hash(lineitem, [L_ORDERKEY], [Aggregate(capi.AGG_SUM, Expression.column(L_QUANTITY))],
                                           keep_result=True)
            stats = device.last_stats()
            facts["aggregate"] = {"groups": output.group_count, "path": stats.path}
            if timed:
                times["aggregate"].append(stats.device_ms)
            if repeat == 0:
                log("aggregated")
            table = device.aggregate_table(output.result_handle, columns)
            stats = device.last_stats()
            facts["result_table"] = {"rows": stats.output_rows, "kernel_launches": stats.kernel_launches,
                                     "algorithmic_bytes": stats.algorithmic_bytes}
            if timed:
                times["result_table"].append(stats.device_ms)
                times["result_table_kernel"].append(stats.dominant_kernel_ms)
            if repeat == 0:
                log("table built")
            having = device.table_scan(table, Predicate(1, capi.PRED_GREATER_THAN, QUANTITY))
            stats = device.last_stats()
            facts["having_scan"] = {"rows": having.info()[0]}
            if timed:
                times["having_scan"].append(stats.device_ms)
            if repeat == 0:
                log("scanned")
            semi = device.join_hash(table, 0, orders, O_ORDERKEY, capi.JOIN_SEMI, build_filter=having)
            stats = device.last_stats()
            facts["semi_join"] = {"rows": semi.info()[0], "path": hex(stats.path)}
            if timed:
                times["semi_join"].append(stats.device_ms)
            if repeat == 0:  # the HAVING rows against the aggregate's own sums
                sums = output.values[0]
                assert facts["having_scan"]["rows"] == int(np.count_nonzero(sums > QUANTITY))
            semi.free()
            having.free()
            table.drop()
            device.free_aggregate_result(output.result_handle)
    result = {"gpu": gpu, "scale_factor": args.sf, "lineitem_rows": data.lineitem.row_count,
              "warmup": WARMUP, "iterations": ITERATIONS}
    for label in ("aggregate", "having_scan", "semi_join"):
        result[label] = summary(times[label], facts[label])
    median = float(np.median(times["result_table"]))
    result["result_table"] = summary(times["result_table"], dict(
        facts["result_table"], gather_kernel_ms_median=round(float(np.median(times["result_table_kernel"])), 3),
        achieved_gb_per_s=round(facts["result_table"]["algorithmic_bytes"] / median / 1e6, 1)))
    print(json.dumps(result))
    data.close()


if __name__ == "__main__":
    main()
