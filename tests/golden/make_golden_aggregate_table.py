#!/usr/bin/env python
"""Copies the TPC-H sf-0.01 columns the aggregate-table queries need into tests/golden/ (run where /root/reference is
mounted; the tests only read tests/golden/). Existing fixtures stay unchanged: the columns go into new files.

Sources (all under /root/reference/resources/test_data/tbl, hyrise/hyrise @ 2f7bedf3):
  * tpch/sf-0.01 orders (o_orderkey, o_custkey, o_orderdate, o_totalprice: TPC-H Q18) -> sf-0.01_orders_totalprice.npz
  * tpch/sf-0.01 supplier (s_suppkey, s_name: TPC-H Q15) -> sf-0.01_supplier.npz
Stored as compressed .npz. Data only — no reference source code is copied.
"""
import os
import sys

from make_golden import REF, HERE, tbl_to_npz


def main():
    if not os.path.isdir(REF):
        sys.exit("reference test data not mounted; nothing to do")
    tpch = os.path.join(REF, "tpch", "sf-0.01")
    tbl_to_npz(os.path.join(tpch, "orders.tbl"), os.path.join(HERE, "tpch", "sf-0.01_orders_totalprice.npz"),
               ["o_orderkey", "o_custkey", "o_orderdate", "o_totalprice"])
    tbl_to_npz(os.path.join(tpch, "supplier.tbl"), os.path.join(HERE, "tpch", "sf-0.01_supplier.npz"),
               ["s_suppkey", "s_name"])


if __name__ == "__main__":
    main()
