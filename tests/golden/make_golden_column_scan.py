#!/usr/bin/env python
"""Copies the reference's TPC-H lineitem date columns for the column-vs-column scans into tests/golden/ (run where
/root/reference is mounted; the tests only read tests/golden/). Existing fixtures stay unchanged: the columns go into a
new file, sf-0.01_lineitem_dates.npz.

Source: /root/reference/resources/test_data/tbl/tpch/sf-0.01/lineitem.tbl (hyrise/hyrise @ 2f7bedf3), the columns
l_orderkey, l_linenumber, l_shipdate, l_commitdate, l_receiptdate and l_shipmode (TPC-H Q4, Q12, Q21), stored as
compressed .npz. Data only — no reference source code is copied.
"""
import os
import sys

from make_golden import REF, HERE, tbl_to_npz


def main():
    if not os.path.isdir(REF):
        sys.exit("reference test data not mounted; nothing to do")
    tbl_to_npz(os.path.join(REF, "tpch", "sf-0.01", "lineitem.tbl"),
               os.path.join(HERE, "tpch", "sf-0.01_lineitem_dates.npz"),
               ["l_orderkey", "l_linenumber", "l_shipdate", "l_commitdate", "l_receiptdate", "l_shipmode"])


if __name__ == "__main__":
    main()
