#!/usr/bin/env python
"""Copies the reference's golden inputs for the [NOT] IN scans into tests/golden/ (run where /root/reference is mounted;
the tests only read tests/golden/). Existing fixtures stay unchanged: the part columns go into a new file,
sf-0.01_part_in.npz.

Sources (all under /root/reference/resources/test_data/tbl, hyrise/hyrise @ 2f7bedf3):
  * expression_evaluator/input_a.tbl: table_a of src/test/lib/expression/expression_evaluator_to_values_test.cpp
    (InListSeries, NotInListSeries), copied as expression_evaluator_input_a.tbl
  * tpch/sf-0.01 part (p_partkey, p_brand, p_size: TPC-H Q16), stored as compressed .npz
Data only — no reference source code is copied.
"""
import os
import shutil
import sys

from make_golden import REF, HERE, tbl_to_npz


def main():
    if not os.path.isdir(REF):
        sys.exit("reference test data not mounted; nothing to do")
    target = os.path.join(HERE, "tbl", "expression_evaluator_input_a.tbl")
    shutil.copyfile(os.path.join(REF, "expression_evaluator", "input_a.tbl"), target)
    os.chmod(target, 0o644)
    tbl_to_npz(os.path.join(REF, "tpch", "sf-0.01", "part.tbl"), os.path.join(HERE, "tpch", "sf-0.01_part_in.npz"),
               ["p_partkey", "p_brand", "p_size"])


if __name__ == "__main__":
    main()
