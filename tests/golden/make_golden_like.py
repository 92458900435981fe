#!/usr/bin/env python
"""Copies the reference's golden inputs for the LIKE scans into tests/golden/ (run where /root/reference is mounted; the
tests only read tests/golden/). Complements make_golden.py, whose outputs it leaves unchanged: the existing fixtures are
inputs of tests that must keep reading exactly what they read before, so o_comment goes into a second orders file
(sf-0.01_orders_comment.npz) instead of being added to sf-0.01_orders.npz.

Sources (all under /root/reference/resources/test_data/tbl, hyrise/hyrise @ 2f7bedf3):
  * int_string_like*.tbl: inputs and expected row sets of the LIKE cases of
    src/test/lib/operators/table_scan_string_test.cpp
  * tpch/sf-0.01 orders (o_orderkey, o_comment: Q13) and part (p_partkey, p_name, p_type, p_container: Q2, Q9, Q16,
    Q20), stored as compressed .npz
Data files only — no reference source code is copied.
"""
import os
import shutil
import sys

from make_golden import REF, HERE, tbl_to_npz

LIKE_TBL = [
    "int_string_like.tbl", "int_string_like_containing.tbl", "int_string_like_containing2.tbl",
    "int_string_like_containing_wildcard.tbl", "int_string_like_ending.tbl", "int_string_like_starting.tbl",
    "int_string_like_not_starting.tbl", "int_string_like_without_null.tbl", "int_string_like_special_chars.tbl",
    "int_string_like_special_chars_1.tbl", "int_string_like_special_chars_2.tbl", "int_string_like_special_chars_3.tbl",
]


def main():
    if not os.path.isdir(REF):
        sys.exit("reference test data not mounted; nothing to do")
    out_tbl = os.path.join(HERE, "tbl")
    for name in LIKE_TBL:
        shutil.copyfile(os.path.join(REF, name), os.path.join(out_tbl, name))
        os.chmod(os.path.join(out_tbl, name), 0o644)
    tpch = os.path.join(HERE, "tpch")
    tbl_to_npz(os.path.join(REF, "tpch", "sf-0.01", "orders.tbl"), os.path.join(tpch, "sf-0.01_orders_comment.npz"),
               ["o_orderkey", "o_comment"])
    tbl_to_npz(os.path.join(REF, "tpch", "sf-0.01", "part.tbl"), os.path.join(tpch, "sf-0.01_part.npz"),
               ["p_partkey", "p_name", "p_type", "p_container"])


if __name__ == "__main__":
    main()
