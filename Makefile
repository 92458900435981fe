# Builds the sm_90a (H100) C-ABI library, the TPC-H generator and the CPU oracle (test infrastructure).
# `python -c "import __graft_entry__ as g; g.build()"` drives this.
NVCC      ?= nvcc
CXX       ?= g++
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVCCFLAGS := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall,-Wno-unused-function -Xptxas -v
CSRC      := hyrise_b200/csrc
LIB       := hyrise_b200/lib/libhyrise_b200.so
CU_SRCS   := $(wildcard $(CSRC)/*.cu)
CU_OBJS   := $(patsubst $(CSRC)/%.cu,build/%.o,$(CU_SRCS))
HDRS      := $(wildcard $(CSRC)/*.hpp) $(wildcard $(CSRC)/*.cuh) include/hyrise_b200.h

TPCH_LIB  := hyrise_b200/lib/libhyb_tpch.so

COLUMN_SCAN_ORACLE := build/libcolumn_scan_oracle.so
AGGREGATE_DISTINCT_ORACLE := build/libaggregate_distinct_oracle.so
IN_SCAN_ORACLE := build/libin_scan_oracle.so
EXPRESSION_SCAN_ORACLE := build/libexpression_scan_oracle.so
JOIN_PREDICATES_ORACLE := build/libjoin_predicates_oracle.so

all: $(LIB) $(TPCH_LIB) oracle $(COLUMN_SCAN_ORACLE) $(AGGREGATE_DISTINCT_ORACLE) $(IN_SCAN_ORACLE) \
     $(EXPRESSION_SCAN_ORACLE) $(JOIN_PREDICATES_ORACLE)

build/%.o: $(CSRC)/%.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -c $< -o $@ 2> build/$*.ptxas.log || (cat build/$*.ptxas.log; exit 1)

$(LIB): $(CU_OBJS)
	@mkdir -p hyrise_b200/lib
	$(NVCC) $(ARCH) -shared -o $@ $(CU_OBJS) -cudart shared

$(TPCH_LIB): $(CSRC)/tpch_gen.cpp include/hyrise_b200_tpch.h include/hyrise_b200.h
	@mkdir -p hyrise_b200/lib
	$(CXX) -O3 -march=x86-64-v3 -std=c++17 -fPIC -Wall -pthread -shared -o $@ $(CSRC)/tpch_gen.cpp

oracle:
	$(MAKE) -C oracle

# The C++ host-side mirror of the reference operator interface (include/hyrise_b200.hpp) driving the three operators.
example: build/tpch_operators
build/tpch_operators: examples/tpch_operators.cpp include/hyrise_b200.hpp include/hyrise_b200.h include/hyrise_b200_tpch.h $(LIB) $(TPCH_LIB)
	@mkdir -p build
	$(CXX) -O2 -std=c++17 -Wall -Wextra -Iinclude -o $@ examples/tpch_operators.cpp -Lhyrise_b200/lib -lhyrise_b200 -lhyb_tpch \
		-Wl,-rpath,'$$ORIGIN/../hyrise_b200/lib'

# Host-only check of the mirror's predicate normalisation against the reference's own test expectations.
build/predicate_cast_check: tests/cpp/predicate_cast_check.cpp include/hyrise_b200.hpp include/hyrise_b200.h $(LIB)
	@mkdir -p build
	$(CXX) -O1 -std=c++17 -Wall -Wextra -Iinclude -o $@ tests/cpp/predicate_cast_check.cpp -Lhyrise_b200/lib -lhyrise_b200 \
		-Wl,-rpath,'$$ORIGIN/../hyrise_b200/lib'

# Column-vs-column TableScan through the mirror on the GPU (one string and one numeric comparison).
build/column_scan_check: tests/cpp/column_scan_check.cpp include/hyrise_b200.hpp include/hyrise_b200.h $(LIB)
	@mkdir -p build
	$(CXX) -O1 -std=c++17 -Wall -Wextra -Iinclude -o $@ tests/cpp/column_scan_check.cpp -Lhyrise_b200/lib -lhyrise_b200 \
		-Wl,-rpath,'$$ORIGIN/../hyrise_b200/lib'

# JoinHash with secondary predicates through the mirror on the GPU (the overload and its predicate flip).
build/join_predicates_check: tests/cpp/join_predicates_check.cpp include/hyrise_b200.hpp include/hyrise_b200.h $(LIB)
	@mkdir -p build
	$(CXX) -O1 -std=c++17 -Wall -Wextra -Iinclude -o $@ tests/cpp/join_predicates_check.cpp -Lhyrise_b200/lib -lhyrise_b200 \
		-Wl,-rpath,'$$ORIGIN/../hyrise_b200/lib'

# CPU restatement of JoinHash with secondary predicates on top of the CPU oracle's join steps (test infrastructure,
# tests/join_predicates_oracle.py). No -ffast-math: the evaluator's comparisons must follow IEEE and C++'s conversions.
$(JOIN_PREDICATES_ORACLE): tests/cpp/join_predicates_oracle.cpp oracle/oracle.cpp oracle/oracle.h include/hyrise_b200.h
	@mkdir -p build
	$(CXX) -O2 -std=c++17 -fPIC -Wall -Wextra -Wno-unused-parameter -Wno-unused-function -pthread -shared -o $@ \
		tests/cpp/join_predicates_oracle.cpp

# CPU restatement of ColumnVsColumnTableScanImpl on decoded numeric values (test infrastructure, tests/column_scan_oracle.py).
# No -ffast-math: the comparisons must follow IEEE and C++'s arithmetic conversions exactly.
$(COLUMN_SCAN_ORACLE): tests/cpp/column_scan_oracle.cpp include/hyrise_b200.h
	@mkdir -p build
	$(CXX) -O2 -std=c++17 -fPIC -Wall -Wextra -shared -o $@ tests/cpp/column_scan_oracle.cpp

# CPU restatement of the COUNT(DISTINCT) / STDDEV_SAMP accumulators (test infrastructure, tests/aggregate_distinct_oracle.py).
# No -ffast-math: NaN and signed zeros must compare as in the reference's sets.
$(AGGREGATE_DISTINCT_ORACLE): tests/cpp/aggregate_distinct_oracle.cpp include/hyrise_b200.h
	@mkdir -p build
	$(CXX) -O2 -std=c++17 -fPIC -Wall -Wextra -Iinclude -shared -o $@ tests/cpp/aggregate_distinct_oracle.cpp

# COUNT(DISTINCT) and STDDEV_SAMP through the mirror's AggregateHash on the GPU.
build/aggregate_distinct_check: tests/cpp/aggregate_distinct_check.cpp include/hyrise_b200.hpp include/hyrise_b200.h $(LIB)
	@mkdir -p build
	$(CXX) -O1 -std=c++17 -Wall -Wextra -Iinclude -o $@ tests/cpp/aggregate_distinct_check.cpp -Lhyrise_b200/lib -lhyrise_b200 \
		-Wl,-rpath,'$$ORIGIN/../hyrise_b200/lib'

# String MIN / MAX / COUNT and ANY through the mirror on the GPU, over a reference binary fixture.
build/string_aggregate_check: tests/cpp/string_aggregate_check.cpp include/hyrise_b200.hpp include/hyrise_b200.h $(LIB)
	@mkdir -p build
	$(CXX) -O1 -std=c++17 -Wall -Wextra -Iinclude -o $@ tests/cpp/string_aggregate_check.cpp -Lhyrise_b200/lib -lhyrise_b200 \
		-Wl,-rpath,'$$ORIGIN/../hyrise_b200/lib'

# CPU restatement of the ExpressionEvaluator's IN over a literal list (test infrastructure, tests/in_scan_oracle.py).
# No -ffast-math: NaN and signed zeros must compare as std::equal_to does.
$(IN_SCAN_ORACLE): tests/cpp/in_scan_oracle.cpp include/hyrise_b200.h
	@mkdir -p build
	$(CXX) -O2 -std=c++17 -fPIC -Wall -Wextra -shared -o $@ tests/cpp/in_scan_oracle.cpp

# [NOT] IN TableScans through the mirror on the GPU (a numeric and a string list).
build/in_scan_check: tests/cpp/in_scan_check.cpp include/hyrise_b200.hpp include/hyrise_b200.h $(LIB)
	@mkdir -p build
	$(CXX) -O1 -std=c++17 -Wall -Wextra -Iinclude -o $@ tests/cpp/in_scan_check.cpp -Lhyrise_b200/lib -lhyrise_b200 \
		-Wl,-rpath,'$$ORIGIN/../hyrise_b200/lib'

# CPU restatement of the ExpressionEvaluator's predicates over arithmetic operands (test infrastructure,
# tests/expression_scan_oracle.py). No -ffast-math: NaN, signed zeros, std::fmod and the conversions must follow IEEE and C++.
$(EXPRESSION_SCAN_ORACLE): tests/cpp/expression_scan_oracle.cpp include/hyrise_b200.h
	@mkdir -p build
	$(CXX) -O2 -std=c++17 -fPIC -Wall -Wextra -shared -o $@ tests/cpp/expression_scan_oracle.cpp

# Expression-predicate TableScans through the mirror on the GPU.
build/expression_scan_check: tests/cpp/expression_scan_check.cpp include/hyrise_b200.hpp include/hyrise_b200.h $(LIB)
	@mkdir -p build
	$(CXX) -O1 -std=c++17 -Wall -Wextra -Iinclude -o $@ tests/cpp/expression_scan_check.cpp -Lhyrise_b200/lib -lhyrise_b200 \
		-Wl,-rpath,'$$ORIGIN/../hyrise_b200/lib'

# Expression trees with column-test leaves through the mirror on the GPU.
build/expression_tests_check: tests/cpp/expression_tests_check.cpp include/hyrise_b200.hpp include/hyrise_b200.h $(LIB)
	@mkdir -p build
	$(CXX) -O1 -std=c++17 -Wall -Wextra -Iinclude -o $@ tests/cpp/expression_tests_check.cpp -Lhyrise_b200/lib -lhyrise_b200 \
		-Wl,-rpath,'$$ORIGIN/../hyrise_b200/lib'

# AggregateHash with an expression-tree WHERE clause through the mirror on the GPU.
build/aggregate_expression_check: tests/cpp/aggregate_expression_check.cpp include/hyrise_b200.hpp include/hyrise_b200.h $(LIB)
	@mkdir -p build
	$(CXX) -O1 -std=c++17 -Wall -Wextra -Iinclude -o $@ tests/cpp/aggregate_expression_check.cpp -Lhyrise_b200/lib -lhyrise_b200 \
		-Wl,-rpath,'$$ORIGIN/../hyrise_b200/lib'

# Sort (hyb_sort, hyb_aggregate_result_sort) through the mirror on the GPU.
build/sort_check: tests/cpp/sort_check.cpp include/hyrise_b200.hpp include/hyrise_b200.h $(LIB)
	@mkdir -p build
	$(CXX) -O1 -std=c++17 -Wall -Wextra -Iinclude -o $@ tests/cpp/sort_check.cpp -Lhyrise_b200/lib -lhyrise_b200 \
		-Wl,-rpath,'$$ORIGIN/../hyrise_b200/lib'

# AggregateOutput::to_table, a HAVING TableScan and a semi JoinHash over it through the mirror on the GPU.
build/aggregate_table_check: tests/cpp/aggregate_table_check.cpp include/hyrise_b200.hpp include/hyrise_b200.h $(LIB)
	@mkdir -p build
	$(CXX) -O1 -std=c++17 -Wall -Wextra -Iinclude -o $@ tests/cpp/aggregate_table_check.cpp -Lhyrise_b200/lib -lhyrise_b200 \
		-Wl,-rpath,'$$ORIGIN/../hyrise_b200/lib'

clean:
	rm -rf build $(LIB) $(TPCH_LIB)
	$(MAKE) -C oracle clean

.PHONY: all oracle clean example
