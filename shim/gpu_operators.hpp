#pragma once

#include <memory>
#include <vector>

#include "all_type_variant.hpp"
#include "operators/operator_join_predicate.hpp"
#include "storage/table.hpp"
#include "types.hpp"

namespace hyrise {

class AbstractExpression;
class DeviceColumnPool;
class InExpression;
class WindowFunctionExpression;

// Process-wide access for the operators (set by the plugin's start(), cleared by stop()). nullptr: no GPU path.
DeviceColumnPool* gpu_column_pool();
void set_gpu_column_pool(DeviceColumnPool* pool);

// Each returns the operator's output table, or nullptr for "not on the device path — run the CPU body"
// (hyb_status HYB_ERR_UNSUPPORTED, table not in the pool, predicate shape the ABI does not take). Any other error is Fail().

// TableScan::_on_execute (table_scan.cpp:97-240): column <condition> value | BETWEEN | IS [NOT] NULL on a stored table or on
// a reference table over one stored table.
std::shared_ptr<const Table> try_gpu_table_scan(const std::shared_ptr<const Table>& in_table, ColumnID column_id,
                                                PredicateCondition condition, const AllTypeVariant& value,
                                                const std::optional<AllTypeVariant>& value2);

// TableScan::_on_execute when create_impl would pick a ColumnVsColumnTableScanImpl (table_scan.cpp:312-452): the single
// OperatorScanPredicate compares two columns of a stored table. String columns need dictionary segments.
std::shared_ptr<const Table> try_gpu_column_scan(const std::shared_ptr<const Table>& in_table, ColumnID left_column_id,
                                                 PredicateCondition condition, ColumnID right_column_id);

// TableScan::_on_execute when create_impl would fall back to an ExpressionEvaluatorTableScanImpl for
// `<column> [NOT] IN (<literal>, ...)` (expression_evaluator.cpp:404-511): the operand is a column of a stored table and every
// list element a ValueExpression. String columns need dictionary segments. Subqueries and non-literal elements: nullptr.
std::shared_ptr<const Table> try_gpu_in_scan(const std::shared_ptr<const Table>& in_table, const InExpression& in_expression);

// TableScan::_on_execute for the numeric predicates create_impl hands to an ExpressionEvaluatorTableScanImpl
// (table_scan.cpp:312-452) and for the literals hyb_lossless_predicate_cast / hyb_lossless_between_cast cannot cast
// (`int_col > 5.5f`): comparisons, BETWEEN and IS [NOT] NULL over columns, numeric literals, NULL and + - * / %, under
// AND / OR, on a stored table. Leaves the standalone scans take (string comparisons and BETWEEN against literals, LIKE,
// IN over a literal list, numeric comparisons with a lossless literal) run as column-test leaves
// (hyb_table_scan_expression_tests). String operands, functions and anything the ABI does not take: nullptr.
std::shared_ptr<const Table> try_gpu_expression_scan(const std::shared_ptr<const Table>& in_table,
                                                     const AbstractExpression& predicate);

// JoinHash::_on_execute (join_hash.cpp:116-225), after the build/probe side selection and the radix-bit calculation.
std::shared_ptr<const Table> try_gpu_join_hash(const std::shared_ptr<const Table>& build_table,
                                               const std::shared_ptr<const Table>& probe_table, ColumnID build_column_id,
                                               ColumnID probe_column_id, JoinMode mode, size_t radix_bits,
                                               bool build_is_left_input,
                                               const std::vector<OperatorJoinPredicate>& secondary_predicates);

// AggregateHash::_on_execute (aggregate_hash.cpp:1180-1372).
std::shared_ptr<const Table> try_gpu_aggregate_hash(const std::shared_ptr<const Table>& in_table,
                                                    const std::vector<ColumnID>& groupby_column_ids,
                                                    const std::vector<std::shared_ptr<WindowFunctionExpression>>& aggregates);

// Sort::_on_execute (sort.cpp:287-516) of a stored table with ForceMaterialization::No: every definition names a column of
// that one table (the must_materialize test at :339-371 answers "no"), so the output is ReferenceSegments over the sorted
// RowIDs, cut every output_chunk_size rows. A string column's order ranks are attached on first use
// (DeviceColumnPool::ensure_string_order); when that is not possible the CPU body runs.
std::shared_ptr<const Table> try_gpu_sort(const std::shared_ptr<const Table>& in_table,
                                          const std::vector<SortColumnDefinition>& sort_definitions,
                                          ChunkOffset output_chunk_size);

}  // namespace hyrise
