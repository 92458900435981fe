#pragma once

#include <memory>
#include <vector>

#include "all_type_variant.hpp"
#include "operators/operator_join_predicate.hpp"
#include "storage/table.hpp"
#include "types.hpp"

namespace hyrise {

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

// JoinHash::_on_execute (join_hash.cpp:116-225), after the build/probe side selection and the radix-bit calculation.
std::shared_ptr<const Table> try_gpu_join_hash(const std::shared_ptr<const Table>& build_table,
                                               const std::shared_ptr<const Table>& probe_table, ColumnID build_column_id,
                                               ColumnID probe_column_id, JoinMode mode, size_t radix_bits,
                                               bool build_is_left_input);

// AggregateHash::_on_execute (aggregate_hash.cpp:1180-1372).
std::shared_ptr<const Table> try_gpu_aggregate_hash(const std::shared_ptr<const Table>& in_table,
                                                    const std::vector<ColumnID>& groupby_column_ids,
                                                    const std::vector<std::shared_ptr<WindowFunctionExpression>>& aggregates);

}  // namespace hyrise
