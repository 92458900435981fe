// hyrise_b200.hpp — C++17 host-side mirror of the reference's operator interface for the three operators of the hot path,
// header-only, on top of the C-ABI (hyrise_b200.h). It is what a C++ caller that is not Hyrise itself uses (examples,
// tools, a standalone executor), and it documents, in compilable form, the mapping the INTEGRATION.md shims implement:
//
//   reference (hyrise/hyrise @ 2f7bedf3)                          here
//   AbstractOperator::execute() / get_output()                    Operator::execute() / typed get_output()
//     src/lib/operators/abstract_operator.hpp:72-129
//   TableScan(in, predicate)          table_scan.hpp:23-47         TableScan(context, input, ColumnVsValue / Between / IsNull)
//   JoinHash(left, right, mode, OperatorJoinPredicate, radix_bits) JoinHash(context, left, right, mode, predicate, radix_bits)
//   JoinHash(left, right, mode, primary, secondary, radix_bits)    the same with secondary predicates (hyb_join_hash_predicates)
//     join_hash.hpp:27-39, operator_join_predicate.hpp:16-44         build/probe side selection as join_hash.cpp:139-155
//   AggregateHash(in, aggregates, groupby_column_ids)             AggregateHash(context, input, aggregates, groupby_column_ids)
//     aggregate_hash.hpp:86-90, abstract_aggregate_operator.hpp
//   PredicateCondition, JoinMode, RowID, ColumnID                  same names, same numeric values (types.hpp:97-210)
//   WindowFunction                                                 same names, HYB_AGG_* values (see the enum)
//   Fail()/Assert -> std::logic_error  utils/assert.hpp:48-82      every non-zero hyb_status -> std::logic_error;
//                                                                  HYB_ERR_UNSUPPORTED -> UnsupportedOnDevice (run the CPU operator)
//
// Operators are single-use like the reference's (execute() once, then get_output()); outputs stay device-resident and
// can feed the next operator (a TableScan's PosList as the filter of a JoinHash / AggregateHash / second TableScan).
#pragma once

#include <algorithm>
#include <cstdint>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <utility>
#include <variant>
#include <vector>

#include "hyrise_b200.h"

namespace hyrise_b200 {

using ColumnID = uint32_t;
using ChunkID = uint32_t;
using RowID = hyb_row_id;                                   // types.hpp:97-117, layout-identical
using AllTypeVariant = std::variant<int32_t, int64_t, float, double>;  // the types that reach the device as values

enum class PredicateCondition : int32_t {  // types.hpp:160-179
  Equals = HYB_PRED_EQUALS,
  NotEquals = HYB_PRED_NOT_EQUALS,
  LessThan = HYB_PRED_LESS_THAN,
  LessThanEquals = HYB_PRED_LESS_THAN_EQUALS,
  GreaterThan = HYB_PRED_GREATER_THAN,
  GreaterThanEquals = HYB_PRED_GREATER_THAN_EQUALS,
  BetweenInclusive = HYB_PRED_BETWEEN_INCLUSIVE,
  BetweenLowerExclusive = HYB_PRED_BETWEEN_LOWER_EXCLUSIVE,
  BetweenUpperExclusive = HYB_PRED_BETWEEN_UPPER_EXCLUSIVE,
  BetweenExclusive = HYB_PRED_BETWEEN_EXCLUSIVE,
  In = HYB_PRED_IN,        // InList (hyb_table_scan_in) only
  NotIn = HYB_PRED_NOT_IN,  // InList (hyb_table_scan_in) only
  IsNull = HYB_PRED_IS_NULL,
  IsNotNull = HYB_PRED_IS_NOT_NULL
};

enum class JoinMode : int32_t {  // types.hpp:210
  Inner = HYB_JOIN_INNER,
  Left = HYB_JOIN_LEFT,
  Right = HYB_JOIN_RIGHT,
  FullOuter = HYB_JOIN_FULL_OUTER,
  Cross = HYB_JOIN_CROSS,
  Semi = HYB_JOIN_SEMI,
  AntiNullAsTrue = HYB_JOIN_ANTI_NULL_AS_TRUE,
  AntiNullAsFalse = HYB_JOIN_ANTI_NULL_AS_FALSE
};

// expression/window_function_expression.hpp, with the HYB_AGG_* values: these agree with the reference's numbering up to
// Count only (the reference has no CountStar, so its CountDistinct is 5 and StandardDeviationSample 6).
// Result types (WindowFunctionTraits): CountDistinct -> int64, never NULL; StandardDeviationSample -> double, NULL below
// 2 non-NULL values.
enum class WindowFunction : int32_t {
  Min = HYB_AGG_MIN,
  Max = HYB_AGG_MAX,
  Sum = HYB_AGG_SUM,
  Avg = HYB_AGG_AVG,
  Count = HYB_AGG_COUNT,
  CountStar = HYB_AGG_COUNT_STAR,
  CountDistinct = HYB_AGG_COUNT_DISTINCT,
  StandardDeviationSample = HYB_AGG_STDDEV_SAMP,
  Any = HYB_AGG_ANY  // one column, no values: the column at AggregateOutput::group_row_ids()
};

// HYB_ERR_UNSUPPORTED: the caller runs the reference's CPU operator instead (IN scans, string join keys, ...).
class UnsupportedOnDevice : public std::logic_error {
 public:
  using std::logic_error::logic_error;
};

inline void check(int status) {
  if (status == HYB_OK) return;
  const std::string message = std::string("hyb_status ") + std::to_string(status) + ": " + hyb_last_error();
  if (status == HYB_ERR_UNSUPPORTED) throw UnsupportedOnDevice(message);
  throw std::logic_error(message);  // what Fail() throws, utils/assert.hpp:48-82
}

// One per (process, GPU). Owns the device column pool and every result handle created through it.
class DeviceContext {
 public:
  explicit DeviceContext(int device_index = 0) { check(hyb_context_create(device_index, &_context)); }
  ~DeviceContext() { hyb_context_destroy(_context); }
  DeviceContext(const DeviceContext&) = delete;
  DeviceContext& operator=(const DeviceContext&) = delete;
  hyb_context* get() const { return _context; }
  void synchronize() const { check(hyb_context_synchronize(_context)); }
  hyb_operator_stats last_operator_stats() const {
    hyb_operator_stats stats{};
    check(hyb_last_operator_stats(_context, &stats));
    return stats;
  }

 private:
  hyb_context* _context = nullptr;
};

// A table file in Hyrise's binary format (BinaryParser::parse, import_export/binary/binary_parser.cpp:40-344), parsed into
// pinned host blocks in the device pool's layout. Parsing needs no GPU; DeviceTable(context, binary_table) uploads it with
// one DMA per block.
class BinaryTable {
 public:
  explicit BinaryTable(const std::string& path, bool pinned = true) { check(hyb_binary_table_open(path.c_str(), pinned ? 1 : 0, &_table)); }
  ~BinaryTable() { hyb_binary_table_close(_table); }
  BinaryTable(const BinaryTable&) = delete;
  BinaryTable& operator=(const BinaryTable&) = delete;
  const hyb_binary_table* get() const { return _table; }
  uint32_t chunk_count() const {
    uint32_t chunks = 0;
    check(hyb_binary_table_info(_table, nullptr, &chunks, nullptr));
    return chunks;
  }
  uint32_t column_count() const {
    uint32_t columns = 0;
    check(hyb_binary_table_info(_table, nullptr, nullptr, &columns));
    return columns;
  }
  std::string column_name(uint32_t column) const {
    const char* name = nullptr;
    check(hyb_binary_table_column(_table, column, &name, nullptr, nullptr));
    return name;
  }
  // hyb_scan_predicate.value_id_bounds of a string predicate: DictionarySegment::lower_bound / upper_bound per chunk
  std::vector<uint32_t> value_id_bounds(uint32_t column, const std::string& value, const std::optional<std::string>& value2 = std::nullopt) const {
    std::vector<uint32_t> bounds(size_t{chunk_count()} * (value2 ? 4 : 2));
    check(hyb_binary_table_value_id_bounds(_table, column, value.data(), value.size(), value2 ? value2->data() : nullptr,
                                           value2 ? value2->size() : 0, bounds.data()));
    return bounds;
  }
  // hyb_scan_predicate.value_id_bounds of a LIKE predicate: the per-chunk dictionary match bitmaps (LikeMatcher over every
  // chunk's dictionary, column_like_table_scan_impl.cpp:75-140)
  std::vector<uint32_t> like_value_id_bitmaps(uint32_t column, const std::string& pattern, int32_t condition) const {
    uint32_t words = 0;
    check(hyb_binary_table_like_bitmaps(_table, column, pattern.data(), pattern.size(), condition, nullptr, &words));
    std::vector<uint32_t> bitmaps(std::max<uint32_t>(words, 1));
    check(hyb_binary_table_like_bitmaps(_table, column, pattern.data(), pattern.size(), condition, bitmaps.data(), &words));
    return bitmaps;
  }
  // hyb_in_predicate.dictionary_matches of `<string column> [NOT] IN (elements)`: every chunk's dictionary entries that
  // the list holds (inverted for NotIn), by bytewise equality (hyb_in_dictionary_matches)
  std::vector<uint32_t> in_value_id_bitmaps(uint32_t column, PredicateCondition condition,
                                            const std::vector<std::string>& elements) const {
    std::string chars;
    std::vector<uint64_t> offsets{0};
    for (const auto& element : elements) {
      chars += element;
      offsets.push_back(chars.size());
    }
    const auto count = static_cast<uint32_t>(elements.size());
    const char* data = chars.empty() ? nullptr : chars.data();
    uint32_t words = 0;
    check(hyb_binary_table_in_bitmaps(_table, column, static_cast<int32_t>(condition), data, offsets.data(), count, nullptr,
                                      &words));
    std::vector<uint32_t> bitmaps(std::max<uint32_t>(words, 1));
    check(hyb_binary_table_in_bitmaps(_table, column, static_cast<int32_t>(condition), data, offsets.data(), count,
                                      bitmaps.data(), &words));
    return bitmaps;
  }
  // hyb_column_scan_predicate.right_in_left of `left <condition> right` on two string columns: every chunk's right
  // dictionary translated into its left dictionary's value-ID space (hyb_dictionary_translate)
  std::vector<uint32_t> column_translation(uint32_t left_column, uint32_t right_column) const {
    uint32_t words = 0;
    check(hyb_binary_table_column_translation(_table, left_column, right_column, nullptr, &words));
    std::vector<uint32_t> translation(std::max<uint32_t>(words, 1));
    check(hyb_binary_table_column_translation(_table, left_column, right_column, translation.data(), &words));
    return translation;
  }
  // The order ranks of a string column (hyb_binary_table_string_order_ranks): DeviceTable::set_string_order's words
  std::vector<uint32_t> string_order_ranks(uint32_t column) const {
    uint32_t words = 0;
    check(hyb_binary_table_string_order_ranks(_table, column, nullptr, &words));
    std::vector<uint32_t> ranks(std::max<uint32_t>(words, 1));
    check(hyb_binary_table_string_order_ranks(_table, column, ranks.data(), &words));
    ranks.resize(words);
    return ranks;
  }
  // One dictionary entry of a string column (a string MIN / MAX result names one).
  std::string dictionary_entry(uint32_t chunk, uint32_t column, uint32_t value_id) const {
    const char* chars = nullptr;
    const uint64_t* offsets = nullptr;
    uint32_t count = 0;
    check(hyb_binary_table_string_dictionary(_table, chunk, column, &chars, &offsets, &count));
    if (value_id >= count) throw std::out_of_range("value-ID outside the dictionary");
    return std::string(chars ? chars + offsets[value_id] : "", offsets[value_id + 1] - offsets[value_id]);
  }

 private:
  hyb_binary_table* _table = nullptr;
};

// A stored table in the device column pool (StorageManager::add_table's device twin).
class DeviceTable {
 public:
  DeviceTable(std::shared_ptr<DeviceContext> context, const hyb_table_view& view) : _context(std::move(context)) {
    check(hyb_table_upload(_context->get(), &view, &_handle));
  }
  DeviceTable(std::shared_ptr<DeviceContext> context, const BinaryTable& file) : _context(std::move(context)) {
    check(hyb_table_upload_binary(_context->get(), file.get(), &_handle));
  }
  // Takes ownership of a table the library created (AggregateOutput::to_table).
  DeviceTable(std::shared_ptr<DeviceContext> context, hyb_table_t handle) : _context(std::move(context)), _handle(handle) {}
  ~DeviceTable() { hyb_table_drop(_context->get(), _handle); }
  DeviceTable(const DeviceTable&) = delete;
  DeviceTable& operator=(const DeviceTable&) = delete;
  hyb_table_t handle() const { return _handle; }
  const std::shared_ptr<DeviceContext>& context() const { return _context; }
  // Attach the order ranks MIN / MAX over a string column need (dropped when chunks are appended).
  void set_string_order(uint32_t column, const std::vector<uint32_t>& ranks) {
    check(hyb_table_set_string_order(_context->get(), _handle, column, ranks.data(), ranks.size()));
  }
  uint64_t row_count() const {
    uint64_t rows = 0;
    check(hyb_table_info(_context->get(), _handle, nullptr, nullptr, &rows, nullptr));
    return rows;
  }
  uint32_t chunk_count() const {
    uint32_t chunks = 0;
    check(hyb_table_info(_context->get(), _handle, &chunks, nullptr, nullptr, nullptr));
    return chunks;
  }

 private:
  std::shared_ptr<DeviceContext> _context;
  hyb_table_t _handle = 0;
};

// What TableScan::get_output() references: per input chunk an ascending RowIDPosList (table_scan.cpp:199-217), device
// resident, flat with chunk boundaries.
class PosListSet {
 public:
  PosListSet(std::shared_ptr<const DeviceTable> table, hyb_pos_list_t handle) : _table(std::move(table)), _handle(handle) {}
  ~PosListSet() { hyb_pos_list_free(_table->context()->get(), _handle); }
  PosListSet(const PosListSet&) = delete;
  PosListSet& operator=(const PosListSet&) = delete;
  hyb_pos_list_t handle() const { return _handle; }
  const std::shared_ptr<const DeviceTable>& table() const { return _table; }
  uint64_t size() const {
    uint64_t total = 0;
    check(hyb_pos_list_info(_table->context()->get(), _handle, &total, nullptr));
    return total;
  }
  std::vector<uint64_t> chunk_offsets() const {  // chunk_count + 1 entries
    std::vector<uint64_t> offsets(_table->chunk_count() + 1);
    check(hyb_pos_list_chunk_offsets(_table->context()->get(), _handle, offsets.data()));
    return offsets;
  }
  std::vector<RowID> row_ids() const {
    std::vector<RowID> out(size());
    if (!out.empty()) check(hyb_pos_list_copy(_table->context()->get(), _handle, 0, out.size(), out.data()));
    return out;
  }

 private:
  std::shared_ptr<const DeviceTable> _table;
  hyb_pos_list_t _handle;
};

// An operator input: a stored table, optionally restricted to the positions a previous scan produced (a reference table
// whose segments point into the stored table, table_scan.cpp:150-197).
struct OperatorInput {
  std::shared_ptr<const DeviceTable> table;
  std::shared_ptr<const PosListSet> filter;  // may be null
  OperatorInput(std::shared_ptr<const DeviceTable> stored_table) : table(std::move(stored_table)) {}  // NOLINT
  OperatorInput(std::shared_ptr<const PosListSet> scan_output) : table(scan_output->table()), filter(std::move(scan_output)) {}  // NOLINT
  hyb_pos_list_t filter_handle() const { return filter ? filter->handle() : 0; }
};

// AbstractOperator's life cycle (abstract_operator.hpp:72-129): construct, execute() once, get_output().
template <typename Output>
class Operator {
 public:
  virtual ~Operator() = default;
  void execute() {
    if (_executed) throw std::logic_error("Operator has already been executed");  // abstract_operator.cpp:80-84
    _output = _on_execute();
    _executed = true;
  }
  bool executed() const { return _executed; }
  const std::shared_ptr<const Output>& get_output() const {
    if (!_executed) throw std::logic_error("Trying to get_output of operator which was not executed");
    return _output;
  }
  hyb_operator_stats performance_data{};  // operator_performance_data.hpp:46-97

 protected:
  virtual std::shared_ptr<const Output> _on_execute() = 0;

 private:
  bool _executed = false;
  std::shared_ptr<const Output> _output;
};

namespace detail {
inline hyb_value to_value(const AllTypeVariant& variant) {
  hyb_value value{};
  std::visit(
      [&](const auto typed) {
        using T = std::decay_t<decltype(typed)>;
        if constexpr (std::is_same_v<T, int32_t>) {
          value.i32 = typed;
        } else if constexpr (std::is_same_v<T, int64_t>) {
          value.i64 = typed;
        } else if constexpr (std::is_same_v<T, float>) {
          value.f32 = typed;
        } else {
          value.f64 = typed;
        }
      },
      variant);
  return value;
}
}  // namespace detail

enum class DataType : int32_t {  // all_type_variant.hpp:34-39, the numeric types
  Int = HYB_TYPE_INT32,
  Long = HYB_TYPE_INT64,
  Float = HYB_TYPE_FLOAT32,
  Double = HYB_TYPE_FLOAT64
};

inline DataType data_type_from_all_type_variant(const AllTypeVariant& variant) {
  return static_cast<DataType>(variant.index());  // the variant's alternatives are in DataType order
}

namespace detail {
inline AllTypeVariant to_variant(DataType type, const hyb_value& value) {
  switch (type) {
    case DataType::Int:
      return value.i32;
    case DataType::Long:
      return static_cast<int64_t>(value.i64);
    case DataType::Float:
      return value.f32;
    default:
      return value.f64;
  }
}
}  // namespace detail

// types.cpp:51-82. Throws std::logic_error (the reference's Fail) for conditions that cannot be flipped.
inline PredicateCondition flip_predicate_condition(PredicateCondition condition) {
  int32_t flipped = 0;
  check(hyb_flip_predicate_condition(static_cast<int32_t>(condition), &flipped));
  return static_cast<PredicateCondition>(flipped);
}

// lossless_predicate_variant_cast (utils/lossless_predicate_cast.hpp:64-66, .cpp:40-73): the literal in the column's type
// and the possibly adjusted condition (`float_col < 3.1` -> `float_col <= 3.0999999f`), or nullopt when no lossless form
// exists — the reference then falls back to the ExpressionEvaluator, i.e. the CPU operator runs.
inline std::optional<std::pair<PredicateCondition, AllTypeVariant>> lossless_predicate_variant_cast(
    PredicateCondition condition, const AllTypeVariant& variant, DataType target_data_type) {
  const hyb_literal literal{static_cast<int32_t>(data_type_from_all_type_variant(variant)), detail::to_value(variant)};
  int32_t adjusted = 0;
  hyb_value value{};
  const int status = hyb_lossless_predicate_cast(static_cast<int32_t>(condition), &literal, static_cast<int32_t>(target_data_type), 0,
                                                 &adjusted, &value);
  if (status == HYB_ERR_UNSUPPORTED) return std::nullopt;
  check(status);
  return std::make_pair(static_cast<PredicateCondition>(adjusted), detail::to_variant(target_data_type, value));
}

// column <condition> value | column BETWEEN lower AND upper | column IS [NOT] NULL. Values must have the column's data
// type: ScanPredicate::normalized() does what TableScan::create_impl does with a literal of another type
// (table_scan.cpp:340-366 and :399-441), through the library's hyb_lossless_predicate_cast / hyb_lossless_between_cast.
struct ScanPredicate {
  ColumnID column_id;
  PredicateCondition condition;
  std::optional<AllTypeVariant> value;   // binary conditions and the lower bound of BETWEEN
  std::optional<AllTypeVariant> value2;  // upper bound of BETWEEN
  // string dictionaries: per-chunk bounds; for the LIKE conditions the per-chunk dictionary match bitmaps
  // (BinaryTable::like_value_id_bitmaps, hyb_like_dictionary_matches); see hyb_scan_predicate
  std::vector<uint32_t> string_value_id_bounds;

  // The predicate with its literal(s) cast to `column_type`; nullopt: no lossless form (run the CPU operator).
  std::optional<ScanPredicate> normalized(DataType column_type) const {
    ScanPredicate result = *this;
    const bool between = condition >= PredicateCondition::BetweenInclusive && condition <= PredicateCondition::BetweenExclusive;
    if (between && value && value2) {
      const hyb_literal lower{static_cast<int32_t>(data_type_from_all_type_variant(*value)), detail::to_value(*value)};
      const hyb_literal upper{static_cast<int32_t>(data_type_from_all_type_variant(*value2)), detail::to_value(*value2)};
      int32_t adjusted = 0;
      hyb_value low{}, high{};
      const int status = hyb_lossless_between_cast(static_cast<int32_t>(condition), &lower, &upper, static_cast<int32_t>(column_type),
                                                   &adjusted, &low, &high);
      if (status == HYB_ERR_UNSUPPORTED) return std::nullopt;
      check(status);
      result.condition = static_cast<PredicateCondition>(adjusted);
      result.value = detail::to_variant(column_type, low);
      result.value2 = detail::to_variant(column_type, high);
    } else if (value) {
      const auto cast = lossless_predicate_variant_cast(condition, *value, column_type);
      if (!cast) return std::nullopt;
      result.condition = cast->first;
      result.value = cast->second;
    }
    return result;
  }

  hyb_scan_predicate to_abi() const {
    hyb_scan_predicate predicate{};
    predicate.column_id = column_id;
    predicate.condition = static_cast<int32_t>(condition);
    if (value) predicate.lower = detail::to_value(*value);
    if (value2) predicate.upper = detail::to_value(*value2);
    predicate.value_id_bounds = string_value_id_bounds.empty() ? nullptr : string_value_id_bounds.data();
    return predicate;
  }
};

// left column <condition> right column (ColumnVsColumnTableScanImpl): condition is one of Equals .. GreaterThanEquals.
// String pairs carry the per-chunk translation of the right dictionaries into the left ones
// (BinaryTable::column_translation, hyb_dictionary_translate); numeric pairs leave it empty.
struct ColumnComparison {
  ColumnID left_column_id;
  PredicateCondition condition;
  ColumnID right_column_id;
  std::vector<uint32_t> right_in_left;

  hyb_column_scan_predicate to_abi() const {
    hyb_column_scan_predicate predicate{};
    predicate.left_column_id = left_column_id;
    predicate.condition = static_cast<int32_t>(condition);
    predicate.right_column_id = right_column_id;
    predicate.right_in_left = right_in_left.empty() ? nullptr : right_in_left.data();
    return predicate;
  }
};

// column [NOT] IN (<literal>, ...) (ExpressionEvaluator::_evaluate_in_expression on a literal list): condition is In or
// NotIn. A numeric column takes the list's numeric literals (any numeric type, compared in the common type) and whether it
// holds a NULL; its string literals are dropped. A string column takes the dictionary bitmaps of the list's string
// literals (BinaryTable::in_value_id_bitmaps, hyb_in_dictionary_matches) and has_string_element; without a string element
// the bitmaps stay empty. The library applies the reference's rules for NULL and for lists without a compatible element.
struct InList {
  ColumnID column_id;
  PredicateCondition condition;
  std::vector<AllTypeVariant> numeric_elements;
  bool has_null_element = false;
  bool has_string_element = false;
  std::vector<uint32_t> dictionary_matches;

  hyb_in_predicate to_abi(std::vector<hyb_literal>& literals) const {
    literals.clear();
    for (const auto& element : numeric_elements) {
      literals.push_back(hyb_literal{static_cast<int32_t>(data_type_from_all_type_variant(element)), detail::to_value(element)});
    }
    if (has_string_element && dictionary_matches.empty()) {
      throw std::invalid_argument("a string IN list needs its dictionary bitmaps (BinaryTable::in_value_id_bitmaps)");
    }
    hyb_in_predicate predicate{};
    predicate.column_id = column_id;
    predicate.condition = static_cast<int32_t>(condition);
    predicate.element_count = static_cast<uint32_t>(literals.size());
    predicate.has_null_element = has_null_element;
    predicate.elements = literals.empty() ? nullptr : literals.data();
    predicate.dictionary_matches = has_string_element ? dictionary_matches.data() : nullptr;
    return predicate;
  }
};

// The numeric predicates of the ExpressionEvaluatorTableScanImpl fallback (hyb_table_scan_expression): comparisons,
// BETWEEN and IS [NOT] NULL over reverse-Polish operands of columns, literals, NULL and + - * / %, combined with AND / OR.
//   auto a_minus_b = ExpressionPredicate::operand({column(0), column(1), op(HYB_EXPR_SUB)});
//   auto predicate = ExpressionPredicate::leaf(PredicateCondition::LessThan, {a_minus_b, {literal(int32_t{0})}});
// The header's rules apply: node types, NULL propagation, NULL on a zero divisor, AND / OR as intersection / union.
// Column-test leaves take a single-column predicate or an IN list as the standalone scans do, and mix freely with the
// operand leaves (hyb_table_scan_expression_tests): ExpressionPredicate::scan(p) || ExpressionPredicate::in_list(l).
// A numeric ScanPredicate literal must have the column's type (ScanPredicate::normalized); when it has no lossless form,
// write the comparison as an operand leaf.
struct ExpressionPredicate {
  std::vector<hyb_expression_term> terms;  // postfix
  std::vector<ScanPredicate> scans;        // the HYB_TERM_SCAN leaves, in postfix order
  std::vector<InList> ins;                 // the HYB_TERM_IN leaves, in postfix order

  static hyb_expr_node column(ColumnID column_id) {
    hyb_expr_node node{};
    node.op = HYB_EXPR_COLUMN;
    node.column_id = column_id;
    return node;
  }
  static hyb_expr_node literal(const AllTypeVariant& value) {
    hyb_expr_node node{};
    node.op = HYB_EXPR_LITERAL;
    node.literal_type = static_cast<int32_t>(data_type_from_all_type_variant(value));
    node.literal = detail::to_value(value);
    return node;
  }
  static hyb_expr_node null() {
    hyb_expr_node node{};
    node.op = HYB_EXPR_NULL;
    return node;
  }
  static hyb_expr_node op(hyb_expr_op arithmetic) {
    hyb_expr_node node{};
    node.op = arithmetic;
    return node;
  }
  static std::vector<hyb_expr_node> operand(std::vector<hyb_expr_node> nodes) { return nodes; }

  // operands: = .. >=: {left, right}; BETWEEN: {value, lower, upper}; IS [NOT] NULL: {operand}. An operand longer than
  // HYB_MAX_EXPR_NODES does not fit the ABI: UnsupportedOnDevice, as the library answers.
  static ExpressionPredicate leaf(PredicateCondition condition, const std::vector<std::vector<hyb_expr_node>>& operands) {
    if (operands.size() > 3) throw std::invalid_argument("a leaf takes at most three operands");
    hyb_expression_term term{};
    term.kind = HYB_TERM_LEAF;
    term.condition = static_cast<int32_t>(condition);
    for (size_t slot = 0; slot < operands.size(); ++slot) {
      if (operands[slot].size() > HYB_MAX_EXPR_NODES) throw UnsupportedOnDevice("operand longer than HYB_MAX_EXPR_NODES");
      std::copy(operands[slot].begin(), operands[slot].end(), term.operands[slot]);
      term.node_counts[slot] = static_cast<uint32_t>(operands[slot].size());
    }
    return {{term}, {}, {}};
  }
  static ExpressionPredicate scan(ScanPredicate predicate) {
    hyb_expression_term term{};
    term.kind = HYB_TERM_SCAN;
    return {{term}, {std::move(predicate)}, {}};
  }
  static ExpressionPredicate in_list(InList list) {
    hyb_expression_term term{};
    term.kind = HYB_TERM_IN;
    return {{term}, {}, {std::move(list)}};
  }
  bool has_tests() const { return !scans.empty() || !ins.empty(); }
  ExpressionPredicate operator&&(const ExpressionPredicate& other) const { return combine(other, HYB_TERM_AND); }
  ExpressionPredicate operator||(const ExpressionPredicate& other) const { return combine(other, HYB_TERM_OR); }

  hyb_expression_scan_predicate to_abi() const {
    hyb_expression_scan_predicate predicate{};
    predicate.term_count = static_cast<uint32_t>(terms.size());
    predicate.terms = terms.data();
    return predicate;
  }

 private:
  ExpressionPredicate combine(const ExpressionPredicate& other, hyb_expression_term_kind kind) const {
    ExpressionPredicate out{terms, scans, ins};
    out.terms.insert(out.terms.end(), other.terms.begin(), other.terms.end());
    out.scans.insert(out.scans.end(), other.scans.begin(), other.scans.end());
    out.ins.insert(out.ins.end(), other.ins.begin(), other.ins.end());
    hyb_expression_term node{};
    node.kind = kind;
    out.terms.push_back(node);
    return out;
  }
};

class TableScan : public Operator<PosListSet> {
 public:
  TableScan(OperatorInput input, ScanPredicate predicate) : _input(std::move(input)), _predicate(std::move(predicate)) {}
  TableScan(OperatorInput input, ColumnComparison comparison)
      : _input(std::move(input)), _comparison(std::move(comparison)) {}
  TableScan(OperatorInput input, InList in_list) : _input(std::move(input)), _in_list(std::move(in_list)) {}
  TableScan(OperatorInput input, ExpressionPredicate expression)
      : _input(std::move(input)), _expression(std::move(expression)) {}

 protected:
  std::shared_ptr<const PosListSet> _on_execute() override {
    hyb_context* context = _input.table->context()->get();
    hyb_pos_list_t handle = 0;
    if (_comparison) {
      const auto abi = _comparison->to_abi();
      check(hyb_table_scan_columns(context, _input.table->handle(), &abi, _input.filter_handle(), &handle));
    } else if (_expression && _expression->has_tests()) {
      const auto abi = _expression->to_abi();
      std::vector<hyb_scan_predicate> scans;
      for (const auto& scan : _expression->scans) scans.push_back(scan.to_abi());
      std::vector<std::vector<hyb_literal>> literals(_expression->ins.size());
      std::vector<hyb_in_predicate> ins;
      for (size_t i = 0; i < _expression->ins.size(); ++i) ins.push_back(_expression->ins[i].to_abi(literals[i]));
      const hyb_expression_leaf_tests tests{static_cast<uint32_t>(scans.size()), static_cast<uint32_t>(ins.size()),
                                            scans.data(), ins.data()};
      check(hyb_table_scan_expression_tests(context, _input.table->handle(), &abi, &tests, _input.filter_handle(), &handle));
    } else if (_expression) {
      const auto abi = _expression->to_abi();
      check(hyb_table_scan_expression(context, _input.table->handle(), &abi, _input.filter_handle(), &handle));
    } else if (_in_list) {
      std::vector<hyb_literal> literals;
      const auto abi = _in_list->to_abi(literals);
      check(hyb_table_scan_in(context, _input.table->handle(), &abi, _input.filter_handle(), &handle));
    } else {
      const auto abi = _predicate->to_abi();
      check(hyb_table_scan(context, _input.table->handle(), &abi, _input.filter_handle(), &handle));
    }
    check(hyb_last_operator_stats(context, &performance_data));
    return std::make_shared<PosListSet>(_input.table, handle);
  }

 private:
  OperatorInput _input;
  std::optional<ScanPredicate> _predicate;
  std::optional<ColumnComparison> _comparison;
  std::optional<InList> _in_list;
  std::optional<ExpressionPredicate> _expression;
};

// operator_join_predicate.hpp:16-44 — JoinHash supports exactly one equality predicate on the device.
struct OperatorJoinPredicate {
  std::pair<ColumnID, ColumnID> column_ids;  // {left, right}
  PredicateCondition predicate_condition = PredicateCondition::Equals;
};

// The PosList pairs JoinHash emits, in the reference's order: grouped by hash(key) & (2^radix_bits - 1), inside a
// partition in probe-row order, for one probe row in build-row order (join_hash_steps.hpp:624-792).
class JoinOutput {
 public:
  JoinOutput(std::shared_ptr<DeviceContext> context, hyb_join_result_t handle, bool left_is_build, bool has_build_side)
      : left_is_build(left_is_build), _context(std::move(context)), _handle(handle), _has_build_side(has_build_side) {}
  ~JoinOutput() { hyb_join_result_free(_context->get(), _handle); }
  JoinOutput(const JoinOutput&) = delete;
  JoinOutput& operator=(const JoinOutput&) = delete;
  uint64_t size() const {
    uint64_t pairs = 0;
    check(hyb_join_result_info(_context->get(), _handle, &pairs, nullptr, nullptr));
    return pairs;
  }
  int32_t radix_bits() const {
    int32_t bits = 0;
    check(hyb_join_result_info(_context->get(), _handle, nullptr, nullptr, &bits));
    return bits;
  }
  std::vector<uint64_t> partition_offsets() const {
    uint32_t partitions = 0;
    check(hyb_join_result_info(_context->get(), _handle, nullptr, &partitions, nullptr));
    std::vector<uint64_t> offsets(partitions + 1);
    check(hyb_join_result_partition_offsets(_context->get(), _handle, offsets.data()));
    return offsets;
  }
  // {build-side RowIDs (empty for Semi/Anti), probe-side RowIDs}
  std::pair<std::vector<RowID>, std::vector<RowID>> row_ids() const {
    const auto count = size();
    std::vector<RowID> build(_has_build_side ? count : 0), probe(count);
    if (count) {
      check(hyb_join_result_copy(_context->get(), _handle, 0, count, _has_build_side ? build.data() : nullptr, probe.data()));
    }
    return {std::move(build), std::move(probe)};
  }
  const bool left_is_build;  // which input the build-side RowIDs refer to

 private:
  std::shared_ptr<DeviceContext> _context;
  hyb_join_result_t _handle;
  bool _has_build_side;
};

class JoinHash : public Operator<JoinOutput> {
 public:
  JoinHash(OperatorInput left, OperatorInput right, JoinMode mode, OperatorJoinPredicate primary_predicate,
           std::optional<int32_t> radix_bits = std::nullopt)
      : _left(std::move(left)), _right(std::move(right)), _mode(mode), _predicate(primary_predicate), _radix_bits(radix_bits) {
    if (_predicate.predicate_condition != PredicateCondition::Equals) {
      throw std::logic_error("JoinHash only supports equi joins");  // join_hash.cpp:60-63
    }
  }
  // join_hash.hpp:35: secondary predicates `left <condition> right` after the primary equality (hyb_join_hash_predicates).
  // Flipped with the inputs when the right input builds (join_hash.cpp:158-165); UnsupportedOnDevice where the library
  // answers HYB_ERR_UNSUPPORTED (string pairs, AntiNullAsTrue, more than HYB_MAX_JOIN_PREDICATES).
  JoinHash(OperatorInput left, OperatorInput right, JoinMode mode, OperatorJoinPredicate primary_predicate,
           std::vector<OperatorJoinPredicate> secondary_predicates, std::optional<int32_t> radix_bits = std::nullopt)
      : JoinHash(std::move(left), std::move(right), mode, primary_predicate, radix_bits) {
    _secondary = std::move(secondary_predicates);
  }

 protected:
  std::shared_ptr<const JoinOutput> _on_execute() override {
    hyb_context* context = _left.table->context()->get();
    // Build side = the smaller input for Inner joins, the right input for every other mode (join_hash.cpp:139-155).
    uint64_t left_rows = 0, right_rows = 0;
    const hyb_join_side left{_left.table->handle(), _predicate.column_ids.first, _left.filter_handle()};
    const hyb_join_side right{_right.table->handle(), _predicate.column_ids.second, _right.filter_handle()};
    check(hyb_join_side_positions(context, &left, &left_rows));
    check(hyb_join_side_positions(context, &right, &right_rows));
    const bool left_is_build = _mode == JoinMode::Inner && left_rows <= right_rows;
    const hyb_join_side& build = left_is_build ? left : right;
    const hyb_join_side& probe = left_is_build ? right : left;
    hyb_join_result_t handle = 0;
    if (_secondary.empty()) {
      check(hyb_join_hash(context, &build, &probe, static_cast<int32_t>(_mode), _radix_bits.value_or(-1), &handle));
    } else {
      std::vector<hyb_join_predicate> adjusted;
      for (const auto& predicate : _secondary) {
        const auto [left_column, right_column] = predicate.column_ids;
        adjusted.push_back(left_is_build ? hyb_join_predicate{left_column, right_column, static_cast<int32_t>(predicate.predicate_condition), 0}
                                         : hyb_join_predicate{right_column, left_column,
                                                              static_cast<int32_t>(flip_predicate_condition(predicate.predicate_condition)), 0});
      }
      check(hyb_join_hash_predicates(context, &build, &probe, static_cast<int32_t>(_mode), _radix_bits.value_or(-1), adjusted.data(),
                                     static_cast<uint32_t>(adjusted.size()), &handle));
    }
    check(hyb_last_operator_stats(context, &performance_data));
    const bool semi_or_anti = _mode == JoinMode::Semi || _mode == JoinMode::AntiNullAsTrue || _mode == JoinMode::AntiNullAsFalse;
    return std::make_shared<JoinOutput>(_left.table->context(), handle, left_is_build, !semi_or_anti);
  }

 private:
  OperatorInput _left, _right;
  JoinMode _mode;
  OperatorJoinPredicate _predicate;
  std::vector<OperatorJoinPredicate> _secondary;
  std::optional<int32_t> _radix_bits;
};

// ---- multi-GPU (one process per GPU) --------------------------------------------------------------------------------------
// hyb_peer_group: this rank's exchange arena plus the mappings of its peers' arenas. The host transport (MPI, torch.distributed,
// sockets ...) is only needed once, to all-gather the HYB_IPC_HANDLE_BYTES-byte handles.
class PeerGroup {
 public:
  PeerGroup(std::shared_ptr<DeviceContext> context, uint32_t rank, uint32_t world, uint64_t tuple_capacity)
      : _context(std::move(context)), _rank(rank), _world(world), _ipc_handle(HYB_IPC_HANDLE_BYTES) {
    check(hyb_peer_group_create(_context->get(), rank, world, tuple_capacity, _ipc_handle.data(), &_handle));
  }
  ~PeerGroup() { hyb_peer_group_destroy(_context->get(), _handle); }
  PeerGroup(const PeerGroup&) = delete;
  PeerGroup& operator=(const PeerGroup&) = delete;
  const std::vector<unsigned char>& ipc_handle() const { return _ipc_handle; }  // all-gather these, in rank order ...
  void connect(const std::vector<unsigned char>& all_ipc_handles) {             // ... and hand the concatenation back
    if (all_ipc_handles.size() != size_t{_world} * HYB_IPC_HANDLE_BYTES) throw std::logic_error("world x HYB_IPC_HANDLE_BYTES bytes expected");
    check(hyb_peer_group_connect(_context->get(), _handle, all_ipc_handles.data()));
  }
  hyb_peer_group_t handle() const { return _handle; }
  uint32_t rank() const { return _rank; }
  uint32_t world() const { return _world; }
  const std::shared_ptr<DeviceContext>& context() const { return _context; }
  hyb_distributed_stats stats() const {
    hyb_distributed_stats stats{};
    check(hyb_peer_group_stats(_context->get(), _handle, &stats));
    return stats;
  }

 private:
  std::shared_ptr<DeviceContext> _context;
  uint32_t _rank, _world;
  std::vector<unsigned char> _ipc_handle;
  hyb_peer_group_t _handle = 0;
};

// Inner JoinHash over the shards of all ranks (hyb_join_hash_distributed): `build` / `probe` are this rank's shards, the chunk
// bases the global ids of their first chunks. get_output() holds GLOBAL RowIDs; stats().colocated tells the layout (1: this
// rank's slice of every partition, 0: the partitions p with p % world == rank).
class DistributedJoinHash : public Operator<JoinOutput> {
 public:
  DistributedJoinHash(std::shared_ptr<PeerGroup> group, OperatorInput build, OperatorInput probe, OperatorJoinPredicate predicate,
                      ChunkID build_chunk_base, ChunkID probe_chunk_base, std::optional<int32_t> radix_bits = std::nullopt)
      : _group(std::move(group)), _build(std::move(build)), _probe(std::move(probe)), _predicate(predicate),
        _build_chunk_base(build_chunk_base), _probe_chunk_base(probe_chunk_base), _radix_bits(radix_bits) {}

 protected:
  std::shared_ptr<const JoinOutput> _on_execute() override {
    hyb_context* context = _group->context()->get();
    const hyb_join_side build{_build.table->handle(), _predicate.column_ids.first, _build.filter_handle()};
    const hyb_join_side probe{_probe.table->handle(), _predicate.column_ids.second, _probe.filter_handle()};
    hyb_join_result_t handle = 0;
    check(hyb_join_hash_distributed(context, _group->handle(), &build, &probe, _build_chunk_base, _probe_chunk_base,
                                    _radix_bits.value_or(-1), &handle));
    check(hyb_last_operator_stats(context, &performance_data));
    return std::make_shared<JoinOutput>(_group->context(), handle, /*left_is_build=*/true, /*emits_build_side=*/true);
  }

 private:
  std::shared_ptr<PeerGroup> _group;
  OperatorInput _build, _probe;
  OperatorJoinPredicate _predicate;
  ChunkID _build_chunk_base, _probe_chunk_base;
  std::optional<int32_t> _radix_bits;
};

// An aggregate over a column, or over arithmetic on columns the reference would evaluate in a Projection below the
// aggregate (fused here). COUNT(*) has no argument (INVALID_COLUMN_ID in the reference).
struct AggregateDefinition {
  WindowFunction function;
  std::vector<hyb_expr_node> argument;  // reverse Polish; one COLUMN node for a plain column

  static AggregateDefinition on_column(WindowFunction function, ColumnID column_id) {
    hyb_expr_node node{};
    node.op = HYB_EXPR_COLUMN;
    node.column_id = column_id;
    return {function, {node}};
  }
  static AggregateDefinition count_star() { return {WindowFunction::CountStar, {}}; }
};

class AggregateOutput {
 public:
  AggregateOutput(std::shared_ptr<DeviceContext> context, hyb_aggregate_result_t handle) : _context(std::move(context)), _handle(handle) {}
  ~AggregateOutput() { hyb_aggregate_result_free(_context->get(), _handle); }
  AggregateOutput(const AggregateOutput&) = delete;
  AggregateOutput& operator=(const AggregateOutput&) = delete;
  uint64_t group_count() const {
    uint64_t groups = 0;
    check(hyb_aggregate_result_info(_context->get(), _handle, &groups, nullptr));
    return groups;
  }
  // One representative row per group, in the reference's group order (aggregate_hash.cpp:367,394,421-537).
  std::vector<RowID> group_row_ids() const {
    std::vector<RowID> rows(group_count());
    if (!rows.empty()) check(hyb_aggregate_result_row_ids(_context->get(), _handle, rows.data()));
    return rows;
  }
  // Values of one aggregate as doubles (the result type per WindowFunctionTraits is returned in *value_type) + NULL flags.
  std::pair<std::vector<double>, std::vector<uint8_t>> values(uint32_t aggregate_index, int32_t* value_type = nullptr) const {
    const auto groups = group_count();
    std::vector<uint64_t> raw(groups);
    std::vector<uint8_t> nulls(groups);
    int32_t type = 0;
    if (groups) check(hyb_aggregate_result_values(_context->get(), _handle, aggregate_index, raw.data(), nulls.data(), &type));
    std::vector<double> out(groups);
    for (uint64_t g = 0; g < groups; ++g) {
      const void* cell = type == HYB_TYPE_INT32 || type == HYB_TYPE_FLOAT32
                             ? static_cast<const void*>(reinterpret_cast<const uint32_t*>(raw.data()) + g)
                             : static_cast<const void*>(raw.data() + g);
      switch (type) {
        case HYB_TYPE_INT32:
          out[g] = *static_cast<const int32_t*>(cell);
          break;
        case HYB_TYPE_INT64:
          out[g] = static_cast<double>(*static_cast<const int64_t*>(cell));
          break;
        case HYB_TYPE_FLOAT32:
          out[g] = *static_cast<const float*>(cell);
          break;
        default:
          out[g] = *static_cast<const double*>(cell);
          break;
      }
    }
    if (value_type) *value_type = type;
    return {std::move(out), std::move(nulls)};
  }
  // Sort over the groups (hyb_aggregate_result_sort): every group index in sorted order; LIMIT k is the first k.
  std::vector<uint32_t> sorted_group_indexes(const std::vector<hyb_aggregate_sort_key>& keys) const {
    std::vector<uint32_t> out(group_count());
    check(hyb_aggregate_result_sort(_context->get(), _handle, keys.data(), static_cast<uint32_t>(keys.size()), out.data()));
    return out;
  }
  // The output as a stored table (hyb_aggregate_result_table): column c = columns[c], an aggregate or a column of the
  // aggregated table at the representative rows. A HAVING is a TableScan over it, an IN subquery a semi JoinHash onto
  // it. The table lives on after this output and the aggregated table are gone.
  std::shared_ptr<DeviceTable> to_table(const std::vector<hyb_aggregate_output_column>& columns,
                                        uint32_t chunk_size = HYB_DEFAULT_CHUNK_SIZE) const {
    hyb_table_t table = 0;
    check(hyb_aggregate_result_table(_context->get(), _handle, columns.data(), static_cast<uint32_t>(columns.size()),
                                     chunk_size, &table));
    return std::make_shared<DeviceTable>(_context, table);
  }
  // A string MIN / MAX: per group the string (std::nullopt for NULL), read from the table the aggregate ran on.
  std::vector<std::optional<std::string>> strings(uint32_t aggregate_index, const BinaryTable& table, uint32_t column) const {
    const auto groups = group_count();
    std::vector<hyb_dictionary_position> positions(groups);
    std::vector<uint8_t> nulls(groups);
    int32_t type = 0;
    if (groups) check(hyb_aggregate_result_values(_context->get(), _handle, aggregate_index, positions.data(), nulls.data(), &type));
    if (groups && type != HYB_TYPE_STRING) throw std::invalid_argument("not a string aggregate");
    std::vector<std::optional<std::string>> out(groups);
    for (uint64_t g = 0; g < groups; ++g) {
      if (!nulls[g]) out[g] = table.dictionary_entry(positions[g].chunk_id, column, positions[g].value_id);
    }
    return out;
  }

 private:
  std::shared_ptr<DeviceContext> _context;
  hyb_aggregate_result_t _handle;
};

class AggregateHash : public Operator<AggregateOutput> {
 public:
  // `fused_predicates`: conjunctive scans the optimizer placed directly below the aggregate (TPC-H Q1/Q6 shape); they are
  // evaluated inside the aggregation kernel instead of materialising a PosList first.
  AggregateHash(OperatorInput input, std::vector<AggregateDefinition> aggregates, std::vector<ColumnID> groupby_column_ids,
                std::vector<ScanPredicate> fused_predicates = {})
      : _input(std::move(input)),
        _aggregates(std::move(aggregates)),
        _groupby_column_ids(std::move(groupby_column_ids)),
        _fused_predicates(std::move(fused_predicates)) {}
  // `expression`: an ExpressionEvaluator tree (AND / OR over operand, scan and IN leaves) the optimizer placed below the
  // aggregate, evaluated inside the aggregation kernel with the fused predicates (hyb_aggregate_hash_expression).
  AggregateHash(OperatorInput input, std::vector<AggregateDefinition> aggregates, std::vector<ColumnID> groupby_column_ids,
                ExpressionPredicate expression, std::vector<ScanPredicate> fused_predicates = {})
      : _input(std::move(input)),
        _aggregates(std::move(aggregates)),
        _groupby_column_ids(std::move(groupby_column_ids)),
        _fused_predicates(std::move(fused_predicates)),
        _expression(std::move(expression)) {}

 protected:
  std::shared_ptr<const AggregateOutput> _on_execute() override {
    std::vector<hyb_aggregate_def> definitions(_aggregates.size());
    for (size_t index = 0; index < _aggregates.size(); ++index) {
      const auto& aggregate = _aggregates[index];
      if (aggregate.argument.size() > HYB_MAX_EXPR_NODES) throw UnsupportedOnDevice("aggregate argument too long");
      definitions[index].function = static_cast<int32_t>(aggregate.function);
      definitions[index].node_count = static_cast<uint32_t>(aggregate.argument.size());
      for (size_t node = 0; node < aggregate.argument.size(); ++node) definitions[index].nodes[node] = aggregate.argument[node];
    }
    std::vector<hyb_scan_predicate> predicates;
    predicates.reserve(_fused_predicates.size());
    for (const auto& predicate : _fused_predicates) predicates.push_back(predicate.to_abi());
    hyb_aggregate_query query{};
    query.table = _input.table->handle();
    query.filter = _input.filter_handle();
    query.predicate_count = static_cast<uint32_t>(predicates.size());
    query.predicates = predicates.data();
    query.groupby_count = static_cast<uint32_t>(_groupby_column_ids.size());
    query.groupby_column_ids = _groupby_column_ids.data();
    query.aggregate_count = static_cast<uint32_t>(definitions.size());
    query.aggregates = definitions.data();
    hyb_context* context = _input.table->context()->get();
    hyb_aggregate_result_t handle = 0;
    if (_expression) {
      if (_group) throw UnsupportedOnDevice("distributed aggregation with an expression predicate");
      const auto abi = _expression->to_abi();
      std::vector<hyb_scan_predicate> scans;
      for (const auto& scan : _expression->scans) scans.push_back(scan.to_abi());
      std::vector<std::vector<hyb_literal>> literals(_expression->ins.size());
      std::vector<hyb_in_predicate> ins;
      for (size_t i = 0; i < _expression->ins.size(); ++i) ins.push_back(_expression->ins[i].to_abi(literals[i]));
      const hyb_expression_leaf_tests tests{static_cast<uint32_t>(scans.size()), static_cast<uint32_t>(ins.size()),
                                            scans.data(), ins.data()};
      check(hyb_aggregate_hash_expression(context, &query, &abi, _expression->has_tests() ? &tests : nullptr, &handle));
    } else if (_group) {
      // every rank aggregates its shard; low cardinality: every rank gets the complete result, high cardinality: the groups
      // this rank owns (PeerGroup::stats().aggregate_partitioned)
      check(hyb_aggregate_hash_distributed(context, _group->handle(), &query, _chunk_id_base, _position_base, &handle));
    } else {
      check(hyb_aggregate_hash(context, &query, &handle));
    }
    check(hyb_last_operator_stats(context, &performance_data));
    return std::make_shared<AggregateOutput>(_input.table->context(), handle);
  }

 public:
  // Multi-GPU: `input` is this rank's shard; chunk_id_base = global id of its first chunk, position_base = rows of the global
  // table before it (call before execute()).
  void set_peer_group(std::shared_ptr<PeerGroup> group, ChunkID chunk_id_base, uint64_t position_base) {
    _group = std::move(group);
    _chunk_id_base = chunk_id_base;
    _position_base = position_base;
  }

 private:
  OperatorInput _input;
  std::vector<AggregateDefinition> _aggregates;
  std::vector<ColumnID> _groupby_column_ids;
  std::vector<ScanPredicate> _fused_predicates;
  std::optional<ExpressionPredicate> _expression;
  std::shared_ptr<PeerGroup> _group;
  ChunkID _chunk_id_base = 0;
  uint64_t _position_base = 0;
};

// sort_definition.hpp: the two modes the Sort operator accepts (sort.cpp:294-296 asserts the NULLS LAST ones away).
enum class SortMode : int32_t { AscendingNullsFirst = 0, DescendingNullsFirst = 1 };
struct SortColumnDefinition {
  ColumnID column;
  SortMode sort_mode = SortMode::AscendingNullsFirst;
};

// Sort (operators/sort.cpp:287-516) of a stored table or of a scan / join output on it. The output references the input's
// table: one PosList in sorted order. Every definition names one column of that one table, the reference's own
// must_materialize test (:339-371) answered "no"; materialised output and output chunk sizes stay with the caller.
class Sort : public Operator<PosListSet> {
 public:
  Sort(OperatorInput input, std::vector<SortColumnDefinition> definitions)
      : _input(std::move(input)), _definitions(std::move(definitions)) {}

 protected:
  std::shared_ptr<const PosListSet> _on_execute() override {
    std::vector<hyb_sort_column> columns;
    for (const auto& definition : _definitions) {
      columns.push_back(hyb_sort_column{definition.column, definition.sort_mode == SortMode::DescendingNullsFirst ? 1 : 0});
    }
    hyb_context* context = _input.table->context()->get();
    hyb_pos_list_t handle = 0;
    check(hyb_sort(context, _input.table->handle(), _input.filter_handle(), columns.data(),
                   static_cast<uint32_t>(columns.size()), &handle));
    check(hyb_last_operator_stats(context, &performance_data));
    return std::make_shared<PosListSet>(_input.table, handle);
  }

 private:
  OperatorInput _input;
  std::vector<SortColumnDefinition> _definitions;
};

}  // namespace hyrise_b200
