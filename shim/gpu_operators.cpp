#include "gpu_operators.hpp"

#include <algorithm>
#include <atomic>
#include <deque>

#include "device_column_pool.hpp"
#include "expression/arithmetic_expression.hpp"
#include "expression/between_expression.hpp"
#include "expression/binary_predicate_expression.hpp"
#include "expression/evaluation/like_matcher.hpp"
#include "expression/expression_utils.hpp"
#include "expression/in_expression.hpp"
#include "expression/is_null_expression.hpp"
#include "expression/list_expression.hpp"
#include "expression/logical_expression.hpp"
#include "expression/pqp_column_expression.hpp"
#include "expression/value_expression.hpp"
#include "expression/window_function_expression.hpp"
#include "hyrise_b200.h"
#include "operators/join_helper/join_output_writing.hpp"
#include "resolve_type.hpp"
#include "storage/dictionary_segment.hpp"
#include "storage/fixed_string_dictionary_segment.hpp"
#include "storage/pos_lists/row_id_pos_list.hpp"
#include "storage/reference_segment.hpp"
#include "storage/value_segment.hpp"
#include "utils/assert.hpp"
#include "utils/lossless_predicate_cast.hpp"

namespace hyrise {

namespace {

std::atomic<DeviceColumnPool*> global_pool{nullptr};

static_assert(sizeof(RowID) == sizeof(hyb_row_id), "RowID {ChunkID, ChunkOffset} and hyb_row_id share their layout (types.hpp:97-117)");

// DataType is {Null, Int, Long, Float, Double, String} (all_type_variant.hpp:52); hyb_data_type starts at Int.
int32_t hyb_type(DataType data_type) {
  return static_cast<int32_t>(data_type) - 1;
}

hyb_value to_hyb_value(const AllTypeVariant& variant, DataType column_type) {
  auto value = hyb_value{};
  switch (column_type) {
    case DataType::Int:
      value.i32 = boost::get<int32_t>(variant);
      break;
    case DataType::Long:
      value.i64 = boost::get<int64_t>(variant);
      break;
    case DataType::Float:
      value.f32 = boost::get<float>(variant);
      break;
    case DataType::Double:
      value.f64 = boost::get<double>(variant);
      break;
    default:
      Fail("string literals travel as value-ID bounds");
  }
  return value;
}

// DictionarySegment::lower_bound / upper_bound per chunk (dictionary_segment.cpp:94-119): what the reference's dictionary scan
// does at the start of every chunk (column_vs_value_table_scan_impl.cpp:63-139), here once per call for all chunks.
bool string_value_id_bounds(const Table& stored, ColumnID column_id, const AllTypeVariant& value,
                            const std::optional<AllTypeVariant>& value2, std::vector<uint32_t>& bounds) {
  const auto chunk_count = stored.chunk_count();
  const auto values = value2 ? 2u : 1u;
  bounds.resize(size_t{chunk_count} * values * 2);
  for (auto chunk_id = ChunkID{0}; chunk_id < chunk_count; ++chunk_id) {
    const auto segment = std::dynamic_pointer_cast<const BaseDictionarySegment>(stored.get_chunk(chunk_id)->get_segment(column_id));
    if (!segment) {
      return false;
    }
    auto* out = bounds.data() + size_t{chunk_id} * values * 2;
    out[0] = segment->lower_bound(value);
    out[1] = segment->upper_bound(value);
    if (value2) {
      out[2] = segment->lower_bound(*value2);
      out[3] = segment->upper_bound(*value2);
    }
  }
  return true;
}

// ColumnLikeTableScanImpl's dictionary path (column_like_table_scan_impl.cpp:75-140) for every chunk at once: the
// reference's own LikeMatcher over each dictionary, one bit per entry, ceil(size / 32) words per chunk in chunk order.
bool like_dictionary_bitmaps(const Table& stored, ColumnID column_id, PredicateCondition condition, const pmr_string& pattern,
                             std::vector<uint32_t>& words) {
  const auto matcher = LikeMatcher{pattern, condition};
  for (auto chunk_id = ChunkID{0}; chunk_id < stored.chunk_count(); ++chunk_id) {
    const auto segment = stored.get_chunk(chunk_id)->get_segment(column_id);
    const auto append = [&](const size_t size, const auto& entry_at) {
      const auto first = words.size();
      words.resize(first + (size + 31) / 32, 0);
      matcher.resolve([&](const auto& predicate) {
        for (auto entry = size_t{0}; entry < size; ++entry) {
          words[first + entry / 32] |= predicate(entry_at(entry)) ? (1u << (entry % 32)) : 0u;
        }
      });
    };
    if (const auto dictionary_segment = std::dynamic_pointer_cast<const DictionarySegment<pmr_string>>(segment)) {
      const auto& dictionary = *dictionary_segment->dictionary();
      append(dictionary.size(), [&](const size_t entry) -> const pmr_string& { return dictionary[entry]; });
    } else if (const auto fixed_segment = std::dynamic_pointer_cast<const FixedStringDictionarySegment<pmr_string>>(segment)) {
      const auto& dictionary = *fixed_segment->fixed_string_dictionary();
      append(dictionary.size(), [&](const size_t entry) { return dictionary.get_string_at(entry); });
    } else {
      return false;
    }
  }
  return true;
}

// hyb_column_scan_predicate.right_in_left: per chunk, every right dictionary entry as 2 * lower_bound in the left dictionary
// + (found ? 1 : 0), one merge of the two sorted dictionaries; one word per right entry, chunk after chunk. Only
// DictionarySegment<pmr_string> / FixedStringDictionarySegment dictionaries (false: the CPU operator runs).
// The sorted dictionary of a string segment (DictionarySegment<pmr_string> or FixedStringDictionarySegment), or nullopt.
std::optional<std::vector<pmr_string>> string_dictionary(const Table& stored, const ChunkID chunk_id, const ColumnID column_id) {
  const auto segment = stored.get_chunk(chunk_id)->get_segment(column_id);
  if (const auto dictionary_segment = std::dynamic_pointer_cast<const DictionarySegment<pmr_string>>(segment)) {
    const auto& dictionary = *dictionary_segment->dictionary();
    return std::vector<pmr_string>(dictionary.begin(), dictionary.end());
  }
  if (const auto fixed_segment = std::dynamic_pointer_cast<const FixedStringDictionarySegment<pmr_string>>(segment)) {
    const auto& dictionary = *fixed_segment->fixed_string_dictionary();
    auto entries = std::vector<pmr_string>{};
    entries.reserve(dictionary.size());
    for (auto entry = size_t{0}; entry < dictionary.size(); ++entry) {
      entries.emplace_back(dictionary.get_string_at(entry));
    }
    return entries;
  }
  return std::nullopt;
}

bool column_translation(const Table& stored, ColumnID left_column_id, ColumnID right_column_id, std::vector<uint32_t>& words) {
  const auto dictionary_of = [&](const ChunkID chunk_id, const ColumnID column_id) {
    return string_dictionary(stored, chunk_id, column_id);
  };
  for (auto chunk_id = ChunkID{0}; chunk_id < stored.chunk_count(); ++chunk_id) {
    const auto left = dictionary_of(chunk_id, left_column_id);
    const auto right = dictionary_of(chunk_id, right_column_id);
    if (!left || !right || left->size() >= (size_t{1} << 31) || right->size() >= (size_t{1} << 31)) {
      return false;
    }
    auto position = size_t{0};
    for (const auto& value : *right) {
      while (position < left->size() && (*left)[position] < value) {
        ++position;
      }
      const auto found = position < left->size() && (*left)[position] == value;
      words.push_back(static_cast<uint32_t>(2 * position + (found ? 1 : 0)));
    }
  }
  return true;
}

// hyb_scan_predicate of `column <condition> value [AND value2]` on a stored table: string literals become per-chunk value-ID
// bounds, LIKE patterns dictionary bitmaps (both in `bounds`, which must outlive the predicate), numeric literals are cast
// losslessly to the column type. false: no device form (the CPU operator, or an operand leaf, takes it).
bool scan_predicate(const Table& in_table, ColumnID column_id, PredicateCondition condition, const AllTypeVariant& value,
                    const std::optional<AllTypeVariant>& value2, std::vector<uint32_t>& bounds, hyb_scan_predicate& predicate) {
  const auto column_type = in_table.column_data_type(column_id);
  predicate = hyb_scan_predicate{};
  predicate.column_id = column_id;
  predicate.condition = static_cast<int32_t>(condition);  // PredicateCondition and hyb_predicate_condition share values
  bounds.clear();
  const auto needs_value = condition != PredicateCondition::IsNull && condition != PredicateCondition::IsNotNull;
  const auto is_like = condition == PredicateCondition::Like || condition == PredicateCondition::NotLike ||
                       condition == PredicateCondition::LikeInsensitive || condition == PredicateCondition::NotLikeInsensitive;
  if (is_like) {
    if (column_type != DataType::String ||
        !like_dictionary_bitmaps(in_table, column_id, condition, boost::get<pmr_string>(value), bounds)) {
      return false;  // the reference operator reports LIKE on a non-string column itself
    }
    bounds.push_back(0);  // never a NULL pointer, even when no chunk has a dictionary entry
    predicate.value_id_bounds = bounds.data();
  } else if (needs_value && column_type == DataType::String) {
    if (!string_value_id_bounds(in_table, column_id, value, value2, bounds)) {
      return false;
    }
    predicate.value_id_bounds = bounds.data();
  } else if (needs_value) {
    // table_scan.cpp:340-366 / :399-441: literals of another type are cast losslessly (or the scan runs on the CPU)
    if (is_between_predicate_condition(condition)) {
      const auto lower = hyb_literal{hyb_type(data_type_from_all_type_variant(value)),
                                     to_hyb_value(value, data_type_from_all_type_variant(value))};
      const auto upper = hyb_literal{hyb_type(data_type_from_all_type_variant(*value2)),
                                     to_hyb_value(*value2, data_type_from_all_type_variant(*value2))};
      if (hyb_lossless_between_cast(predicate.condition, &lower, &upper, hyb_type(column_type), &predicate.condition,
                                    &predicate.lower, &predicate.upper) != HYB_OK) {
        return false;
      }
    } else {
      const auto literal = hyb_literal{hyb_type(data_type_from_all_type_variant(value)),
                                       to_hyb_value(value, data_type_from_all_type_variant(value))};
      if (hyb_lossless_predicate_cast(predicate.condition, &literal, hyb_type(column_type), 0, &predicate.condition,
                                      &predicate.lower) != HYB_OK) {
        return false;
      }
    }
  }
  return true;
}

// hyb_in_predicate of `column [NOT] IN (<literal list>)` on a stored table: numeric elements in `literals`, the string
// elements' dictionary bitmaps in `words` (both must outlive the predicate). false: a non-literal element, or a string
// column without dictionaries (the CPU operator runs).
bool in_predicate(const Table& in_table, ColumnID column_id, bool negated, const ListExpression& list,
                  std::vector<hyb_literal>& literals, std::vector<uint32_t>& words, hyb_in_predicate& predicate) {
  literals.clear();
  words.clear();
  auto strings = std::vector<pmr_string>{};
  auto has_null_element = false;
  for (const auto& element : list.elements()) {
    const auto value_expression = std::dynamic_pointer_cast<const ValueExpression>(element);
    if (!value_expression) {
      return false;  // a non-literal element (`13 * 13`, a column, a parameter) stays on the CPU
    }
    const auto& value = value_expression->value;
    if (variant_is_null(value)) {
      has_null_element = true;
    } else if (value.type() == typeid(pmr_string)) {
      strings.emplace_back(boost::get<pmr_string>(value));
    } else {
      auto literal = hyb_literal{};
      if (value.type() == typeid(int32_t)) {
        literal.data_type = HYB_TYPE_INT32;
        literal.value.i32 = boost::get<int32_t>(value);
      } else if (value.type() == typeid(int64_t)) {
        literal.data_type = HYB_TYPE_INT64;
        literal.value.i64 = boost::get<int64_t>(value);
      } else if (value.type() == typeid(float)) {
        literal.data_type = HYB_TYPE_FLOAT32;
        literal.value.f32 = boost::get<float>(value);
      } else {
        literal.data_type = HYB_TYPE_FLOAT64;
        literal.value.f64 = boost::get<double>(value);
      }
      literals.push_back(literal);
    }
  }
  predicate = hyb_in_predicate{};
  predicate.column_id = column_id;
  predicate.condition = negated ? HYB_PRED_NOT_IN : HYB_PRED_IN;
  if (in_table.column_data_type(column_id) == DataType::String) {
    // the library drops numeric and NULL elements of a string column itself; only the string elements become bitmaps
    if (!strings.empty()) {
      auto element_chars = std::string{};
      auto element_offsets = std::vector<uint64_t>{0};
      for (const auto& string : strings) {
        element_chars.append(string.data(), string.size());
        element_offsets.push_back(element_chars.size());
      }
      for (auto chunk_id = ChunkID{0}; chunk_id < in_table.chunk_count(); ++chunk_id) {
        const auto dictionary = string_dictionary(in_table, chunk_id, column_id);
        if (!dictionary) {
          return false;
        }
        auto chars = std::string{};
        auto offsets = std::vector<uint64_t>{0};
        for (const auto& value : *dictionary) {
          chars.append(value.data(), value.size());
          offsets.push_back(chars.size());
        }
        const auto first = words.size();
        words.resize(first + (dictionary->size() + 31) / 32);
        Assert(hyb_in_dictionary_matches(predicate.condition, element_chars.data(), element_offsets.data(),
                                         static_cast<uint32_t>(strings.size()), chars.data(), offsets.data(),
                                         static_cast<uint32_t>(dictionary->size()), words.data() + first, nullptr) == HYB_OK,
               hyb_last_error());
      }
      words.push_back(0);  // never a NULL pointer, even when no chunk has a dictionary entry
      predicate.dictionary_matches = words.data();
    }
  } else {
    // string elements of a numeric column are dropped, as rewrite_in_list_expression drops them
    predicate.element_count = static_cast<uint32_t>(literals.size());
    predicate.has_null_element = has_null_element;
    predicate.elements = literals.data();
  }
  return true;
}

// One operand of an expression predicate as a hyb_expr_node program (reverse Polish): columns, numeric literals, NULL and
// + - * / %. Anything else (strings, functions, CASE, parameters, subqueries): false, the CPU operator runs.
bool expression_program(const AbstractExpression& expression, std::vector<hyb_expr_node>& nodes) {
  auto node = hyb_expr_node{};
  if (const auto* column = dynamic_cast<const PQPColumnExpression*>(&expression)) {
    node.op = HYB_EXPR_COLUMN;
    node.column_id = column->column_id;
  } else if (const auto* value_expression = dynamic_cast<const ValueExpression*>(&expression)) {
    const auto& value = value_expression->value;
    if (variant_is_null(value)) {
      node.op = HYB_EXPR_NULL;
    } else if (value.type() == typeid(pmr_string)) {
      return false;
    } else {
      node.op = HYB_EXPR_LITERAL;
      node.literal_type = hyb_type(data_type_from_all_type_variant(value));
      node.literal = to_hyb_value(value, data_type_from_all_type_variant(value));
    }
  } else if (const auto* arithmetic = dynamic_cast<const ArithmeticExpression*>(&expression)) {
    if (!expression_program(*arithmetic->left_operand(), nodes) || !expression_program(*arithmetic->right_operand(), nodes)) {
      return false;
    }
    switch (arithmetic->arithmetic_operator) {
      case ArithmeticOperator::Addition:
        node.op = HYB_EXPR_ADD;
        break;
      case ArithmeticOperator::Subtraction:
        node.op = HYB_EXPR_SUB;
        break;
      case ArithmeticOperator::Multiplication:
        node.op = HYB_EXPR_MUL;
        break;
      case ArithmeticOperator::Division:
        node.op = HYB_EXPR_DIV;
        break;
      case ArithmeticOperator::Modulo:
        node.op = HYB_EXPR_MOD;
        break;
    }
  } else {
    return false;
  }
  if (nodes.size() == HYB_MAX_EXPR_NODES) {
    return false;  // longer than the ABI takes
  }
  nodes.push_back(node);
  return true;
}

// The column-test leaves of hyb_table_scan_expression_tests with the buffers their pointers refer to (deques: appending
// never moves an element).
struct LeafTests {
  std::vector<hyb_scan_predicate> scans;
  std::vector<hyb_in_predicate> ins;
  std::deque<std::vector<uint32_t>> words;
  std::deque<std::vector<hyb_literal>> literals;
};

// A leaf the standalone scans take, as a column-test term: a bare column against string literals (comparisons, BETWEEN,
// LIKE; a literal on the left is flipped), a numeric comparison / BETWEEN whose literals cast losslessly to the column
// type, and IN over a literal list of a bare column. false: not such a leaf (an operand leaf may still take it).
bool column_test_term(const Table& stored, const AbstractExpression& expression, LeafTests& tests,
                      std::vector<hyb_expression_term>& terms) {
  const auto column_of = [](const std::shared_ptr<AbstractExpression>& operand) {
    return std::dynamic_pointer_cast<const PQPColumnExpression>(operand);
  };
  const auto value_of = [](const std::shared_ptr<AbstractExpression>& operand) -> std::optional<AllTypeVariant> {
    const auto value = std::dynamic_pointer_cast<const ValueExpression>(operand);
    if (!value || variant_is_null(value->value)) {
      return std::nullopt;
    }
    return value->value;
  };
  auto term = hyb_expression_term{};
  if (const auto* in = dynamic_cast<const InExpression*>(&expression)) {
    const auto column = column_of(in->operand());
    const auto list = std::dynamic_pointer_cast<const ListExpression>(in->set());
    auto predicate = hyb_in_predicate{};
    auto& literals = tests.literals.emplace_back();
    auto& words = tests.words.emplace_back();
    if (!column || !list || !in_predicate(stored, column->column_id, in->is_negated(), *list, literals, words, predicate)) {
      return false;
    }
    tests.ins.push_back(predicate);
    term.kind = HYB_TERM_IN;
    terms.push_back(term);
    return true;
  }
  auto column = std::shared_ptr<const PQPColumnExpression>{};
  auto condition = PredicateCondition{};
  auto value = std::optional<AllTypeVariant>{};
  auto value2 = std::optional<AllTypeVariant>{};
  if (const auto* between = dynamic_cast<const BetweenExpression*>(&expression)) {
    column = column_of(between->operand());
    condition = between->predicate_condition;
    value = value_of(between->lower_bound());
    value2 = value_of(between->upper_bound());
    if (!value2) {
      return false;
    }
  } else if (const auto* binary = dynamic_cast<const BinaryPredicateExpression*>(&expression)) {
    condition = binary->predicate_condition;
    column = column_of(binary->left_operand());
    value = value_of(binary->right_operand());
    const auto like = condition == PredicateCondition::Like || condition == PredicateCondition::NotLike ||
                      condition == PredicateCondition::LikeInsensitive || condition == PredicateCondition::NotLikeInsensitive;
    if (!column && !like) {  // `literal <op> column`
      column = column_of(binary->right_operand());
      value = value_of(binary->left_operand());
      condition = flip_predicate_condition(condition);
    }
  }
  if (!column || !value) {
    return false;
  }
  const auto column_is_string = stored.column_data_type(column->column_id) == DataType::String;
  if (column_is_string != (value->type() == typeid(pmr_string)) || (value2 && column_is_string != (value2->type() == typeid(pmr_string)))) {
    return false;  // a string against a number: the operand path reports it
  }
  auto predicate = hyb_scan_predicate{};
  auto& bounds = tests.words.emplace_back();
  if (!scan_predicate(stored, column->column_id, condition, *value, value2, bounds, predicate)) {
    return false;  // no lossless literal: the operand leaf compares in the common type
  }
  tests.scans.push_back(predicate);
  term.kind = HYB_TERM_SCAN;
  terms.push_back(term);
  return true;
}

// A predicate tree as the postfix terms of hyb_expression_scan_predicate: comparisons, BETWEEN and IS [NOT] NULL leaves,
// AND / OR nodes. With `tests`, the leaves the standalone scans take become column-test leaves (column_test_term).
// Anything else (EXISTS, NOT, a bare value, and without `tests` IN and LIKE): false.
bool expression_terms(const AbstractExpression& expression, std::vector<hyb_expression_term>& terms,
                      const Table* stored = nullptr, LeafTests* tests = nullptr) {
  if (const auto* logical = dynamic_cast<const LogicalExpression*>(&expression)) {
    if (!expression_terms(*logical->left_operand(), terms, stored, tests) ||
        !expression_terms(*logical->right_operand(), terms, stored, tests)) {
      return false;
    }
    auto term = hyb_expression_term{};
    term.kind = logical->logical_operator == LogicalOperator::And ? HYB_TERM_AND : HYB_TERM_OR;
    terms.push_back(term);
    return true;
  }
  if (tests && column_test_term(*stored, expression, *tests, terms)) {
    return true;
  }
  auto operands = std::vector<std::shared_ptr<AbstractExpression>>{};
  if (const auto* between = dynamic_cast<const BetweenExpression*>(&expression)) {
    operands = {between->operand(), between->lower_bound(), between->upper_bound()};
  } else if (const auto* is_null = dynamic_cast<const IsNullExpression*>(&expression)) {
    operands = {is_null->operand()};
  } else if (const auto* binary = dynamic_cast<const BinaryPredicateExpression*>(&expression)) {
    operands = {binary->left_operand(), binary->right_operand()};
  } else {
    return false;
  }
  auto term = hyb_expression_term{};
  term.kind = HYB_TERM_LEAF;
  // PredicateCondition and hyb_predicate_condition share values; LIKE leaves come back as HYB_ERR_UNSUPPORTED
  term.condition = static_cast<int32_t>(static_cast<const AbstractPredicateExpression&>(expression).predicate_condition);
  for (auto slot = size_t{0}; slot < operands.size(); ++slot) {
    auto nodes = std::vector<hyb_expr_node>{};
    if (!expression_program(*operands[slot], nodes)) {
      return false;
    }
    std::copy(nodes.begin(), nodes.end(), term.operands[slot]);
    term.node_counts[slot] = static_cast<uint32_t>(nodes.size());
  }
  terms.push_back(term);
  return true;
}

// PosLists of a device result -> one output chunk of ReferenceSegments per input chunk with matches (table_scan.cpp:199-217).
std::shared_ptr<const Table> wrap_pos_lists(hyb_context* context, const std::shared_ptr<const Table>& stored, hyb_pos_list_t result) {
  auto chunk_count = uint32_t{0};
  auto total = uint64_t{0};
  Assert(hyb_pos_list_info(context, result, &total, &chunk_count) == HYB_OK, hyb_last_error());
  auto offsets = std::vector<uint64_t>(size_t{chunk_count} + 1);
  Assert(hyb_pos_list_chunk_offsets(context, result, offsets.data()) == HYB_OK, hyb_last_error());
  auto output_chunks = std::vector<std::shared_ptr<Chunk>>{};
  for (auto chunk_id = ChunkID{0}; chunk_id < chunk_count; ++chunk_id) {
    const auto matches = offsets[chunk_id + 1] - offsets[chunk_id];
    if (matches == 0) {
      continue;
    }
    auto pos_list = std::make_shared<RowIDPosList>(matches);
    Assert(hyb_pos_list_copy(context, result, offsets[chunk_id], matches, reinterpret_cast<hyb_row_id*>(pos_list->data())) == HYB_OK,
           hyb_last_error());
    pos_list->guarantee_single_chunk();
    auto segments = Segments{};
    for (auto column_id = ColumnID{0}; column_id < stored->column_count(); ++column_id) {
      segments.emplace_back(std::make_shared<ReferenceSegment>(stored, column_id, pos_list));
    }
    output_chunks.emplace_back(std::make_shared<Chunk>(std::move(segments)));
  }
  hyb_pos_list_free(context, result);
  return std::make_shared<Table>(stored->column_definitions(), TableType::References, std::move(output_chunks));
}

}  // namespace

DeviceColumnPool* gpu_column_pool() {
  return global_pool.load();
}

void set_gpu_column_pool(DeviceColumnPool* pool) {
  global_pool.store(pool);
}

std::shared_ptr<const Table> try_gpu_table_scan(const std::shared_ptr<const Table>& in_table, ColumnID column_id,
                                                PredicateCondition condition, const AllTypeVariant& value,
                                                const std::optional<AllTypeVariant>& value2) {
  auto* pool = gpu_column_pool();
  if (!pool || in_table->type() != TableType::Data) {
    return nullptr;  // reference-table inputs: the shim keeps the previous operator's hyb_pos_list_t next to the table it
                     // produced and passes it as input_filter; omitted here for brevity
  }
  const auto* entry = pool->find(in_table);
  if (!entry) {
    return nullptr;
  }
  auto predicate = hyb_scan_predicate{};
  auto bounds = std::vector<uint32_t>{};
  if (!scan_predicate(*in_table, column_id, condition, value, value2, bounds, predicate)) {
    return nullptr;
  }
  auto result = hyb_pos_list_t{};
  const auto status = hyb_table_scan(pool->context(), entry->handle, &predicate, 0, &result);
  if (status == HYB_ERR_UNSUPPORTED) {
    return nullptr;
  }
  Assert(status == HYB_OK, hyb_last_error());
  return wrap_pos_lists(pool->context(), in_table, result);
}

std::shared_ptr<const Table> try_gpu_column_scan(const std::shared_ptr<const Table>& in_table, ColumnID left_column_id,
                                                 PredicateCondition condition, ColumnID right_column_id) {
  auto* pool = gpu_column_pool();
  if (!pool || in_table->type() != TableType::Data) {
    return nullptr;  // reference-table inputs: as in try_gpu_table_scan
  }
  const auto* entry = pool->find(in_table);
  if (!entry) {
    return nullptr;
  }
  auto predicate = hyb_column_scan_predicate{};
  predicate.left_column_id = left_column_id;
  predicate.condition = static_cast<int32_t>(condition);  // PredicateCondition and hyb_predicate_condition share values
  predicate.right_column_id = right_column_id;
  auto words = std::vector<uint32_t>{};
  if (in_table->column_data_type(left_column_id) == DataType::String &&
      in_table->column_data_type(right_column_id) == DataType::String) {
    if (!column_translation(*in_table, left_column_id, right_column_id, words)) {
      return nullptr;
    }
    words.push_back(0);  // never a NULL pointer, even when no chunk has a dictionary entry
    predicate.right_in_left = words.data();
  }
  auto result = hyb_pos_list_t{};
  const auto status = hyb_table_scan_columns(pool->context(), entry->handle, &predicate, 0, &result);
  if (status == HYB_ERR_UNSUPPORTED) {
    return nullptr;  // LIKE between two columns: the reference operator reports it itself
  }
  Assert(status == HYB_OK, hyb_last_error());
  return wrap_pos_lists(pool->context(), in_table, result);
}

std::shared_ptr<const Table> try_gpu_in_scan(const std::shared_ptr<const Table>& in_table, const InExpression& in_expression) {
  auto* pool = gpu_column_pool();
  if (!pool || in_table->type() != TableType::Data) {
    return nullptr;  // reference-table inputs: as in try_gpu_table_scan
  }
  const auto* entry = pool->find(in_table);
  const auto column = std::dynamic_pointer_cast<const PQPColumnExpression>(in_expression.operand());
  const auto list = std::dynamic_pointer_cast<const ListExpression>(in_expression.set());
  if (!entry || !column || !list) {
    return nullptr;  // IN over a subquery or an expression: ExpressionEvaluator
  }
  auto predicate = hyb_in_predicate{};
  auto literals = std::vector<hyb_literal>{};
  auto words = std::vector<uint32_t>{};
  if (!in_predicate(*in_table, column->column_id, in_expression.is_negated(), *list, literals, words, predicate)) {
    return nullptr;
  }
  auto result = hyb_pos_list_t{};
  const auto status = hyb_table_scan_in(pool->context(), entry->handle, &predicate, 0, &result);
  if (status == HYB_ERR_UNSUPPORTED) {
    return nullptr;
  }
  Assert(status == HYB_OK, hyb_last_error());
  return wrap_pos_lists(pool->context(), in_table, result);
}

std::shared_ptr<const Table> try_gpu_expression_scan(const std::shared_ptr<const Table>& in_table,
                                                     const AbstractExpression& predicate) {
  auto* pool = gpu_column_pool();
  if (!pool || in_table->type() != TableType::Data) {
    return nullptr;  // reference-table inputs: as in try_gpu_table_scan
  }
  const auto* entry = pool->find(in_table);
  auto terms = std::vector<hyb_expression_term>{};
  auto tests = LeafTests{};
  if (!entry || !expression_terms(predicate, terms, in_table.get(), &tests)) {
    return nullptr;
  }
  auto expression_predicate = hyb_expression_scan_predicate{};
  expression_predicate.term_count = static_cast<uint32_t>(terms.size());
  expression_predicate.terms = terms.data();
  auto result = hyb_pos_list_t{};
  auto status = HYB_OK;
  if (tests.scans.empty() && tests.ins.empty()) {
    status = hyb_table_scan_expression(pool->context(), entry->handle, &expression_predicate, 0, &result);
  } else {
    const auto leaf_tests = hyb_expression_leaf_tests{static_cast<uint32_t>(tests.scans.size()),
                                                      static_cast<uint32_t>(tests.ins.size()), tests.scans.data(),
                                                      tests.ins.data()};
    status = hyb_table_scan_expression_tests(pool->context(), entry->handle, &expression_predicate, &leaf_tests, 0, &result);
  }
  if (status == HYB_ERR_UNSUPPORTED) {
    return nullptr;  // string operands, more leaves, columns or postfix depth than the ABI takes
  }
  Assert(status == HYB_OK, hyb_last_error());
  return wrap_pos_lists(pool->context(), in_table, result);
}

std::shared_ptr<const Table> try_gpu_join_hash(const std::shared_ptr<const Table>& build_table,
                                               const std::shared_ptr<const Table>& probe_table, ColumnID build_column_id,
                                               ColumnID probe_column_id, JoinMode mode, size_t radix_bits,
                                               bool build_is_left_input,
                                               const std::vector<OperatorJoinPredicate>& secondary_predicates) {
  auto* pool = gpu_column_pool();
  if (!pool) {
    return nullptr;
  }
  const auto* build_entry = pool->find(build_table);
  const auto* probe_entry = pool->find(probe_table);
  if (!build_entry || !probe_entry || build_table->type() != TableType::Data || probe_table->type() != TableType::Data) {
    return nullptr;
  }
  const auto build = hyb_join_side{build_entry->handle, build_column_id, 0};
  const auto probe = hyb_join_side{probe_entry->handle, probe_column_id, 0};
  // the secondary predicates arrive adjusted to `build <condition> probe` (join_hash.cpp:158-165)
  auto predicates = std::vector<hyb_join_predicate>{};
  for (const auto& predicate : secondary_predicates) {
    predicates.push_back(hyb_join_predicate{static_cast<uint32_t>(predicate.column_ids.first),
                                            static_cast<uint32_t>(predicate.column_ids.second),
                                            static_cast<int32_t>(predicate.predicate_condition), 0});
  }
  auto result = hyb_join_result_t{};
  const auto status = hyb_join_hash_predicates(pool->context(), &build, &probe, static_cast<int32_t>(mode),
                                               static_cast<int32_t>(radix_bits), predicates.data(),
                                               static_cast<uint32_t>(predicates.size()), &result);
  if (status == HYB_ERR_UNSUPPORTED) {
    return nullptr;  // string / float keys, string secondary predicates, AntiNullAsTrue with secondary predicates
  }
  Assert(status == HYB_OK, hyb_last_error());
  // The pairs arrive in the order probe() emits them (partition, probe row, build row): one PosList pair per partition, then
  // the reference's own write_output_chunks (join_helper/join_output_writing.cpp:205-340) merges / splits and builds the chunks.
  auto pair_count = uint64_t{0};
  auto partition_count = uint32_t{0};
  Assert(hyb_join_result_info(pool->context(), result, &pair_count, &partition_count, nullptr) == HYB_OK, hyb_last_error());
  auto offsets = std::vector<uint64_t>(size_t{partition_count} + 1);
  Assert(hyb_join_result_partition_offsets(pool->context(), result, offsets.data()) == HYB_OK, hyb_last_error());
  const auto emits_build_side = mode != JoinMode::Semi && mode != JoinMode::AntiNullAsTrue && mode != JoinMode::AntiNullAsFalse;
  auto build_pos_lists = std::vector<RowIDPosList>(partition_count);
  auto probe_pos_lists = std::vector<RowIDPosList>(partition_count);
  for (auto partition = size_t{0}; partition < partition_count; ++partition) {
    const auto rows = offsets[partition + 1] - offsets[partition];
    probe_pos_lists[partition].resize(rows);
    if (emits_build_side) {
      build_pos_lists[partition].resize(rows);
    }
    Assert(hyb_join_result_copy(pool->context(), result, offsets[partition], rows,
                                emits_build_side ? reinterpret_cast<hyb_row_id*>(build_pos_lists[partition].data()) : nullptr,
                                reinterpret_cast<hyb_row_id*>(probe_pos_lists[partition].data())) == HYB_OK,
           hyb_last_error());
  }
  hyb_join_result_free(pool->context(), result);
  auto& left_pos_lists = build_is_left_input ? build_pos_lists : probe_pos_lists;
  auto& right_pos_lists = build_is_left_input ? probe_pos_lists : build_pos_lists;
  const auto& left_table = build_is_left_input ? build_table : probe_table;
  const auto& right_table = build_is_left_input ? probe_table : build_table;
  auto output_chunks = write_output_chunks(left_pos_lists, right_pos_lists, left_table, right_table, /*create_left_side_pos_lists_by_column=*/false,
                                           /*create_right_side_pos_lists_by_column=*/false, OutputColumnOrder::LeftFirstRightSecond,
                                           /*allow_partition_merge=*/true);
  auto definitions = left_table->column_definitions();
  if (emits_build_side) {
    const auto& right_definitions = right_table->column_definitions();
    definitions.insert(definitions.end(), right_definitions.begin(), right_definitions.end());
  }
  return std::make_shared<Table>(definitions, TableType::References, std::move(output_chunks));
}

std::shared_ptr<const Table> try_gpu_aggregate_hash(const std::shared_ptr<const Table>& in_table,
                                                    const std::vector<ColumnID>& groupby_column_ids,
                                                    const std::vector<std::shared_ptr<WindowFunctionExpression>>& aggregates) {
  auto* pool = gpu_column_pool();
  if (!pool || in_table->type() != TableType::Data) {
    return nullptr;
  }
  const auto* entry = pool->find(in_table);
  if (!entry) {
    return nullptr;
  }
  // function + argument column (the reference has materialised arithmetic in a Projection below the aggregate; a fusing shim
  // passes the Projection's expressions as RPN programs and the scans below it as query.predicates instead, and a scan that
  // try_gpu_expression_scan would run as an expression tree as hyb_aggregate_hash_expression's predicate and leaf tests)
  auto nodes = std::vector<hyb_expr_node>(aggregates.size());
  auto definitions = std::vector<hyb_aggregate_def>(aggregates.size());
  for (auto index = size_t{0}; index < aggregates.size(); ++index) {
    const auto& aggregate = *aggregates[index];
    auto& definition = definitions[index];
    // WindowFunction and hyb_aggregate_function agree up to Count only (CountDistinct = 5 is HYB_AGG_COUNT_STAR's value),
    // so every function is mapped by name.
    switch (aggregate.window_function) {
      case WindowFunction::Min:
        definition.function = HYB_AGG_MIN;
        break;
      case WindowFunction::Max:
        definition.function = HYB_AGG_MAX;
        break;
      case WindowFunction::Sum:
        definition.function = HYB_AGG_SUM;
        break;
      case WindowFunction::Avg:
        definition.function = HYB_AGG_AVG;
        break;
      case WindowFunction::Count:
        definition.function = HYB_AGG_COUNT;
        break;
      case WindowFunction::CountDistinct:
        // over a string column the pool's segments carry the dictionary_codes the library compares instead of strings
        definition.function = HYB_AGG_COUNT_DISTINCT;
        break;
      case WindowFunction::StandardDeviationSample:
        definition.function = HYB_AGG_STDDEV_SAMP;
        break;
      case WindowFunction::Any:
        // no accumulator: the column at the representative RowIDs (DependentGroupByReductionRule, SELECT DISTINCT)
        definition.function = HYB_AGG_ANY;
        break;
      default:
        return nullptr;  // the window functions: the CPU operator
    }
    const auto column = std::dynamic_pointer_cast<const PQPColumnExpression>(aggregate.argument());
    if (aggregate.window_function == WindowFunction::Count && (!column || column->column_id == INVALID_COLUMN_ID)) {
      definition.function = HYB_AGG_COUNT_STAR;
      continue;
    }
    if (!column) {
      return nullptr;
    }
    nodes[index] = hyb_expr_node{};
    nodes[index].op = HYB_EXPR_COLUMN;
    nodes[index].column_id = column->column_id;
    definition.nodes = &nodes[index];
    definition.node_count = 1;
    const auto string_extreme = (aggregate.window_function == WindowFunction::Min ||
                                 aggregate.window_function == WindowFunction::Max) &&
                                in_table->column_data_type(column->column_id) == DataType::String;
    if (string_extreme && !pool->ensure_string_order(in_table, column->column_id)) {
      return nullptr;
    }
  }
  auto groupby = std::vector<uint32_t>(groupby_column_ids.begin(), groupby_column_ids.end());
  auto query = hyb_aggregate_query{};
  query.table = entry->handle;
  query.groupby_count = static_cast<uint32_t>(groupby.size());
  query.groupby_column_ids = groupby.data();
  query.aggregate_count = static_cast<uint32_t>(definitions.size());
  query.aggregates = definitions.data();
  auto result = hyb_aggregate_result_t{};
  const auto status = hyb_aggregate_hash(pool->context(), &query, &result);
  if (status == HYB_ERR_UNSUPPORTED) {
    return nullptr;  // SUM / AVG / expressions of strings, more aggregates or group-by columns than the device takes
  }
  Assert(status == HYB_OK, hyb_last_error());
  // Output: group-by columns as ReferenceSegments over the representative RowIDs (write_groupby_output, aggregate_hash.cpp:
  // 421-537), aggregate columns as ValueSegments (write_aggregate_output, :1374-1456), split into 65 535-row chunks like
  // split_results_chunk_wise (:237-294). hyb_aggregate_result_row_ids / hyb_aggregate_result_values deliver both in group order.
  auto group_count = uint64_t{0};
  Assert(hyb_aggregate_result_info(pool->context(), result, &group_count, nullptr) == HYB_OK, hyb_last_error());
  auto row_ids = std::make_shared<RowIDPosList>(group_count);
  Assert(hyb_aggregate_result_row_ids(pool->context(), result, reinterpret_cast<hyb_row_id*>(row_ids->data())) == HYB_OK,
         hyb_last_error());
  auto output_definitions = TableColumnDefinitions{};
  auto segments = Segments{};
  for (const auto column_id : groupby_column_ids) {
    output_definitions.emplace_back(in_table->column_definitions()[column_id]);
    segments.emplace_back(std::make_shared<ReferenceSegment>(in_table, column_id, row_ids));
  }
  for (auto index = size_t{0}; index < aggregates.size(); ++index) {
    const auto result_type = aggregates[index]->data_type();  // WindowFunctionTraits (window_function_traits.hpp:14-77)
    if (aggregates[index]->window_function == WindowFunction::Any) {
      // write_groupby_output (aggregate_hash.cpp:421-537): ANY columns are ReferenceSegments like the group-by columns
      const auto column_id = std::static_pointer_cast<const PQPColumnExpression>(aggregates[index]->argument())->column_id;
      segments.emplace_back(std::make_shared<ReferenceSegment>(in_table, column_id, row_ids));
      output_definitions.emplace_back(aggregates[index]->as_column_name(), result_type, true);
      continue;
    }
    resolve_data_type(result_type, [&](const auto type) {
      using AggregateType = typename decltype(type)::type;
      if constexpr (std::is_same_v<AggregateType, pmr_string>) {
        // MIN / MAX of a string column: one dictionary position per group, the string read from the stored table's
        // DictionarySegment (its dictionary entry); NULL groups stay empty strings under their NULL flag
        auto positions = std::vector<hyb_dictionary_position>(group_count);
        auto null_bytes = std::vector<uint8_t>(group_count);
        auto value_type = int32_t{0};
        Assert(hyb_aggregate_result_values(pool->context(), result, static_cast<uint32_t>(index), positions.data(),
                                           null_bytes.data(), &value_type) == HYB_OK,
               hyb_last_error());
        Assert(value_type == HYB_TYPE_STRING, "result type mismatch between the shim and the library");
        const auto column_id = std::static_pointer_cast<const PQPColumnExpression>(aggregates[index]->argument())->column_id;
        auto values = pmr_vector<pmr_string>(group_count);
        for (auto group = uint64_t{0}; group < group_count; ++group) {
          if (null_bytes[group]) {
            continue;
          }
          const auto segment = std::static_pointer_cast<const DictionarySegment<pmr_string>>(
              in_table->get_chunk(ChunkID{positions[group].chunk_id})->get_segment(column_id));
          values[group] = (*segment->dictionary())[positions[group].value_id];
        }
        auto nulls = pmr_vector<bool>(null_bytes.begin(), null_bytes.end());
        segments.emplace_back(std::make_shared<ValueSegment<pmr_string>>(std::move(values), std::move(nulls)));
      } else {
        auto values = pmr_vector<AggregateType>(group_count);
        auto null_bytes = std::vector<uint8_t>(group_count);
        auto value_type = int32_t{0};
        Assert(hyb_aggregate_result_values(pool->context(), result, static_cast<uint32_t>(index), values.data(), null_bytes.data(),
                                           &value_type) == HYB_OK,
               hyb_last_error());
        Assert(value_type == hyb_type(result_type), "result type mismatch between the shim and the library");
        auto nulls = pmr_vector<bool>(null_bytes.begin(), null_bytes.end());
        segments.emplace_back(std::make_shared<ValueSegment<AggregateType>>(std::move(values), std::move(nulls)));
      }
    });
    output_definitions.emplace_back(aggregates[index]->as_column_name(), result_type, true);
  }
  hyb_aggregate_result_free(pool->context(), result);
  auto output = std::make_shared<Table>(output_definitions, TableType::Data);
  if (group_count > 0) {
    output->append_chunk(segments);  // > 65 535 groups: slice the vectors per Chunk::DEFAULT_SIZE first (:237-294)
  }
  return output;
}

std::shared_ptr<const Table> try_gpu_sort(const std::shared_ptr<const Table>& in_table,
                                          const std::vector<SortColumnDefinition>& sort_definitions,
                                          ChunkOffset output_chunk_size) {
  auto* pool = gpu_column_pool();
  if (!pool || in_table->type() != TableType::Data) {
    return nullptr;  // reference-table inputs: as in try_gpu_table_scan (the scan's hyb_pos_list_t is the input_filter)
  }
  const auto* entry = pool->find(in_table);
  if (!entry) {
    return nullptr;
  }
  auto columns = std::vector<hyb_sort_column>{};
  for (const auto& definition : sort_definitions) {
    if (definition.sort_mode != SortMode::AscendingNullsFirst && definition.sort_mode != SortMode::DescendingNullsFirst) {
      return nullptr;  // the reference asserts these away (sort.cpp:294-296)
    }
    // a string column sorts by its order ranks: attach them on first use, as string MIN / MAX does
    if (in_table->column_data_type(definition.column) == DataType::String &&
        !pool->ensure_string_order(in_table, definition.column)) {
      return nullptr;
    }
    columns.push_back(hyb_sort_column{definition.column, definition.sort_mode == SortMode::DescendingNullsFirst ? 1 : 0});
  }
  auto result = hyb_pos_list_t{};
  const auto status = hyb_sort(pool->context(), entry->handle, 0, columns.data(), static_cast<uint32_t>(columns.size()), &result);
  if (status == HYB_ERR_UNSUPPORTED) {
    return nullptr;
  }
  Assert(status == HYB_OK, hyb_last_error());
  // one flat list in sorted order, cut into output chunks of output_chunk_size rows (sort.cpp:456-501)
  auto total = uint64_t{0};
  Assert(hyb_pos_list_info(pool->context(), result, &total, nullptr) == HYB_OK, hyb_last_error());
  auto output_chunks = std::vector<std::shared_ptr<Chunk>>{};
  for (auto begin = uint64_t{0}; begin < total; begin += output_chunk_size) {
    const auto rows = std::min<uint64_t>(output_chunk_size, total - begin);
    auto pos_list = std::make_shared<RowIDPosList>(rows);
    Assert(hyb_pos_list_copy(pool->context(), result, begin, rows, reinterpret_cast<hyb_row_id*>(pos_list->data())) == HYB_OK,
           hyb_last_error());
    auto segments = Segments{};
    for (auto column_id = ColumnID{0}; column_id < in_table->column_count(); ++column_id) {
      segments.emplace_back(std::make_shared<ReferenceSegment>(in_table, column_id, pos_list));
    }
    output_chunks.emplace_back(std::make_shared<Chunk>(std::move(segments)));
  }
  hyb_pos_list_free(pool->context(), result);
  return std::make_shared<Table>(in_table->column_definitions(), TableType::References, std::move(output_chunks));
}

}  // namespace hyrise
