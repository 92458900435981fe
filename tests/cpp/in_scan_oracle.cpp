// `<column> [NOT] IN (<literal>, ...)` row by row (CPU, test infrastructure only).
//
// A restatement of ExpressionEvaluator::_evaluate_in_expression on a ListExpression of ValueExpressions
// (expression_evaluator.cpp:404-511), of rewrite_in_list_expression (:117-163) and of the ternary OR / AND the rewritten
// expression evaluates to. It never builds intervals or dictionary bitmaps:
//   - only elements whose "is a string" agrees with the column's count (a NULL element's type is Null, not String);
//   - no such element (the empty list included): the literal `negated` for every row, NULL rows included;
//   - every element a value of exactly the column's type (fast path): std::find over the values, NULL rows are NULL;
//   - otherwise (slow path): `a = e1 OR a = e2 ...` / `a != e1 AND a != e2 ...` in SQL's three-valued logic, each
//     comparison std::equal_to / std::not_equal_to in std::common_type_t<column type, element type>, NULL if either side is.
// A row is selected iff the result is non-zero and not NULL (ExpressionEvaluator::evaluate_expression_to_pos_list).
#include <algorithm>
#include <cstdint>
#include <functional>
#include <string_view>
#include <type_traits>
#include <vector>

#include "../../include/hyrise_b200.h"

namespace {

constexpr int32_t kNullElement = -1;

enum Ternary { kFalse = 0, kTrue = 1, kNull = 2 };

struct Elements {
  uint32_t count;
  const int32_t* types;  // HYB_TYPE_* or kNullElement
  const hyb_value* values;
  const char* chars;
  const uint64_t* offsets;
  std::string_view string(uint32_t i) const {
    return std::string_view(chars ? chars + offsets[i] : "", offsets[i + 1] - offsets[i]);
  }
};

template <typename Left, typename Right>
bool equal(Left left, Right right) {
  if constexpr (std::is_same_v<Left, std::string_view> || std::is_same_v<Right, std::string_view>) {
    if constexpr (std::is_same_v<Left, Right>) {
      return left == right;
    } else {
      return false;  // never called: incompatible elements are dropped first
    }
  } else {
    using Common = std::common_type_t<Left, Right>;
    return std::equal_to<Common>{}(static_cast<Common>(left), static_cast<Common>(right));
  }
}

template <typename Left>
bool equals_element(Left left, const Elements& elements, uint32_t i) {
  switch (elements.types[i]) {
    case HYB_TYPE_INT32:
      return equal(left, elements.values[i].i32);
    case HYB_TYPE_INT64:
      return equal(left, static_cast<int64_t>(elements.values[i].i64));
    case HYB_TYPE_FLOAT32:
      return equal(left, elements.values[i].f32);
    case HYB_TYPE_FLOAT64:
      return equal(left, elements.values[i].f64);
    default:
      return equal(left, elements.string(i));
  }
}

template <typename Left>
Left element_as(const Elements& elements, uint32_t i) {
  if constexpr (std::is_same_v<Left, std::string_view>) {
    return elements.string(i);
  } else if constexpr (std::is_same_v<Left, int32_t>) {
    return elements.values[i].i32;
  } else if constexpr (std::is_same_v<Left, int64_t>) {
    return static_cast<int64_t>(elements.values[i].i64);
  } else if constexpr (std::is_same_v<Left, float>) {
    return elements.values[i].f32;
  } else {
    return elements.values[i].f64;
  }
}

template <typename Left, typename Row>
void evaluate(int32_t column_type, const Row& row_value, const uint8_t* nulls, uint64_t rows, bool negated,
              const Elements& elements, uint8_t* out) {
  const bool left_is_string = column_type == HYB_TYPE_STRING;
  std::vector<uint32_t> compatible;
  bool all_values_of_left_type = true;
  for (uint32_t i = 0; i < elements.count; ++i) {
    if ((elements.types[i] == HYB_TYPE_STRING) == left_is_string) compatible.push_back(i);
    if (elements.types[i] != column_type) all_values_of_left_type = false;
  }
  if (compatible.empty()) {  // `x IN ()` is false, `x NOT IN ()` is true: an unnullable literal
    std::fill(out, out + rows, static_cast<uint8_t>(negated));
    return;
  }
  if (all_values_of_left_type) {
    std::vector<Left> right_values;
    for (const uint32_t i : compatible) right_values.push_back(element_as<Left>(elements, i));
    for (uint64_t row = 0; row < rows; ++row) {
      if (nulls[row]) {
        out[row] = 0;  // NULL
        continue;
      }
      const Left value = row_value(row);
      const auto it = std::find(right_values.cbegin(), right_values.cend(), value);
      const bool found = it != right_values.cend() && *it == value;
      out[row] = found != negated;
    }
    return;
  }
  for (uint64_t row = 0; row < rows; ++row) {
    Ternary result = negated ? kTrue : kFalse;
    for (const uint32_t i : compatible) {
      Ternary term;
      if (nulls[row] || elements.types[i] == kNullElement) {
        term = kNull;
      } else {
        term = equals_element(row_value(row), elements, i) != negated ? kTrue : kFalse;
      }
      if (!negated) {  // OR: TRUE wins, then NULL
        if (term == kTrue || result == kTrue) {
          result = kTrue;
        } else if (term == kNull) {
          result = kNull;
        }
      } else {  // AND: FALSE wins, then NULL
        if (term == kFalse || result == kFalse) {
          result = kFalse;
        } else if (term == kNull) {
          result = kNull;
        }
      }
    }
    out[row] = result == kTrue;
  }
}

template <typename Left>
void evaluate_numeric(int32_t column_type, const void* values, const uint8_t* nulls, uint64_t rows, bool negated,
                      const Elements& elements, uint8_t* out) {
  const auto* typed = static_cast<const Left*>(values);
  evaluate<Left>(column_type, [typed](uint64_t row) { return typed[row]; }, nulls, rows, negated, elements, out);
}

}  // namespace

extern "C" {

// out_selected[row] = 1 iff `row [NOT] IN (elements)` is non-zero and not NULL. Numeric columns: `values` holds rows
// values of the column type. STRING columns: row r is chars[offsets[r] .. offsets[r + 1]). element_types: HYB_TYPE_* or
// -1 for a NULL element; string element i is element_chars[element_offsets[i] .. element_offsets[i + 1]) (the offsets
// cover every element, non-string ones with empty ranges).
int ino_scan(int32_t column_type, const void* values, const char* chars, const uint64_t* offsets, const uint8_t* nulls,
             uint64_t rows, int32_t negated, uint32_t element_count, const int32_t* element_types,
             const hyb_value* element_values, const char* element_chars, const uint64_t* element_offsets,
             uint8_t* out_selected) {
  const Elements elements{element_count, element_types, element_values, element_chars, element_offsets};
  switch (column_type) {
    case HYB_TYPE_INT32:
      evaluate_numeric<int32_t>(column_type, values, nulls, rows, negated != 0, elements, out_selected);
      return 0;
    case HYB_TYPE_INT64:
      evaluate_numeric<int64_t>(column_type, values, nulls, rows, negated != 0, elements, out_selected);
      return 0;
    case HYB_TYPE_FLOAT32:
      evaluate_numeric<float>(column_type, values, nulls, rows, negated != 0, elements, out_selected);
      return 0;
    case HYB_TYPE_FLOAT64:
      evaluate_numeric<double>(column_type, values, nulls, rows, negated != 0, elements, out_selected);
      return 0;
    case HYB_TYPE_STRING: {
      const auto row_value = [chars, offsets](uint64_t row) {
        return std::string_view(chars ? chars + offsets[row] : "", offsets[row + 1] - offsets[row]);
      };
      evaluate<std::string_view>(column_type, row_value, nulls, rows, negated != 0, elements, out_selected);
      return 0;
    }
    default:
      return HYB_ERR_INVALID;
  }
}

}  // extern "C"
