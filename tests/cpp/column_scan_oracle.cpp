// Column-vs-column TableScan on decoded numeric values (CPU, test infrastructure only).
//
// A restatement of ColumnVsColumnTableScanImpl::_typed_scan_chunk_with_iterators and the two-iterator branch of
// AbstractTableScanImpl::_scan_with_iterators<true> (abstract_table_scan_impl.hpp:56-84): a row matches iff neither value
// is NULL and the reference's comparator holds. The comparators are the real std::equal_to<void>, std::not_equal_to<void>
// and std::less<void> / std::less_equal<void>, so C++ itself applies the usual arithmetic conversions (int x float in
// float, int64 x double in double, ...). As in the reference, > and >= swap the operands and use < and <=.
// The values come decoded (tests/column_scan_oracle.py decodes the segments with the CPU oracle), one array per side.
#include <cstdint>
#include <functional>

#include "../../include/hyrise_b200.h"

namespace {

template <typename Left, typename Right, typename Comparator>
void scan(const Left* left, const uint8_t* left_nulls, const Right* right, const uint8_t* right_nulls, uint64_t rows,
          bool swap, const Comparator& comparator, uint8_t* out) {
  for (uint64_t row = 0; row < rows; ++row) {
    if (left_nulls[row] || right_nulls[row]) {
      out[row] = 0;
      continue;
    }
    out[row] = swap ? comparator(right[row], left[row]) : comparator(left[row], right[row]);
  }
}

template <typename Left, typename Right>
int scan_typed(const void* left, const uint8_t* left_nulls, const void* right, const uint8_t* right_nulls, uint64_t rows,
               int32_t condition, uint8_t* out) {
  const auto* l = static_cast<const Left*>(left);
  const auto* r = static_cast<const Right*>(right);
  switch (condition) {
    case HYB_PRED_EQUALS:
      scan(l, left_nulls, r, right_nulls, rows, false, std::equal_to<void>{}, out);
      return 0;
    case HYB_PRED_NOT_EQUALS:
      scan(l, left_nulls, r, right_nulls, rows, false, std::not_equal_to<void>{}, out);
      return 0;
    case HYB_PRED_LESS_THAN:
      scan(l, left_nulls, r, right_nulls, rows, false, std::less<void>{}, out);
      return 0;
    case HYB_PRED_LESS_THAN_EQUALS:
      scan(l, left_nulls, r, right_nulls, rows, false, std::less_equal<void>{}, out);
      return 0;
    case HYB_PRED_GREATER_THAN:  // column_vs_column_table_scan_impl.cpp: flipped to `right < left`
      scan(l, left_nulls, r, right_nulls, rows, true, std::less<void>{}, out);
      return 0;
    case HYB_PRED_GREATER_THAN_EQUALS:
      scan(l, left_nulls, r, right_nulls, rows, true, std::less_equal<void>{}, out);
      return 0;
    default:
      return HYB_ERR_INVALID;
  }
}

template <typename Left>
int scan_right(int32_t right_type, const void* left, const uint8_t* left_nulls, const void* right,
               const uint8_t* right_nulls, uint64_t rows, int32_t condition, uint8_t* out) {
  switch (right_type) {
    case HYB_TYPE_INT32:
      return scan_typed<Left, int32_t>(left, left_nulls, right, right_nulls, rows, condition, out);
    case HYB_TYPE_INT64:
      return scan_typed<Left, int64_t>(left, left_nulls, right, right_nulls, rows, condition, out);
    case HYB_TYPE_FLOAT32:
      return scan_typed<Left, float>(left, left_nulls, right, right_nulls, rows, condition, out);
    case HYB_TYPE_FLOAT64:
      return scan_typed<Left, double>(left, left_nulls, right, right_nulls, rows, condition, out);
    default:
      return HYB_ERR_INVALID;  // "Trying to compare strings and non-strings"
  }
}

}  // namespace

extern "C" {

// out_matches[row] = 1 iff row matches `left <condition> right`; values are arrays of the columns' types.
int csc_scan_decoded(int32_t left_type, const void* left_values, const uint8_t* left_nulls, int32_t right_type,
                     const void* right_values, const uint8_t* right_nulls, uint64_t rows, int32_t condition,
                     uint8_t* out_matches) {
  switch (left_type) {
    case HYB_TYPE_INT32:
      return scan_right<int32_t>(right_type, left_values, left_nulls, right_values, right_nulls, rows, condition,
                                 out_matches);
    case HYB_TYPE_INT64:
      return scan_right<int64_t>(right_type, left_values, left_nulls, right_values, right_nulls, rows, condition,
                                 out_matches);
    case HYB_TYPE_FLOAT32:
      return scan_right<float>(right_type, left_values, left_nulls, right_values, right_nulls, rows, condition,
                               out_matches);
    case HYB_TYPE_FLOAT64:
      return scan_right<double>(right_type, left_values, left_nulls, right_values, right_nulls, rows, condition,
                                out_matches);
    default:
      return HYB_ERR_INVALID;
  }
}

}  // extern "C"
