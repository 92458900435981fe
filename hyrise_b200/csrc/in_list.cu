// Host-only helpers of `<column> [NOT] IN (<literal>, ...)` scans (hyb_table_scan_in, scan.cu).
//
// hyb_in_list_normalize turns the numeric list into the values of the column type it matches: for every element e, the set
// {v : std::equal_to<std::common_type_t<Column, Element>>{}(v, e)}, which is one closed interval because the conversion of
// v into the common type is monotone (exact, or rounding to nearest). The intervals are sorted and merged, so the device
// tests a row with one binary search. hyb_in_dictionary_matches marks the entries of a string dictionary that the list holds.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <string_view>
#include <type_traits>
#include <vector>

#include "internal.hpp"

namespace hyb {
namespace {

// First v of Column with pred(v) false, where pred holds on a (possibly empty) prefix of the type's range; false if pred
// holds everywhere.
template <typename Column, typename Pred>
bool first_false(Pred pred, Column& out) {
  Column lo = std::numeric_limits<Column>::min(), hi = std::numeric_limits<Column>::max();
  if (pred(hi)) return false;
  using Unsigned = std::make_unsigned_t<Column>;
  while (lo < hi) {
    const Column mid = static_cast<Column>(lo + static_cast<Column>((static_cast<Unsigned>(hi) - static_cast<Unsigned>(lo)) / 2));
    if (pred(mid)) {
      lo = static_cast<Column>(mid + 1);
    } else {
      hi = mid;
    }
  }
  out = lo;
  return true;
}

// The integers of an integer column that equal `element` in the common type: [lo, hi], or false when there is none.
template <typename Column, typename Element>
bool integer_interval(Element element, Column& lo, Column& hi) {
  using Common = std::common_type_t<Column, Element>;
  const Common target = static_cast<Common>(element);
  if (!first_false<Column>([&](Column v) { return static_cast<Common>(v) < target; }, lo)) return false;
  Column above;  // first v with v > element
  if (first_false<Column>([&](Column v) { return !(target < static_cast<Common>(v)); }, above)) {
    if (above == std::numeric_limits<Column>::min()) return false;
    hi = static_cast<Column>(above - 1);
  } else {
    hi = std::numeric_limits<Column>::max();
  }
  return lo <= hi && std::equal_to<Common>{}(static_cast<Common>(lo), target);
}

// The single value of a floating-point column that equals `element` in the common type, or false.
template <typename Column, typename Element>
bool float_point(Element element, Column& value) {
  using Common = std::common_type_t<Column, Element>;
  const Common target = static_cast<Common>(element);
  const Column candidate = static_cast<Column>(target);
  if (!std::equal_to<Common>{}(static_cast<Common>(candidate), target)) return false;  // NaN, or no value of the type
  value = candidate == Column{0} ? Column{0} : candidate;  // -0.0 and +0.0 are one value
  return true;
}

template <typename Column, typename Element>
bool element_interval(Element element, Column& lo, Column& hi) {
  if constexpr (std::is_integral_v<Column>) {
    return integer_interval<Column, Element>(element, lo, hi);
  } else {
    if (!float_point<Column, Element>(element, lo)) return false;
    hi = lo;
    return true;
  }
}

template <typename Column>
bool touches(Column hi, Column next_lo) {
  if (next_lo <= hi) return true;
  if constexpr (std::is_integral_v<Column>) {
    return hi != std::numeric_limits<Column>::max() && next_lo == static_cast<Column>(hi + 1);
  } else {
    return std::nextafter(hi, std::numeric_limits<Column>::infinity()) == next_lo;
  }
}

template <typename Column>
Column& member(hyb_value& value) {
  if constexpr (std::is_same_v<Column, int32_t>) {
    return value.i32;
  } else if constexpr (std::is_same_v<Column, long long>) {
    return reinterpret_cast<long long&>(value.i64);
  } else if constexpr (std::is_same_v<Column, float>) {
    return value.f32;
  } else {
    return value.f64;
  }
}

template <typename Column>
int normalize_typed(const hyb_literal* elements, uint32_t count, std::vector<hyb_value>& out) {
  std::vector<std::pair<Column, Column>> intervals;
  intervals.reserve(count);
  for (uint32_t i = 0; i < count; ++i) {
    Column lo{}, hi{};
    bool found = false;
    switch (elements[i].data_type) {
      case HYB_TYPE_INT32:
        found = element_interval<Column, int32_t>(elements[i].value.i32, lo, hi);
        break;
      case HYB_TYPE_INT64:
        found = element_interval<Column, long long>(static_cast<long long>(elements[i].value.i64), lo, hi);
        break;
      case HYB_TYPE_FLOAT32:
        found = element_interval<Column, float>(elements[i].value.f32, lo, hi);
        break;
      case HYB_TYPE_FLOAT64:
        found = element_interval<Column, double>(elements[i].value.f64, lo, hi);
        break;
      default:
        HYB_CHECK(false, HYB_ERR_INVALID, "IN list element " + std::to_string(i) + " is not numeric");
    }
    if (found) intervals.emplace_back(lo, hi);
  }
  std::sort(intervals.begin(), intervals.end());
  out.clear();
  for (size_t i = 0; i < intervals.size();) {
    Column lo = intervals[i].first, hi = intervals[i].second;
    for (++i; i < intervals.size() && touches(hi, intervals[i].first); ++i) hi = std::max(hi, intervals[i].second);
    hyb_value a{}, b{};
    member<Column>(a) = lo;
    member<Column>(b) = hi;
    out.push_back(a);
    out.push_back(b);
  }
  return HYB_OK;
}

}  // namespace

int normalize_in_list(int32_t column_type, const hyb_literal* elements, uint32_t count, std::vector<hyb_value>& out_bounds) {
  HYB_CHECK(elements || count == 0, HYB_ERR_INVALID, "NULL IN list elements");
  switch (column_type) {
    case HYB_TYPE_INT32:
      return normalize_typed<int32_t>(elements, count, out_bounds);
    case HYB_TYPE_INT64:
      return normalize_typed<long long>(elements, count, out_bounds);
    case HYB_TYPE_FLOAT32:
      return normalize_typed<float>(elements, count, out_bounds);
    case HYB_TYPE_FLOAT64:
      return normalize_typed<double>(elements, count, out_bounds);
    default:
      HYB_CHECK(false, HYB_ERR_INVALID, "IN list intervals need a numeric column");
  }
  return HYB_OK;
}

int in_match_dictionaries(int32_t condition, const LikeDictionary& elements, const LikeDictionary* dictionaries,
                          size_t dictionary_count, uint32_t* out_words, uint64_t* out_match_count) {
  HYB_CHECK(condition == HYB_PRED_IN || condition == HYB_PRED_NOT_IN, HYB_ERR_INVALID,
            "not an IN condition: " + std::to_string(condition));
  const auto valid = [](const LikeDictionary& d) {
    // a list of empty strings has no characters: its `chars` may legitimately be NULL
    return d.count == 0 || (d.offsets && (d.chars || d.offsets[d.count] == d.offsets[0]));
  };
  HYB_CHECK(valid(elements), HYB_ERR_INVALID, "NULL IN list elements");
  for (size_t d = 0; d < dictionary_count; ++d) {
    HYB_CHECK(valid(dictionaries[d]) && (dictionaries[d].count == 0 || out_words), HYB_ERR_INVALID,
              "NULL dictionary or output");
  }
  const auto entry = [](const LikeDictionary& d, uint32_t i) {
    return std::string_view(d.chars ? d.chars + d.offsets[i] : "", d.offsets[i + 1] - d.offsets[i]);
  };
  std::vector<std::string_view> list;
  list.reserve(elements.count);
  for (uint32_t i = 0; i < elements.count; ++i) list.push_back(entry(elements, i));
  std::sort(list.begin(), list.end());
  const bool invert = condition == HYB_PRED_NOT_IN;
  uint64_t matches = 0;
  uint32_t* words = out_words;
  for (size_t d = 0; d < dictionary_count; ++d) {
    const LikeDictionary& dictionary = dictionaries[d];
    for (uint32_t word = 0; word < (dictionary.count + 31) / 32; ++word) words[word] = 0;
    for (uint32_t i = 0; i < dictionary.count; ++i) {
      if (std::binary_search(list.begin(), list.end(), entry(dictionary, i)) != invert) {
        words[i >> 5] |= 1u << (i & 31);
        ++matches;
      }
    }
    words += (dictionary.count + 31) / 32;
  }
  if (out_match_count) *out_match_count = matches;
  return HYB_OK;
}

}  // namespace hyb

using namespace hyb;

extern "C" {

int hyb_in_list_normalize(int32_t column_type, const hyb_literal* elements, uint32_t count, hyb_value* out_bounds,
                          uint32_t* inout_interval_count) {
  HYB_CHECK(inout_interval_count, HYB_ERR_INVALID, "NULL argument");
  std::vector<hyb_value> bounds;
  HYB_TRY(normalize_in_list(column_type, elements, count, bounds));
  const uint32_t intervals = static_cast<uint32_t>(bounds.size() / 2);
  if (out_bounds) {
    HYB_CHECK(*inout_interval_count >= intervals, HYB_ERR_INVALID, "out_bounds holds fewer intervals than the list needs");
    std::copy(bounds.begin(), bounds.end(), out_bounds);
  }
  *inout_interval_count = intervals;
  return HYB_OK;
}

int hyb_in_dictionary_matches(int32_t condition, const char* element_chars, const uint64_t* element_offsets,
                              uint32_t element_count, const char* dictionary_chars, const uint64_t* dictionary_offsets,
                              uint32_t dictionary_count, uint32_t* out_words, uint32_t* out_match_count) {
  const LikeDictionary elements{element_chars, element_offsets, element_count};
  const LikeDictionary dictionary{dictionary_chars, dictionary_offsets, dictionary_count};
  uint64_t matches = 0;
  HYB_TRY(in_match_dictionaries(condition, elements, &dictionary, 1, out_words, &matches));
  if (out_match_count) *out_match_count = static_cast<uint32_t>(matches);
  return HYB_OK;
}

}  // extern "C"
