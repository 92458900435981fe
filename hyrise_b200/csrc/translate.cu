// Column-vs-column scans of two string columns: the right dictionary translated into the left one's value-ID space, on
// the host.
//
// ColumnVsColumnTableScanImpl (column_vs_column_table_scan_impl.cpp) compares the two strings of every row. Both
// dictionaries of a chunk are sorted and unique (dictionary_encoder.hpp:33-103), so one merge gives every right entry j
// the key 2 * lower_bound(left, right[j]) + (found ? 1 : 0), while left value-ID i stands for 2 * i + 1. Keys of the two
// sides then order and compare equal exactly as the strings do, and the device compares value-IDs only. Strings never
// reach the GPU.
#include <queue>
#include <string>
#include <string_view>
#include <vector>

#include "internal.hpp"

namespace hyb {

int translate_dictionary(const LikeDictionary& left, const LikeDictionary& right, uint32_t* out_words) {
  HYB_CHECK(left.count < (1u << 31) && right.count < (1u << 31), HYB_ERR_UNSUPPORTED,
            "column-vs-column scans need dictionaries of fewer than 2^31 entries");
  for (const LikeDictionary* dictionary : {&left, &right}) {
    HYB_CHECK(dictionary->count == 0 || dictionary->offsets, HYB_ERR_INVALID, "NULL dictionary offsets");
    // a dictionary of empty strings has no characters: its `chars` may legitimately be NULL
    HYB_CHECK(dictionary->count == 0 || dictionary->chars || dictionary->offsets[dictionary->count] == dictionary->offsets[0],
              HYB_ERR_INVALID, "NULL dictionary characters");
  }
  HYB_CHECK(right.count == 0 || out_words, HYB_ERR_INVALID, "NULL output");
  const auto entry = [](const LikeDictionary& dictionary, uint32_t index) {
    const char* chars = dictionary.chars ? dictionary.chars : "";
    return std::string_view(chars + dictionary.offsets[index], dictionary.offsets[index + 1] - dictionary.offsets[index]);
  };
  // std::string_view::compare is std::char_traits<char>::compare: bytes as unsigned char, a proper prefix first
  uint32_t i = 0;
  for (uint32_t j = 0; j < right.count; ++j) {
    const std::string_view value = entry(right, j);
    while (i < left.count && entry(left, i).compare(value) < 0) ++i;
    const bool found = i < left.count && entry(left, i).compare(value) == 0;
    out_words[j] = 2 * i + (found ? 1u : 0u);
  }
  return HYB_OK;
}

// MIN / MAX over a string column compare strings of different chunks, whose value-IDs are chunk-local. One k-way merge
// of the sorted per-chunk dictionaries gives every entry its dense rank among the column's distinct strings; ranks order
// exactly as the strings do (char_traits<char>::compare), so the device takes MIN / MAX of rank words instead.
int order_rank_dictionaries(const LikeDictionary* dictionaries, size_t dictionary_count, uint32_t* out_ranks,
                            uint32_t* out_distinct_count) {
  HYB_CHECK(dictionaries || dictionary_count == 0, HYB_ERR_INVALID, "NULL dictionaries");
  std::vector<uint64_t> base(dictionary_count + 1, 0);
  for (size_t d = 0; d < dictionary_count; ++d) {
    const LikeDictionary& dictionary = dictionaries[d];
    HYB_CHECK(dictionary.count == 0 || dictionary.offsets, HYB_ERR_INVALID, "NULL dictionary offsets");
    HYB_CHECK(dictionary.count == 0 || dictionary.chars || dictionary.offsets[dictionary.count] == dictionary.offsets[0],
              HYB_ERR_INVALID, "NULL dictionary characters");
    base[d + 1] = base[d] + dictionary.count;
  }
  HYB_CHECK(base.back() == 0 || out_ranks, HYB_ERR_INVALID, "NULL output");
  const auto entry = [&](size_t d, uint32_t index) {
    const char* chars = dictionaries[d].chars ? dictionaries[d].chars : "";
    const uint64_t* offsets = dictionaries[d].offsets;
    return std::string_view(chars + offsets[index], offsets[index + 1] - offsets[index]);
  };
  for (size_t d = 0; d < dictionary_count; ++d) {
    for (uint32_t i = 1; i < dictionaries[d].count; ++i) {
      HYB_CHECK(entry(d, i - 1).compare(entry(d, i)) < 0, HYB_ERR_INVALID,
                "dictionary " + std::to_string(d) + " is not strictly increasing at entry " + std::to_string(i));
    }
  }
  // heap of {dictionary, next entry}: the smallest string on top, ties in dictionary order
  using Cursor = std::pair<size_t, uint32_t>;
  const auto after = [&](const Cursor& a, const Cursor& b) {
    const int order = entry(a.first, a.second).compare(entry(b.first, b.second));
    return order > 0 || (order == 0 && a.first > b.first);
  };
  std::priority_queue<Cursor, std::vector<Cursor>, decltype(after)> heap(after);
  for (size_t d = 0; d < dictionary_count; ++d) {
    if (dictionaries[d].count) heap.push({d, 0});
  }
  uint64_t distinct = 0;
  std::string_view previous;
  while (!heap.empty()) {
    const Cursor top = heap.top();
    heap.pop();
    const std::string_view value = entry(top.first, top.second);
    if (distinct == 0 || value != previous) {
      HYB_CHECK(distinct < (uint64_t{1} << 31), HYB_ERR_UNSUPPORTED, "a column of 2^31 or more distinct strings");
      ++distinct;
      previous = value;
    }
    out_ranks[base[top.first] + top.second] = static_cast<uint32_t>(distinct - 1);
    if (top.second + 1 < dictionaries[top.first].count) heap.push({top.first, top.second + 1});
  }
  if (out_distinct_count) *out_distinct_count = static_cast<uint32_t>(distinct);
  return HYB_OK;
}

}  // namespace hyb

using namespace hyb;

extern "C" {

int hyb_dictionary_order_ranks(uint32_t dictionary_count, const char* const* chars, const uint64_t* const* offsets,
                               const uint32_t* counts, uint32_t* out_ranks, uint32_t* out_distinct_count) {
  HYB_CHECK(dictionary_count == 0 || (chars && offsets && counts), HYB_ERR_INVALID, "NULL argument");
  std::vector<LikeDictionary> dictionaries(dictionary_count);
  for (uint32_t d = 0; d < dictionary_count; ++d) dictionaries[d] = LikeDictionary{chars[d], offsets[d], counts[d]};
  return order_rank_dictionaries(dictionaries.data(), dictionaries.size(), out_ranks, out_distinct_count);
}

int hyb_dictionary_translate(const char* left_chars, const uint64_t* left_offsets, uint32_t left_count,
                             const char* right_chars, const uint64_t* right_offsets, uint32_t right_count,
                             uint32_t* out_words) {
  return translate_dictionary(LikeDictionary{left_chars, left_offsets, left_count},
                              LikeDictionary{right_chars, right_offsets, right_count}, out_words);
}

}  // extern "C"
