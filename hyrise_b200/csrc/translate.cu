// Column-vs-column scans of two string columns: the right dictionary translated into the left one's value-ID space, on
// the host.
//
// ColumnVsColumnTableScanImpl (column_vs_column_table_scan_impl.cpp) compares the two strings of every row. Both
// dictionaries of a chunk are sorted and unique (dictionary_encoder.hpp:33-103), so one merge gives every right entry j
// the key 2 * lower_bound(left, right[j]) + (found ? 1 : 0), while left value-ID i stands for 2 * i + 1. Keys of the two
// sides then order and compare equal exactly as the strings do, and the device compares value-IDs only. Strings never
// reach the GPU.
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

}  // namespace hyb

using namespace hyb;

extern "C" {

int hyb_dictionary_translate(const char* left_chars, const uint64_t* left_offsets, uint32_t left_count,
                             const char* right_chars, const uint64_t* right_offsets, uint32_t right_count,
                             uint32_t* out_words) {
  return translate_dictionary(LikeDictionary{left_chars, left_offsets, left_count},
                              LikeDictionary{right_chars, right_offsets, right_count}, out_words);
}

}  // extern "C"
