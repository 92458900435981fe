// Column-vs-column TableScan through the C++ mirror (include/hyrise_b200.hpp) on the GPU: one string pair (two dictionary
// columns, right_in_left from hyb_dictionary_translate) and one numeric pair (int32 x float, compared in float).
// Prints "OK" and exits 0 when both PosLists equal the hand-derived RowIDs.
#include <cstdio>
#include <string>
#include <vector>

#include "hyrise_b200.hpp"

using namespace hyrise_b200;

namespace {

struct StringDictionary {
  std::string chars;
  std::vector<uint64_t> offsets{0};
  explicit StringDictionary(const std::vector<std::string>& entries) {
    for (const auto& entry : entries) {
      chars += entry;
      offsets.push_back(chars.size());
    }
  }
  uint32_t size() const { return static_cast<uint32_t>(offsets.size() - 1); }
};

hyb_segment_desc dictionary_segment(const std::vector<uint8_t>& ids, uint32_t dictionary_size) {
  hyb_segment_desc segment{};
  segment.encoding = HYB_ENC_DICTIONARY;
  segment.data_type = HYB_TYPE_STRING;
  segment.vector_type = HYB_VEC_FIXED_1B;
  segment.row_count = static_cast<uint32_t>(ids.size());
  segment.dictionary_size = dictionary_size;
  segment.attribute_vector = ids.data();
  return segment;
}

bool expect(const char* name, const std::vector<RowID>& got, const std::vector<RowID>& want) {
  bool same = got.size() == want.size();
  for (size_t i = 0; same && i < got.size(); ++i) {
    same = got[i].chunk_id == want[i].chunk_id && got[i].chunk_offset == want[i].chunk_offset;
  }
  if (!same) {
    std::printf("%s: got", name);
    for (const auto& row : got) std::printf(" (%u,%u)", row.chunk_id, row.chunk_offset);
    std::printf("\n");
  }
  return same;
}

}  // namespace

int main() {
  auto context = std::make_shared<DeviceContext>(0);

  // l_commitdate < l_receiptdate on one chunk; row 3 has a NULL receipt date (value-ID == dictionary size)
  const StringDictionary commit({"1994-01-02", "1994-01-05", "1995-03-01"});
  const StringDictionary receipt({"1994-01-01", "1994-01-05", "1995-03-01x"});
  const std::vector<uint8_t> commit_ids{0, 1, 2, 0, 1};
  const std::vector<uint8_t> receipt_ids{0, 1, 2, 3, 2};
  const std::vector<hyb_segment_desc> strings{dictionary_segment(commit_ids, commit.size()),
                                              dictionary_segment(receipt_ids, receipt.size())};
  const hyb_table_view string_view{1, 2, strings.data()};
  auto string_table = std::make_shared<const DeviceTable>(context, string_view);
  ColumnComparison comparison{ColumnID{0}, PredicateCondition::LessThan, ColumnID{1}, std::vector<uint32_t>(receipt.size())};
  check(hyb_dictionary_translate(commit.chars.data(), commit.offsets.data(), commit.size(), receipt.chars.data(),
                                 receipt.offsets.data(), receipt.size(), comparison.right_in_left.data()));
  TableScan string_scan(string_table, comparison);
  string_scan.execute();
  // row 0: 1994-01-02 < 1994-01-01 no; row 1: equal, no; row 2: 1995-03-01 < 1995-03-01x yes (proper prefix);
  // row 3: NULL; row 4: 1994-01-05 < 1995-03-01x yes
  const bool strings_ok = expect("string pair", string_scan.get_output()->row_ids(), {{0, 2}, {0, 4}});

  // int32 = float in float: 16777217 rounds to 16777216.0f
  const std::vector<int32_t> ints{16777217, 1, -3, 7};
  const std::vector<float> floats{16777216.0f, 1.5f, -3.0f, 6.5f};
  std::vector<hyb_segment_desc> numbers(2);
  numbers[0].encoding = HYB_ENC_UNENCODED;
  numbers[0].data_type = HYB_TYPE_INT32;
  numbers[0].row_count = static_cast<uint32_t>(ints.size());
  numbers[0].values = ints.data();
  numbers[1].encoding = HYB_ENC_UNENCODED;
  numbers[1].data_type = HYB_TYPE_FLOAT32;
  numbers[1].row_count = static_cast<uint32_t>(floats.size());
  numbers[1].values = floats.data();
  const hyb_table_view number_view{1, 2, numbers.data()};
  auto number_table = std::make_shared<const DeviceTable>(context, number_view);
  TableScan number_scan(number_table, ColumnComparison{ColumnID{0}, PredicateCondition::Equals, ColumnID{1}, {}});
  number_scan.execute();
  const bool numbers_ok = expect("numeric pair", number_scan.get_output()->row_ids(), {{0, 0}, {0, 2}});

  if (!strings_ok || !numbers_ok) return 1;
  std::printf("OK\n");
  return 0;
}
