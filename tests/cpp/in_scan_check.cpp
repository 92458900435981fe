// [NOT] IN TableScans through the C++ mirror (include/hyrise_b200.hpp) on the GPU: a numeric list on an int64 column
// (compared in the common type, so a double element covers two integers and the NULL element empties NOT IN) and a
// string list on a dictionary column (bitmaps from hyb_in_dictionary_matches). Prints "in_scan_check: ok" and exits 0
// when every PosList equals the hand-derived RowIDs.
#include <cstdio>
#include <string>
#include <vector>

#include "hyrise_b200.hpp"

using namespace hyrise_b200;

namespace {

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

std::vector<RowID> scan(const std::shared_ptr<const DeviceTable>& table, InList in_list) {
  TableScan scan(table, std::move(in_list));
  scan.execute();
  return scan.get_output()->row_ids();
}

}  // namespace

int main() {
  auto context = std::make_shared<DeviceContext>(0);
  bool ok = true;

  // int64 values; row 4 is NULL
  const std::vector<int64_t> longs{9007199254740992LL, 9007199254740993LL, 9007199254740994LL, 5, 5, -1};
  const std::vector<uint8_t> nulls{0, 0, 0, 0, 1, 0};
  hyb_segment_desc numbers{};
  numbers.encoding = HYB_ENC_UNENCODED;
  numbers.data_type = HYB_TYPE_INT64;
  numbers.row_count = static_cast<uint32_t>(longs.size());
  numbers.values = longs.data();
  numbers.nulls = nulls.data();
  const hyb_table_view number_view{1, 1, &numbers};
  auto number_table = std::make_shared<const DeviceTable>(context, number_view);
  // 2^53 as a double equals 2^53 and 2^53 + 1 (rounded to double); 5 is an int
  InList numeric{ColumnID{0}, PredicateCondition::In, {AllTypeVariant{9007199254740992.0}, AllTypeVariant{int32_t{5}}}, false, false, {}};
  ok &= expect("int64 IN", scan(number_table, numeric), {{0, 0}, {0, 1}, {0, 3}});
  numeric.condition = PredicateCondition::NotIn;
  ok &= expect("int64 NOT IN", scan(number_table, numeric), {{0, 2}, {0, 5}});
  numeric.has_null_element = true;  // `a NOT IN (..., NULL)` selects nothing
  ok &= expect("int64 NOT IN with NULL", scan(number_table, numeric), {});
  InList empty{ColumnID{0}, PredicateCondition::NotIn, {}, false, false, {}};  // `a NOT IN ()` selects every row, the NULL row included
  ok &= expect("int64 NOT IN ()", scan(number_table, empty), {{0, 0}, {0, 1}, {0, 2}, {0, 3}, {0, 4}, {0, 5}});

  // l_shipmode IN ('MAIL', 'SHIP') on one dictionary chunk; row 5 is NULL (value-ID == dictionary size)
  const std::vector<std::string> entries{"AIR", "MAIL", "RAIL", "SHIP", "TRUCK"};
  std::string chars;
  std::vector<uint64_t> offsets{0};
  for (const auto& entry : entries) {
    chars += entry;
    offsets.push_back(chars.size());
  }
  const std::string list_chars = "MAILSHIP";
  const std::vector<uint64_t> list_offsets{0, 4, 8};
  const std::vector<uint8_t> ids{0, 1, 3, 2, 1, 5, 4};
  hyb_segment_desc strings{};
  strings.encoding = HYB_ENC_DICTIONARY;
  strings.data_type = HYB_TYPE_STRING;
  strings.vector_type = HYB_VEC_FIXED_1B;
  strings.row_count = static_cast<uint32_t>(ids.size());
  strings.dictionary_size = static_cast<uint32_t>(entries.size());
  strings.attribute_vector = ids.data();
  const hyb_table_view string_view{1, 1, &strings};
  auto string_table = std::make_shared<const DeviceTable>(context, string_view);
  for (const auto condition : {PredicateCondition::In, PredicateCondition::NotIn}) {
    InList shipmode{ColumnID{0}, condition, {}, false, true, std::vector<uint32_t>(1)};
    check(hyb_in_dictionary_matches(static_cast<int32_t>(condition), list_chars.data(), list_offsets.data(), 2, chars.data(),
                                    offsets.data(), static_cast<uint32_t>(entries.size()), shipmode.dictionary_matches.data(),
                                    nullptr));
    const std::vector<RowID> want = condition == PredicateCondition::In ? std::vector<RowID>{{0, 1}, {0, 2}, {0, 4}}
                                                                        : std::vector<RowID>{{0, 0}, {0, 3}, {0, 6}};
    ok &= expect(condition == PredicateCondition::In ? "string IN" : "string NOT IN", scan(string_table, shipmode), want);
  }

  if (!ok) return 1;
  std::printf("in_scan_check: ok\n");
  return 0;
}
