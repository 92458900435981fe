// JoinHash with a secondary predicate through the C++ mirror (include/hyrise_b200.hpp) on the GPU: `l.k = r.k AND
// l.x < r.y` (int32 x float, compared in float) as an Inner join built on the left input, as an Inner join built on the
// right input (the predicate flipped to `r.y > l.x`), and as a Semi join (right input builds, flipped). Prints "OK" and
// exits 0 when every output equals the hand-derived RowIDs; an AntiNullAsTrue join must throw UnsupportedOnDevice.
#include <algorithm>
#include <cstdio>
#include <vector>

#include "hyrise_b200.hpp"

using namespace hyrise_b200;

namespace {

hyb_segment_desc plain_segment(int32_t data_type, const void* values, uint32_t rows) {
  hyb_segment_desc segment{};
  segment.encoding = HYB_ENC_UNENCODED;
  segment.data_type = data_type;
  segment.row_count = rows;
  segment.values = values;
  return segment;
}

using Pair = std::pair<std::pair<uint32_t, uint32_t>, std::pair<uint32_t, uint32_t>>;  // {left RowID, right RowID}

std::vector<Pair> left_right_pairs(const JoinOutput& output) {
  const auto [build, probe] = output.row_ids();
  std::vector<Pair> pairs;
  for (size_t i = 0; i < probe.size(); ++i) {
    const RowID& left = output.left_is_build ? build[i] : probe[i];
    const RowID& right = output.left_is_build ? probe[i] : build[i];
    pairs.push_back({{left.chunk_id, left.chunk_offset}, {right.chunk_id, right.chunk_offset}});
  }
  std::sort(pairs.begin(), pairs.end());
  return pairs;
}

bool expect(const char* name, bool ok) {
  if (!ok) std::printf("%s: unexpected output\n", name);
  return ok;
}

}  // namespace

int main() {
  auto context = std::make_shared<DeviceContext>(0);
  // small: k = {1, 2, 2}, x = {5, 16777217, 3}; large: k = {2, 2, 1, 1, 9}, y = {16777216, 4, 6, 5, 0}
  const std::vector<int32_t> small_keys{1, 2, 2}, small_x{5, 16777217, 3};
  const std::vector<int32_t> large_keys{2, 2, 1, 1, 9};
  const std::vector<float> large_y{16777216.0f, 4.0f, 6.0f, 5.0f, 0.0f};
  const std::vector<hyb_segment_desc> small_segments{plain_segment(HYB_TYPE_INT32, small_keys.data(), 3),
                                                     plain_segment(HYB_TYPE_INT32, small_x.data(), 3)};
  const std::vector<hyb_segment_desc> large_segments{plain_segment(HYB_TYPE_INT32, large_keys.data(), 5),
                                                     plain_segment(HYB_TYPE_FLOAT32, large_y.data(), 5)};
  auto small = std::make_shared<const DeviceTable>(context, hyb_table_view{1, 2, small_segments.data()});
  auto large = std::make_shared<const DeviceTable>(context, hyb_table_view{1, 2, large_segments.data()});
  const OperatorJoinPredicate primary{{ColumnID{0}, ColumnID{0}}, PredicateCondition::Equals};

  // small.x < large.y: (1:5) with (1:6); (2:3) with (2:16777216) and (2:4); 16777217 rounds to 16777216.0f, not less
  const std::vector<Pair> expected{{{0, 0}, {0, 2}}, {{0, 2}, {0, 0}}, {{0, 2}, {0, 1}}};
  JoinHash left_builds(small, large, JoinMode::Inner, primary, {{{ColumnID{1}, ColumnID{1}}, PredicateCondition::LessThan}});
  left_builds.execute();
  bool ok = expect("inner, left builds", left_builds.get_output()->left_is_build &&
                                           left_right_pairs(*left_builds.get_output()) == expected);

  // large.y > small.x with the large input on the left: the right input builds, the predicate is flipped
  std::vector<Pair> swapped;
  for (const auto& [l, r] : expected) swapped.push_back({r, l});
  std::sort(swapped.begin(), swapped.end());
  JoinHash right_builds(large, small, JoinMode::Inner, primary, {{{ColumnID{1}, ColumnID{1}}, PredicateCondition::GreaterThan}});
  right_builds.execute();
  ok &= expect("inner, right builds", !right_builds.get_output()->left_is_build &&
                                          left_right_pairs(*right_builds.get_output()) == swapped);

  // Semi: small rows with some large row of their key and x < y -> rows 0 and 2
  JoinHash semi(small, large, JoinMode::Semi, primary, {{{ColumnID{1}, ColumnID{1}}, PredicateCondition::LessThan}}, 0);
  semi.execute();
  const auto semi_rows = semi.get_output()->row_ids().second;
  ok &= expect("semi", semi_rows.size() == 2 && semi_rows[0].chunk_offset == 0 && semi_rows[1].chunk_offset == 2);

  bool unsupported = false;
  try {
    JoinHash anti(small, large, JoinMode::AntiNullAsTrue, primary, {{{ColumnID{1}, ColumnID{1}}, PredicateCondition::LessThan}});
    anti.execute();
  } catch (const UnsupportedOnDevice&) {
    unsupported = true;
  }
  ok &= expect("anti null as true", unsupported);

  if (!ok) return 1;
  std::printf("OK\n");
  return 0;
}
