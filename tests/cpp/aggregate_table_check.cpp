// AggregateOutput::to_table through the C++ mirror (include/hyrise_b200.hpp) on the GPU: the Q18 shape in miniature.
// GROUP BY k, SUM(q) becomes a table (k at the representative rows, the sum), a HAVING TableScan runs over it, and a semi
// JoinHash of the input onto the HAVING rows keeps the input rows of the surviving keys. Prints "aggregate_table_check: ok"
// and exits 0 when every result equals the one derived from the aggregate's own values.
#include <algorithm>
#include <cstdio>
#include <vector>

#include "hyrise_b200.hpp"

using namespace hyrise_b200;

int main() {
  auto context = std::make_shared<DeviceContext>(0);
  bool ok = true;

  const std::vector<int32_t> k{1, 2, 1, 3, 2, 1, 4};
  const std::vector<int32_t> q{10, 5, 20, 7, 30, 1, 2};
  hyb_segment_desc segments[2]{};
  for (int c = 0; c < 2; ++c) {
    segments[c].encoding = HYB_ENC_UNENCODED;
    segments[c].data_type = HYB_TYPE_INT32;
    segments[c].row_count = static_cast<uint32_t>(k.size());
  }
  segments[0].values = k.data();
  segments[1].values = q.data();
  const hyb_table_view view{1, 2, segments};
  auto input = std::make_shared<const DeviceTable>(context, view);

  constexpr uint32_t kChunkSize = 3;
  std::shared_ptr<const DeviceTable> groups;
  std::vector<double> sums;
  std::vector<RowID> representatives;
  {
    AggregateHash aggregate(input, {AggregateDefinition::on_column(WindowFunction::Sum, ColumnID{1})}, {ColumnID{0}});
    aggregate.execute();
    sums = aggregate.get_output()->values(0).first;
    representatives = aggregate.get_output()->group_row_ids();
    groups = aggregate.get_output()->to_table({{HYB_SORT_KEY_COLUMN, 0}, {HYB_SORT_KEY_AGGREGATE, 0}}, kChunkSize);
  }  // the aggregate's result is freed here: the table does not depend on it
  const auto stats = context->last_operator_stats();
  ok &= stats.input_rows == sums.size() && stats.output_rows == sums.size() && stats.kernel_launches == 1;
  ok &= groups->row_count() == sums.size() && groups->chunk_count() == (sums.size() + kChunkSize - 1) / kChunkSize;
  if (!ok) std::printf("table shape or stats differ\n");

  // HAVING SUM(q) > 10
  auto having = std::make_shared<TableScan>(groups, ScanPredicate{ColumnID{1}, PredicateCondition::GreaterThan,
                                                                  AllTypeVariant{int64_t{10}}, std::nullopt, {}});
  having->execute();
  std::vector<RowID> want_rows;
  std::vector<int32_t> kept_keys;
  for (uint32_t g = 0; g < sums.size(); ++g) {
    if (sums[g] > 10) {
      want_rows.push_back(RowID{g / kChunkSize, g % kChunkSize});
      kept_keys.push_back(k[representatives[g].chunk_offset]);
    }
  }
  const auto got_rows = having->get_output()->row_ids();
  bool same = got_rows.size() == want_rows.size();
  for (size_t i = 0; same && i < got_rows.size(); ++i) {
    same = got_rows[i].chunk_id == want_rows[i].chunk_id && got_rows[i].chunk_offset == want_rows[i].chunk_offset;
  }
  if (!same) std::printf("HAVING: %zu rows, expected %zu\n", got_rows.size(), want_rows.size());
  ok &= same;

  // k IN (SELECT k ... HAVING ...): a semi join of the input onto the HAVING rows of the table
  JoinHash semi(input, OperatorInput{having->get_output()}, JoinMode::Semi, OperatorJoinPredicate{{ColumnID{0}, ColumnID{0}}});
  semi.execute();
  std::vector<uint32_t> got_probe;
  for (const auto& row : semi.get_output()->row_ids().second) got_probe.push_back(row.chunk_offset);
  std::sort(got_probe.begin(), got_probe.end());
  std::vector<uint32_t> want_probe;
  for (uint32_t row = 0; row < k.size(); ++row) {
    if (std::find(kept_keys.begin(), kept_keys.end(), k[row]) != kept_keys.end()) want_probe.push_back(row);
  }
  if (got_probe != want_probe) std::printf("semi join: %zu rows, expected %zu\n", got_probe.size(), want_probe.size());
  ok &= got_probe == want_probe;

  if (!ok) return 1;
  std::printf("aggregate_table_check: ok\n");
  return 0;
}
