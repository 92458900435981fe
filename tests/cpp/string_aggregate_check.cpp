// String MIN / MAX / COUNT and ANY through the C++ mirror's AggregateHash (include/hyrise_b200.hpp) on the GPU, over the
// reference's FixedStringDictionaryMultipleChunks fixture (chunk 0: {"This", "a", "is"}, chunk 1: {"test"}). Bytes
// compare unsigned, so "This" < "a" < "is" < "test". Prints "OK" and exits 0 when the results are the hand-derived ones.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "hyrise_b200.hpp"

using namespace hyrise_b200;

int main() {
  const char* path = std::getenv("HYB_BINARY_FIXTURE");
  if (!path) {
    std::printf("HYB_BINARY_FIXTURE is not set\n");
    return 2;
  }
  auto context = std::make_shared<DeviceContext>(0);
  const BinaryTable file(path);
  auto table = std::make_shared<DeviceTable>(context, file);
  table->set_string_order(0, file.string_order_ranks(0));

  AggregateHash aggregate(std::shared_ptr<const DeviceTable>(table),
                          {AggregateDefinition::on_column(WindowFunction::Min, ColumnID{0}),
                           AggregateDefinition::on_column(WindowFunction::Max, ColumnID{0}),
                           AggregateDefinition::on_column(WindowFunction::Count, ColumnID{0}),
                           AggregateDefinition::on_column(WindowFunction::Any, ColumnID{0})},
                          {});
  aggregate.execute();
  const auto output = aggregate.get_output();
  const auto minimum = output->strings(0, file, 0);
  const auto maximum = output->strings(1, file, 0);
  int32_t type = 0;
  const auto [count, count_nulls] = output->values(2, &type);
  const auto rows = output->group_row_ids();
  const bool ok = output->group_count() == 1 && minimum[0] == std::string("This") && maximum[0] == std::string("test") &&
                  type == HYB_TYPE_INT64 && count[0] == static_cast<double>(table->row_count()) && rows.size() == 1 &&
                  rows[0].chunk_id == 0 && rows[0].chunk_offset == 0;
  if (!ok) {
    std::printf("got %zu groups: min %s max %s count %g\n", static_cast<size_t>(output->group_count()),
                minimum.empty() || !minimum[0] ? "NULL" : minimum[0]->c_str(),
                maximum.empty() || !maximum[0] ? "NULL" : maximum[0]->c_str(), count.empty() ? -1.0 : count[0]);
    return 1;
  }
  std::printf("OK\n");
  return 0;
}
