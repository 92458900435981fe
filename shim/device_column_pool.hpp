#pragma once

#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "hyrise_b200.h"
#include "storage/table.hpp"

namespace hyrise {

// The device-resident copies of stored tables (TableType::Data). One pool per process, owned by the plugin.
class DeviceColumnPool {
 public:
  explicit DeviceColumnPool(hyb_context* context) : _context{context} {}
  ~DeviceColumnPool();

  // Uploads all immutable chunks of `table` that are not on the device yet (idempotent; call again after new chunks were
  // finalized). Tables holding a segment type the device path does not read (RunLength, LZ4, FixedStringDictionary) are
  // skipped: their operators keep running on the CPU.
  bool upload(const std::shared_ptr<const Table>& table);

  struct Entry {
    hyb_table_t handle{0};
    ChunkID uploaded_chunks{0};
    std::vector<std::unordered_map<std::string, uint64_t>> string_ids;  // per column: group-by codes of long strings
    std::vector<bool> ordered;  // per column: order ranks attached (hyb_table_set_string_order; appending drops them)
  };

  // The device table of a stored table, or of the single stored table all ReferenceSegments of `table` point to (then
  // `out_referenced` is that table); nullptr if there is none.
  const Entry* find(const std::shared_ptr<const Table>& table, std::shared_ptr<const Table>* out_referenced = nullptr) const;

  // Computes and attaches the order ranks string MIN / MAX need, once per uploaded string column (after new chunks, again).
  // false: the column is no string dictionary column of an uploaded table, or the ranks do not fit (2^31 strings).
  bool ensure_string_order(const std::shared_ptr<const Table>& table, ColumnID column_id);

  hyb_context* context() const {
    return _context;
  }

 private:
  hyb_context* _context;
  mutable std::mutex _mutex;
  std::unordered_map<const Table*, Entry> _entries;
};

}  // namespace hyrise
