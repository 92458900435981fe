#include "device_column_pool.hpp"

#include <cstring>
#include <string>
#include <unordered_map>

#include "resolve_type.hpp"
#include "storage/dictionary_segment.hpp"
#include "storage/frame_of_reference_segment.hpp"
#include "storage/reference_segment.hpp"
#include "storage/value_segment.hpp"
#include "storage/vector_compression/bitpacking/bitpacking_vector.hpp"
#include "storage/vector_compression/fixed_width_integer/fixed_width_integer_vector.hpp"
#include "utils/assert.hpp"

namespace hyrise {

namespace {

template <typename T>
constexpr int32_t hyb_type_of() {
  if constexpr (std::is_same_v<T, int32_t>) return HYB_TYPE_INT32;
  if constexpr (std::is_same_v<T, int64_t>) return HYB_TYPE_INT64;
  if constexpr (std::is_same_v<T, float>) return HYB_TYPE_FLOAT32;
  if constexpr (std::is_same_v<T, double>) return HYB_TYPE_FLOAT64;
  return HYB_TYPE_STRING;
}

// Buffers that exist only for the upload call (pmr_vector<bool> is bit-packed; the ABI wants one byte per row).
struct ChunkScratch {
  std::vector<std::vector<uint8_t>> null_bytes;
  std::vector<std::vector<uint64_t>> dictionary_codes;
};

const uint8_t* expand_nulls(const pmr_vector<bool>& nulls, ChunkScratch& scratch) {
  auto& bytes = scratch.null_bytes.emplace_back(nulls.size());
  for (auto index = size_t{0}; index < nulls.size(); ++index) {
    bytes[index] = nulls[index] ? 1 : 0;
  }
  return bytes.data();
}

// compressed_vector_type.hpp:28-33 -> hyb_vector_type; FixedWidthIntegerVector<T>::data() (fixed_width_integer_vector.hpp:31),
// BitPackingVector::data() is a compact::vector whose get() is the packed word array (bitpacking_vector.hpp:27).
bool describe_vector(const BaseCompressedVector& vector, hyb_segment_desc& desc) {
  switch (vector.type()) {
    case CompressedVectorType::FixedWidthInteger1Byte:
      desc.vector_type = HYB_VEC_FIXED_1B;
      desc.attribute_vector = static_cast<const FixedWidthIntegerVector<uint8_t>&>(vector).data().data();
      return true;
    case CompressedVectorType::FixedWidthInteger2Byte:
      desc.vector_type = HYB_VEC_FIXED_2B;
      desc.attribute_vector = static_cast<const FixedWidthIntegerVector<uint16_t>&>(vector).data().data();
      return true;
    case CompressedVectorType::FixedWidthInteger4Byte:
      desc.vector_type = HYB_VEC_FIXED_4B;
      desc.attribute_vector = static_cast<const FixedWidthIntegerVector<uint32_t>&>(vector).data().data();
      return true;
    case CompressedVectorType::BitPacking: {
      const auto& packed = static_cast<const BitPackingVector&>(vector).data();
      desc.vector_type = HYB_VEC_BITPACKED;
      desc.bit_width = static_cast<int32_t>(packed.bits());
      desc.attribute_vector = packed.get();
      return true;
    }
  }
  return false;
}

// One CHUNK-INDEPENDENT uint64 per dictionary entry of a string column, following AggregateHash's key scheme
// (aggregate_hash.cpp:818-925): strings of up to 5 bytes are their own bytes (tagged immediate), longer ones are numbered by
// a map that lives as long as the column's device copy — the same string gets the same code in every chunk.
using StringIds = std::unordered_map<std::string, uint64_t>;

const uint64_t* string_dictionary_codes(const pmr_vector<pmr_string>& dictionary, StringIds& ids, ChunkScratch& scratch) {
  auto& codes = scratch.dictionary_codes.emplace_back(dictionary.size());
  for (auto index = size_t{0}; index < dictionary.size(); ++index) {
    const auto& value = dictionary[index];
    if (value.size() <= 5) {
      auto packed = uint64_t{0};
      std::memcpy(&packed, value.data(), value.size());
      codes[index] = (packed << 8) | (uint64_t{value.size()} << 1) | 1u;  // tag bit: immediate
    } else {
      const auto [iter, inserted] = ids.try_emplace(std::string{value}, uint64_t{ids.size()});
      codes[index] = iter->second << 1;
    }
  }
  return codes.data();
}

bool describe_segment(const AbstractSegment& segment, hyb_segment_desc& desc, StringIds& string_ids, ChunkScratch& scratch) {
  auto supported = true;
  desc = hyb_segment_desc{};
  desc.row_count = static_cast<uint32_t>(segment.size());
  resolve_data_and_segment_type(segment, [&](const auto data_type_t, const auto& typed_segment) {
    using ColumnDataType = typename decltype(data_type_t)::type;
    using SegmentType = std::decay_t<decltype(typed_segment)>;
    desc.data_type = hyb_type_of<ColumnDataType>();
    if constexpr (std::is_same_v<SegmentType, ValueSegment<ColumnDataType>>) {
      if constexpr (std::is_same_v<ColumnDataType, pmr_string>) {
        supported = false;  // unencoded strings stay on the CPU
      } else {
        desc.encoding = HYB_ENC_UNENCODED;
        desc.values = typed_segment.values().data();  // value_segment.hpp:52
        if (typed_segment.is_nullable()) {
          desc.nulls = expand_nulls(typed_segment.null_values(), scratch);  // value_segment.hpp:62
        }
      }
    } else if constexpr (std::is_same_v<SegmentType, DictionarySegment<ColumnDataType>>) {
      desc.encoding = HYB_ENC_DICTIONARY;
      desc.dictionary_size = typed_segment.unique_values_count();  // == null_value_id(), dictionary_segment.hpp:79-83
      if constexpr (std::is_same_v<ColumnDataType, pmr_string>) {
        desc.dictionary_codes = string_dictionary_codes(*typed_segment.dictionary(), string_ids, scratch);
      } else {
        desc.values = typed_segment.dictionary()->data();  // dictionary_segment.hpp:26
      }
      supported = describe_vector(*typed_segment.attribute_vector(), desc);
    } else if constexpr (std::is_same_v<SegmentType, FrameOfReferenceSegment<ColumnDataType>>) {
      desc.encoding = HYB_ENC_FRAME_OF_REFERENCE;
      desc.values = typed_segment.block_minima().data();  // frame_of_reference_segment.hpp:54
      supported = describe_vector(typed_segment.offset_values(), desc);
      if (typed_segment.null_values()) {
        desc.nulls = expand_nulls(*typed_segment.null_values(), scratch);
      }
    } else {
      supported = false;  // RunLength, LZ4, FixedStringDictionary, ReferenceSegment
    }
  });
  return supported;
}

}  // namespace

DeviceColumnPool::~DeviceColumnPool() {
  for (const auto& [table, entry] : _entries) {
    hyb_table_drop(_context, entry.handle);
  }
}

bool DeviceColumnPool::upload(const std::shared_ptr<const Table>& table) {
  if (table->type() != TableType::Data) {
    return false;
  }
  const auto lock = std::lock_guard<std::mutex>{_mutex};
  auto& entry = _entries[table.get()];
  const auto column_count = static_cast<uint32_t>(table->column_count());
  if (entry.handle == 0 && hyb_table_create(_context, column_count, &entry.handle) != HYB_OK) {
    _entries.erase(table.get());
    return false;
  }
  const auto chunk_count = table->chunk_count();
  for (auto chunk_id = entry.uploaded_chunks; chunk_id < chunk_count; ++chunk_id) {
    const auto chunk = table->get_chunk(chunk_id);
    if (!chunk || chunk->is_mutable()) {
      break;  // the mutable tail chunk stays on the CPU; chunks are appended in order
    }
    auto scratch = ChunkScratch{};
    auto descs = std::vector<hyb_segment_desc>(column_count);
    for (auto column_id = ColumnID{0}; column_id < column_count; ++column_id) {
      if (entry.string_ids.size() < column_count) {
        entry.string_ids.resize(column_count);
      }
      if (!describe_segment(*chunk->get_segment(column_id), descs[column_id], entry.string_ids[column_id], scratch)) {
        hyb_table_drop(_context, entry.handle);
        _entries.erase(table.get());
        return false;
      }
    }
    const auto status = hyb_table_append_chunk(_context, entry.handle, descs.data());  // copies every buffer; borrowed for the call
    Assert(status == HYB_OK, hyb_last_error());
    entry.uploaded_chunks = ChunkID{static_cast<uint32_t>(chunk_id) + 1};
    entry.ordered.assign(column_count, false);  // the library dropped the order ranks with the new chunk
  }
  return true;
}

bool DeviceColumnPool::ensure_string_order(const std::shared_ptr<const Table>& table, ColumnID column_id) {
  if (table->column_data_type(column_id) != DataType::String) {
    return false;
  }
  const auto lock = std::lock_guard<std::mutex>{_mutex};
  const auto iter = _entries.find(table.get());
  if (iter == _entries.end() || iter->second.uploaded_chunks != table->chunk_count()) {
    return false;
  }
  auto& entry = iter->second;
  entry.ordered.resize(table->column_count(), false);
  if (entry.ordered[column_id]) {
    return true;
  }
  // the dictionaries of the uploaded chunks in the layout of hyb_dictionary_order_ranks (one k-way merge on the host)
  const auto chunk_count = table->chunk_count();
  auto chars = std::vector<std::string>(chunk_count);
  auto offsets = std::vector<std::vector<uint64_t>>(chunk_count);
  auto char_pointers = std::vector<const char*>(chunk_count);
  auto offset_pointers = std::vector<const uint64_t*>(chunk_count);
  auto counts = std::vector<uint32_t>(chunk_count);
  auto total = uint64_t{0};
  for (auto chunk_id = ChunkID{0}; chunk_id < chunk_count; ++chunk_id) {
    const auto segment =
        std::dynamic_pointer_cast<const DictionarySegment<pmr_string>>(table->get_chunk(chunk_id)->get_segment(column_id));
    if (!segment) {
      return false;
    }
    const auto& dictionary = *segment->dictionary();
    offsets[chunk_id].push_back(0);
    for (const auto& value : dictionary) {
      chars[chunk_id].append(value.data(), value.size());
      offsets[chunk_id].push_back(chars[chunk_id].size());
    }
    char_pointers[chunk_id] = chars[chunk_id].data();
    offset_pointers[chunk_id] = offsets[chunk_id].data();
    counts[chunk_id] = static_cast<uint32_t>(dictionary.size());
    total += dictionary.size();
  }
  auto ranks = std::vector<uint32_t>(total);
  const auto status = hyb_dictionary_order_ranks(static_cast<uint32_t>(chunk_count), char_pointers.data(), offset_pointers.data(),
                                                 counts.data(), ranks.data(), nullptr);
  if (status == HYB_ERR_UNSUPPORTED) {
    return false;
  }
  Assert(status == HYB_OK, hyb_last_error());
  Assert(hyb_table_set_string_order(_context, entry.handle, column_id, ranks.data(), total) == HYB_OK, hyb_last_error());
  entry.ordered[column_id] = true;
  return true;
}

const DeviceColumnPool::Entry* DeviceColumnPool::find(const std::shared_ptr<const Table>& table,
                                                      std::shared_ptr<const Table>* out_referenced) const {
  const auto lock = std::lock_guard<std::mutex>{_mutex};
  auto stored = table;
  if (table->type() == TableType::References) {
    // every segment of every chunk must reference the same stored table (what a chain of TableScans produces)
    stored = nullptr;
    const auto chunk_count = table->chunk_count();
    for (auto chunk_id = ChunkID{0}; chunk_id < chunk_count; ++chunk_id) {
      const auto chunk = table->get_chunk(chunk_id);
      for (auto column_id = ColumnID{0}; column_id < table->column_count(); ++column_id) {
        const auto reference = std::dynamic_pointer_cast<const ReferenceSegment>(chunk->get_segment(column_id));
        if (!reference || (stored && reference->referenced_table() != stored)) {
          return nullptr;
        }
        stored = reference->referenced_table();
      }
    }
    if (!stored) {
      return nullptr;
    }
  }
  const auto iter = _entries.find(stored.get());
  if (iter == _entries.end() || iter->second.uploaded_chunks != stored->chunk_count()) {
    return nullptr;  // not uploaded, or a mutable tail the device copy does not hold
  }
  if (out_referenced) {
    *out_referenced = stored;
  }
  return &iter->second;
}

}  // namespace hyrise
