// Loading path (SURVEY.md 8 f4): Hyrise's binary table format -> host segments in the device pool's layout, in a few large
// pinned host blocks, ready for one DMA per block (hyb_blocks_upload) — the native counterpart of
// hyrise_b200/binary_table.py (the two are compared file by file in tests/test_binary_table.py).
//
// Follows BinaryParser::parse (import_export/binary/binary_parser.cpp:40-344; format tables in binary_writer.hpp:25-230):
//   header   chunk size u32 | chunk count u32 | column count u16 | type names | nullable flags | column names
//            (strings are stored as `size_t lengths[count]` followed by the concatenated characters, :83-96, :106-111)
//   chunk    row count u32 | sorted-column count u32 | {column id u16, sort mode u8} ... | one segment per column (:126-148)
//   segment  EncodingType u8 (storage/encoding_type.hpp:26) + payload (:168-344)
// ValueSegment / DictionarySegment / FrameOfReferenceSegment keep the reference's encoding (FixedWidthInteger and BitPacking
// vectors as stored); RunLengthSegments are expanded to ValueSegments, FixedStringDictionarySegments and unencoded string
// segments become string DictionarySegments; LZ4 -> HYB_ERR_UNSUPPORTED (not on the device path). Host code only.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "internal.hpp"

namespace hyb {
namespace {

constexpr size_t kLoaderBlockBytes = size_t{64} << 20;
constexpr size_t kLoaderAlign = 256;
constexpr size_t kLoaderTailPad = 64;  // kernels may read one 16-byte vector past the last element

enum : uint8_t { kFileUnencoded = 0, kFileDictionary, kFileRunLength, kFileFixedString, kFileFrameOfReference, kFileLZ4 };
enum : uint8_t { kFileBitPacking = 0, kFileFixed1, kFileFixed2, kFileFixed4 };  // compressed_vector_type.hpp:28-33

struct FormatError {
  int status;
  std::string message;
};

// Blocks of host memory with 256-byte aligned slots; pinned (cudaHostAlloc) when a CUDA device is usable, so that the blocks
// can be handed to hyb_blocks_upload as they are.
class LoaderArena {
 public:
  explicit LoaderArena(bool pinned) : _pinned(pinned) {}
  ~LoaderArena() {
    for (auto& block : _blocks) {
      if (block.pinned) {
        cudaFreeHost(block.base);
      } else {
        std::free(block.base);
      }
    }
  }
  void* place(const void* source, size_t bytes) {
    const size_t need = (bytes + kLoaderTailPad + kLoaderAlign - 1) / kLoaderAlign * kLoaderAlign;
    if (_blocks.empty() || _blocks.back().used + need > _blocks.back().size) new_block(need);
    auto& block = _blocks.back();
    char* slot = block.base + block.used;
    block.used += need;
    if (bytes) std::memcpy(slot, source, bytes);
    std::memset(slot + bytes, 0, need - bytes);
    return slot;
  }
  std::vector<hyb_host_block> host_blocks() const {
    std::vector<hyb_host_block> out;
    for (const auto& block : _blocks) {
      if (block.used) out.push_back(hyb_host_block{block.base, block.used});
    }
    return out;
  }

 private:
  struct Block {
    char* base;
    size_t size, used;
    bool pinned;
  };
  void new_block(size_t need) {
    const size_t size = std::max(need, kLoaderBlockBytes);
    void* base = nullptr;
    bool pinned = false;
    if (_pinned && cudaHostAlloc(&base, size, cudaHostAllocPortable) == cudaSuccess) {
      pinned = true;
    } else {
      cudaGetLastError();
      _pinned = false;  // no usable device (CPU-only parse): page-aligned pageable memory
      base = std::aligned_alloc(4096, (size + 4095) / 4096 * 4096);
      if (!base) throw FormatError{HYB_ERR_OOM, "out of host memory"};
    }
    _blocks.push_back({static_cast<char*>(base), size, 0, pinned});
  }
  std::vector<Block> _blocks;
  bool _pinned;
};

struct Reader {
  const unsigned char* data;
  size_t size, position = 0;
  const unsigned char* take(size_t count) {
    if (position + count > size || position + count < position) throw FormatError{HYB_ERR_INVALID, "unexpected end of file"};
    const unsigned char* at = data + position;
    position += count;
    return at;
  }
  template <typename T>
  T value() {
    T out;
    std::memcpy(&out, take(sizeof(T)), sizeof(T));
    return out;
  }
  std::vector<std::string> strings(size_t count) {  // size_t lengths, then the characters (binary_parser.cpp:83-96)
    std::vector<uint64_t> lengths(count);
    if (count) std::memcpy(lengths.data(), take(sizeof(uint64_t) * count), sizeof(uint64_t) * count);
    std::vector<std::string> out(count);
    for (size_t index = 0; index < count; ++index) {
      const unsigned char* chars = take(lengths[index]);
      out[index].assign(reinterpret_cast<const char*>(chars), lengths[index]);
    }
    return out;
  }
};

// AggregateHash's key scheme for string group-by columns (aggregate_hash.cpp:852-925), chunk independent: strings shorter than
// five characters are packed, longer ones get ids from 5 000 000 000 in order of first appearance in this column.
struct StringIds {
  std::map<std::string, uint64_t> ids;
  uint64_t next = 5'000'000'000ull;
  uint64_t code(const std::string& value) {
    if (value.size() < 5) {
      static const uint64_t base[5] = {1, 2, 258, 65'794, 16'843'010};
      uint64_t code = base[value.size()];
      for (size_t i = 0; i < value.size(); ++i) code += static_cast<uint64_t>(static_cast<unsigned char>(value[i])) << (8 * i);
      return code;
    }
    const auto inserted = ids.emplace(value, next);
    if (inserted.second) ++next;
    return inserted.first->second;
  }
};

struct StringDictionary {
  std::vector<char> chars;
  std::vector<uint64_t> offsets;  // count + 1
};

}  // namespace
}  // namespace hyb

using namespace hyb;

struct hyb_binary_table {
  explicit hyb_binary_table(bool pinned) : arena(pinned) {}
  LoaderArena arena;
  uint32_t chunk_size = 0;
  std::vector<std::string> column_names;
  std::vector<int32_t> column_types;
  std::vector<uint8_t> column_nullable;
  std::vector<uint32_t> chunk_rows;
  std::vector<hyb_segment_desc> segments;                         // chunk-major
  std::vector<StringDictionary> string_dictionaries;               // chunk-major; empty for numeric columns
  std::vector<std::vector<std::pair<uint16_t, uint8_t>>> sorted;   // per chunk: (column id, SortMode)
  std::vector<StringIds> string_ids;                               // per column
  std::vector<hyb_host_block> blocks;
};

namespace {

size_t type_size(int32_t data_type) { return data_type == HYB_TYPE_INT32 || data_type == HYB_TYPE_FLOAT32 ? 4 : 8; }

void read_vector(Reader& reader, uint8_t vector_type, uint32_t rows, hyb_binary_table& table, hyb_segment_desc& desc) {
  size_t bytes = 0;
  switch (vector_type) {
    case kFileBitPacking: {
      desc.vector_type = HYB_VEC_BITPACKED;
      desc.bit_width = reader.value<uint8_t>();
      if (desc.bit_width < 1 || desc.bit_width > 32) throw FormatError{HYB_ERR_INVALID, "bit width of a BitPackingVector out of range"};
      bytes = (static_cast<size_t>(rows) * desc.bit_width + 63) / 64 * 8;  // compact::vector::bytes(): whole 64-bit words
      break;
    }
    case kFileFixed1:
      desc.vector_type = HYB_VEC_FIXED_1B;
      bytes = rows;
      break;
    case kFileFixed2:
      desc.vector_type = HYB_VEC_FIXED_2B;
      bytes = size_t{rows} * 2;
      break;
    case kFileFixed4:
      desc.vector_type = HYB_VEC_FIXED_4B;
      bytes = size_t{rows} * 4;
      break;
    default:
      throw FormatError{HYB_ERR_INVALID, "cannot import attribute vector with compressed vector type id " + std::to_string(vector_type)};
  }
  desc.attribute_vector = table.arena.place(reader.take(bytes), bytes);
}

// String values -> sorted unique dictionary + value-IDs (NULL = dictionary size), as DictionaryEncoder does
// (dictionary_encoder.hpp:33-110). `values[i]` is ignored where nulls[i].
void dictionary_encode_strings(const std::vector<std::string>& values, const std::vector<uint8_t>& nulls, hyb_binary_table& table,
                               uint32_t column, hyb_segment_desc& desc, StringDictionary& dictionary) {
  std::vector<std::string> unique;
  for (size_t i = 0; i < values.size(); ++i) {
    if (nulls.empty() || !nulls[i]) unique.push_back(values[i]);
  }
  std::sort(unique.begin(), unique.end());
  unique.erase(std::unique(unique.begin(), unique.end()), unique.end());
  const uint32_t size = static_cast<uint32_t>(unique.size());
  std::vector<uint32_t> ids(values.size(), size);
  for (size_t i = 0; i < values.size(); ++i) {
    if (nulls.empty() || !nulls[i]) ids[i] = static_cast<uint32_t>(std::lower_bound(unique.begin(), unique.end(), values[i]) - unique.begin());
  }
  desc.encoding = HYB_ENC_DICTIONARY;
  desc.dictionary_size = size;
  if (size <= 0xFF) {  // FixedWidthIntegerCompressor: the largest value that can occur is the NULL value-ID
    std::vector<uint8_t> narrow(ids.begin(), ids.end());
    desc.vector_type = HYB_VEC_FIXED_1B;
    desc.attribute_vector = table.arena.place(narrow.data(), narrow.size());
  } else if (size <= 0xFFFF) {
    std::vector<uint16_t> narrow(ids.begin(), ids.end());
    desc.vector_type = HYB_VEC_FIXED_2B;
    desc.attribute_vector = table.arena.place(narrow.data(), narrow.size() * 2);
  } else {
    desc.vector_type = HYB_VEC_FIXED_4B;
    desc.attribute_vector = table.arena.place(ids.data(), ids.size() * 4);
  }
  dictionary.offsets.assign(1, 0);
  std::vector<uint64_t> codes(size);
  for (uint32_t i = 0; i < size; ++i) {
    dictionary.chars.insert(dictionary.chars.end(), unique[i].begin(), unique[i].end());
    dictionary.offsets.push_back(dictionary.chars.size());
    codes[i] = table.string_ids[column].code(unique[i]);
  }
  desc.dictionary_codes = static_cast<const uint64_t*>(table.arena.place(codes.data(), codes.size() * 8));
}

void string_dictionary_from_entries(const std::vector<std::string>& entries, hyb_binary_table& table, uint32_t column,
                                    hyb_segment_desc& desc, StringDictionary& dictionary) {
  dictionary.offsets.assign(1, 0);
  std::vector<uint64_t> codes(entries.size());
  for (size_t i = 0; i < entries.size(); ++i) {
    dictionary.chars.insert(dictionary.chars.end(), entries[i].begin(), entries[i].end());
    dictionary.offsets.push_back(dictionary.chars.size());
    codes[i] = table.string_ids[column].code(entries[i]);
  }
  desc.dictionary_codes = static_cast<const uint64_t*>(table.arena.place(codes.data(), codes.size() * 8));
}

void read_segment(Reader& reader, uint32_t rows, uint32_t column, hyb_binary_table& table, hyb_segment_desc& desc,
                  StringDictionary& dictionary) {
  const int32_t data_type = table.column_types[column];
  const bool is_string = data_type == HYB_TYPE_STRING;
  const bool nullable = table.column_nullable[column] != 0;
  desc = hyb_segment_desc{};
  desc.data_type = data_type;
  desc.row_count = rows;
  const uint8_t encoding = reader.value<uint8_t>();
  switch (encoding) {
    case kFileUnencoded: {
      std::vector<uint8_t> nulls;
      if (nullable && reader.value<uint8_t>()) {  // "segment nullable" is only written for nullable columns
        const unsigned char* flags = reader.take(rows);
        nulls.assign(flags, flags + rows);
      }
      if (is_string) {  // strings reach the device as value-IDs
        dictionary_encode_strings(reader.strings(rows), nulls, table, column, desc, dictionary);
        return;
      }
      desc.encoding = HYB_ENC_UNENCODED;
      const size_t bytes = size_t{rows} * type_size(data_type);
      desc.values = table.arena.place(reader.take(bytes), bytes);
      if (nullable) {
        if (nulls.empty()) nulls.assign(rows, 0);
        desc.nulls = static_cast<const uint8_t*>(table.arena.place(nulls.data(), nulls.size()));
      }
      return;
    }
    case kFileDictionary:
    case kFileFixedString: {
      const uint8_t vector_type = reader.value<uint8_t>();
      desc.encoding = HYB_ENC_DICTIONARY;
      desc.dictionary_size = reader.value<uint32_t>();
      if (encoding == kFileFixedString) {
        if (!is_string) throw FormatError{HYB_ERR_INVALID, "unsupported data type for FixedStringDictionary encoding"};
        const uint32_t length = reader.value<uint32_t>();  // FixedStringVector: string length, then size * length characters
        std::vector<std::string> entries(desc.dictionary_size);
        for (auto& entry : entries) {
          const char* chars = reinterpret_cast<const char*>(reader.take(length));
          entry.assign(chars, strnlen(chars, length));
        }
        string_dictionary_from_entries(entries, table, column, desc, dictionary);
      } else if (is_string) {
        string_dictionary_from_entries(reader.strings(desc.dictionary_size), table, column, desc, dictionary);
      } else {
        const size_t bytes = size_t{desc.dictionary_size} * type_size(data_type);
        desc.values = table.arena.place(reader.take(bytes), bytes);
      }
      read_vector(reader, vector_type, rows, table, desc);
      return;
    }
    case kFileRunLength: {
      const uint32_t runs = reader.value<uint32_t>();
      std::vector<std::string> run_strings;
      const unsigned char* run_values = nullptr;
      const size_t width = is_string ? 0 : type_size(data_type);
      if (is_string) {
        run_strings = reader.strings(runs);
      } else {
        run_values = reader.take(size_t{runs} * width);
      }
      const unsigned char* run_nulls = reader.take(runs);
      std::vector<uint32_t> ends(runs);
      if (runs) std::memcpy(ends.data(), reader.take(size_t{runs} * 4), size_t{runs} * 4);  // inclusive end position of every run
      std::vector<uint8_t> nulls(rows, 0);
      std::vector<unsigned char> values(size_t{rows} * width);
      std::vector<std::string> strings(is_string ? rows : 0);
      bool any_null = false;
      uint32_t row = 0;
      for (uint32_t run = 0; run < runs; ++run) {
        if (ends[run] >= rows) throw FormatError{HYB_ERR_INVALID, "run end beyond the chunk"};
        for (; row <= ends[run]; ++row) {
          nulls[row] = run_nulls[run] ? 1 : 0;
          any_null = any_null || run_nulls[run];
          if (is_string) {
            strings[row] = run_strings[run];
          } else {
            std::memcpy(values.data() + size_t{row} * width, run_values + size_t{run} * width, width);
          }
        }
      }
      if (row != rows) throw FormatError{HYB_ERR_INVALID, "runs do not cover the chunk"};
      if (is_string) {
        dictionary_encode_strings(strings, (any_null || nullable) ? nulls : std::vector<uint8_t>{}, table, column, desc, dictionary);
        return;
      }
      desc.encoding = HYB_ENC_UNENCODED;
      desc.values = table.arena.place(values.data(), values.size());
      if (any_null || nullable) desc.nulls = static_cast<const uint8_t*>(table.arena.place(nulls.data(), nulls.size()));
      return;
    }
    case kFileFrameOfReference: {
      if (data_type != HYB_TYPE_INT32) throw FormatError{HYB_ERR_INVALID, "unsupported data type for FrameOfReference encoding"};
      const uint8_t vector_type = reader.value<uint8_t>();
      const uint32_t blocks = reader.value<uint32_t>();
      desc.encoding = HYB_ENC_FRAME_OF_REFERENCE;
      desc.values = table.arena.place(reader.take(size_t{blocks} * 4), size_t{blocks} * 4);
      if (reader.value<uint8_t>()) desc.nulls = static_cast<const uint8_t*>(table.arena.place(reader.take(rows), rows));
      read_vector(reader, vector_type, rows, table, desc);
      return;
    }
    case kFileLZ4:
      throw FormatError{HYB_ERR_UNSUPPORTED, "LZ4 segments are not read by the device path"};
    default:
      throw FormatError{HYB_ERR_INVALID, "invalid EncodingType " + std::to_string(encoding)};
  }
}

int32_t type_from_name(const std::string& name) {
  if (name == "int") return HYB_TYPE_INT32;
  if (name == "long") return HYB_TYPE_INT64;
  if (name == "float") return HYB_TYPE_FLOAT32;
  if (name == "double") return HYB_TYPE_FLOAT64;
  if (name == "string") return HYB_TYPE_STRING;
  throw FormatError{HYB_ERR_INVALID, "unknown column type '" + name + "'"};
}

}  // namespace

extern "C" {

int hyb_binary_table_open(const char* path, int32_t pinned, hyb_binary_table** out_table) {
  HYB_CHECK(path && out_table, HYB_ERR_INVALID, "NULL argument");
  *out_table = nullptr;
  std::ifstream file(path, std::ios::binary | std::ios::ate);
  HYB_CHECK(file.good(), HYB_ERR_NOT_FOUND, std::string("cannot open ") + path);
  const std::streamsize size = file.tellg();
  file.seekg(0);
  std::vector<unsigned char> bytes(static_cast<size_t>(std::max<std::streamsize>(size, 0)));
  if (size > 0) file.read(reinterpret_cast<char*>(bytes.data()), size);
  HYB_CHECK(file.good() || size == 0, HYB_ERR_INVALID, std::string("cannot read ") + path);
  auto table = std::make_unique<hyb_binary_table>(pinned != 0);
  try {
    Reader reader{bytes.data(), bytes.size()};
    table->chunk_size = reader.value<uint32_t>();
    const uint32_t chunk_count = reader.value<uint32_t>();
    const uint16_t column_count = reader.value<uint16_t>();
    if (column_count == 0) throw FormatError{HYB_ERR_INVALID, "a table needs at least one column"};
    for (const auto& name : reader.strings(column_count)) table->column_types.push_back(type_from_name(name));
    const unsigned char* nullable_flags = reader.take(column_count);
    table->column_nullable.assign(nullable_flags, nullable_flags + column_count);
    table->column_names = reader.strings(column_count);
    table->string_ids.resize(column_count);
    for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
      const uint32_t rows = reader.value<uint32_t>();
      const uint32_t sorted_count = reader.value<uint32_t>();
      table->sorted.emplace_back();
      for (uint32_t s = 0; s < sorted_count; ++s) {
        const uint16_t column = reader.value<uint16_t>();
        table->sorted.back().emplace_back(column, reader.value<uint8_t>());
      }
      table->chunk_rows.push_back(rows);
      for (uint32_t column = 0; column < column_count; ++column) {
        table->segments.emplace_back();
        table->string_dictionaries.emplace_back();
        read_segment(reader, rows, column, *table, table->segments.back(), table->string_dictionaries.back());
      }
    }
  } catch (const FormatError& error) {
    return fail(error.status, std::string(path) + ": " + error.message);
  }
  table->blocks = table->arena.host_blocks();
  *out_table = table.release();
  return HYB_OK;
}

void hyb_binary_table_close(hyb_binary_table* table) { delete table; }

int hyb_binary_table_info(const hyb_binary_table* table, uint32_t* out_chunk_size, uint32_t* out_chunk_count, uint32_t* out_column_count) {
  HYB_CHECK(table, HYB_ERR_INVALID, "NULL argument");
  if (out_chunk_size) *out_chunk_size = table->chunk_size;
  if (out_chunk_count) *out_chunk_count = static_cast<uint32_t>(table->chunk_rows.size());
  if (out_column_count) *out_column_count = static_cast<uint32_t>(table->column_types.size());
  return HYB_OK;
}

int hyb_binary_table_column(const hyb_binary_table* table, uint32_t column, const char** out_name, int32_t* out_data_type,
                            int32_t* out_nullable) {
  HYB_CHECK(table && column < table->column_types.size(), HYB_ERR_INVALID, "column out of range");
  if (out_name) *out_name = table->column_names[column].c_str();
  if (out_data_type) *out_data_type = table->column_types[column];
  if (out_nullable) *out_nullable = table->column_nullable[column] ? 1 : 0;
  return HYB_OK;
}

int hyb_binary_table_view(const hyb_binary_table* table, hyb_table_view* out_view) {
  HYB_CHECK(table && out_view, HYB_ERR_INVALID, "NULL argument");
  out_view->chunk_count = static_cast<uint32_t>(table->chunk_rows.size());
  out_view->column_count = static_cast<uint32_t>(table->column_types.size());
  out_view->segments = table->segments.data();
  return HYB_OK;
}

int hyb_binary_table_blocks(const hyb_binary_table* table, hyb_host_block* out_blocks, uint32_t* out_count) {
  HYB_CHECK(table && out_count, HYB_ERR_INVALID, "NULL argument");
  if (out_blocks) std::copy(table->blocks.begin(), table->blocks.end(), out_blocks);
  *out_count = static_cast<uint32_t>(table->blocks.size());
  return HYB_OK;
}

int hyb_binary_table_sorted_columns(const hyb_binary_table* table, uint32_t chunk, uint16_t* out_column_ids, uint8_t* out_sort_modes,
                                    uint32_t* out_count) {
  HYB_CHECK(table && out_count && chunk < table->sorted.size(), HYB_ERR_INVALID, "chunk out of range");
  const auto& sorted = table->sorted[chunk];
  for (size_t i = 0; i < sorted.size(); ++i) {
    if (out_column_ids) out_column_ids[i] = sorted[i].first;
    if (out_sort_modes) out_sort_modes[i] = sorted[i].second;
  }
  *out_count = static_cast<uint32_t>(sorted.size());
  return HYB_OK;
}

int hyb_binary_table_string_dictionary(const hyb_binary_table* table, uint32_t chunk, uint32_t column, const char** out_chars,
                                       const uint64_t** out_offsets, uint32_t* out_count) {
  HYB_CHECK(table && out_count, HYB_ERR_INVALID, "NULL argument");
  const size_t columns = table->column_types.size();
  HYB_CHECK(chunk < table->chunk_rows.size() && column < columns, HYB_ERR_INVALID, "segment out of range");
  HYB_CHECK(table->column_types[column] == HYB_TYPE_STRING, HYB_ERR_INVALID, "not a string column");
  const auto& dictionary = table->string_dictionaries[size_t{chunk} * columns + column];
  if (out_chars) *out_chars = dictionary.chars.data();
  if (out_offsets) *out_offsets = dictionary.offsets.data();
  *out_count = dictionary.offsets.empty() ? 0 : static_cast<uint32_t>(dictionary.offsets.size() - 1);
  return HYB_OK;
}

int hyb_binary_table_value_id_bounds(const hyb_binary_table* table, uint32_t column, const char* value, uint64_t value_length,
                                     const char* value2, uint64_t value2_length, uint32_t* out_bounds) {
  HYB_CHECK(table && value && out_bounds, HYB_ERR_INVALID, "NULL argument");
  const size_t columns = table->column_types.size();
  HYB_CHECK(column < columns && table->column_types[column] == HYB_TYPE_STRING, HYB_ERR_INVALID, "not a string column");
  const uint32_t values = value2 ? 2 : 1;
  const std::string needles[2] = {std::string(value, value_length), value2 ? std::string(value2, value2_length) : std::string()};
  for (size_t chunk = 0; chunk < table->chunk_rows.size(); ++chunk) {
    const auto& dictionary = table->string_dictionaries[chunk * columns + column];
    const uint32_t size = dictionary.offsets.empty() ? 0 : static_cast<uint32_t>(dictionary.offsets.size() - 1);
    const auto entry = [&](uint32_t index) {
      return std::string(dictionary.chars.data() + dictionary.offsets[index], dictionary.offsets[index + 1] - dictionary.offsets[index]);
    };
    for (uint32_t v = 0; v < values; ++v) {
      // DictionarySegment::lower_bound / upper_bound (dictionary_segment.cpp:94-119): INVALID_VALUE_ID past the end
      uint32_t lower = 0, upper = 0;
      for (uint32_t lo = 0, hi = size;;) {  // first entry >= needle
        if (lo >= hi) {
          lower = lo;
          break;
        }
        const uint32_t mid = lo + (hi - lo) / 2;
        if (entry(mid) < needles[v]) {
          lo = mid + 1;
        } else {
          hi = mid;
        }
      }
      for (uint32_t lo = lower, hi = size;;) {  // first entry > needle
        if (lo >= hi) {
          upper = lo;
          break;
        }
        const uint32_t mid = lo + (hi - lo) / 2;
        if (needles[v] < entry(mid)) {
          hi = mid;
        } else {
          lo = mid + 1;
        }
      }
      uint32_t* out = out_bounds + (chunk * values + v) * 2;
      out[0] = lower >= size ? HYB_INVALID_VALUE_ID : lower;
      out[1] = upper >= size ? HYB_INVALID_VALUE_ID : upper;
    }
  }
  return HYB_OK;
}

int hyb_binary_table_like_bitmaps(const hyb_binary_table* table, uint32_t column, const char* pattern, uint64_t pattern_length,
                                  int32_t condition, uint32_t* out_words, uint32_t* inout_word_count) {
  HYB_CHECK(table && inout_word_count, HYB_ERR_INVALID, "NULL argument");
  const size_t columns = table->column_types.size();
  HYB_CHECK(column < columns && table->column_types[column] == HYB_TYPE_STRING, HYB_ERR_INVALID, "not a string column");
  uint64_t words = 0;
  for (size_t chunk = 0; chunk < table->chunk_rows.size(); ++chunk) {
    const auto& dictionary = table->string_dictionaries[chunk * columns + column];
    const uint64_t size = dictionary.offsets.empty() ? 0 : dictionary.offsets.size() - 1;
    words += (size + 31) / 32;
  }
  HYB_CHECK(words <= UINT32_MAX, HYB_ERR_INVALID, "bitmap exceeds 2^32 words");
  if (!out_words) {
    *inout_word_count = static_cast<uint32_t>(words);
    return HYB_OK;
  }
  HYB_CHECK(*inout_word_count >= words, HYB_ERR_INVALID, "out_words holds fewer words than the bitmaps need");
  std::vector<LikeDictionary> dictionaries(table->chunk_rows.size());
  for (size_t chunk = 0; chunk < table->chunk_rows.size(); ++chunk) {
    const auto& dictionary = table->string_dictionaries[chunk * columns + column];
    const uint32_t size = dictionary.offsets.empty() ? 0 : static_cast<uint32_t>(dictionary.offsets.size() - 1);
    // chars.data() is NULL for a dictionary that holds only the empty string
    dictionaries[chunk] = LikeDictionary{dictionary.chars.data(), dictionary.offsets.data(), size};
  }
  HYB_TRY(like_match_dictionaries(pattern, pattern_length, condition, dictionaries.data(), dictionaries.size(), out_words,
                                  nullptr));
  *inout_word_count = static_cast<uint32_t>(words);
  return HYB_OK;
}

int hyb_binary_table_in_bitmaps(const hyb_binary_table* table, uint32_t column, int32_t condition, const char* element_chars,
                                const uint64_t* element_offsets, uint32_t element_count, uint32_t* out_words,
                                uint32_t* inout_word_count) {
  HYB_CHECK(table && inout_word_count, HYB_ERR_INVALID, "NULL argument");
  const size_t columns = table->column_types.size();
  HYB_CHECK(column < columns && table->column_types[column] == HYB_TYPE_STRING, HYB_ERR_INVALID, "not a string column");
  std::vector<LikeDictionary> dictionaries(table->chunk_rows.size());
  uint64_t words = 0;
  for (size_t chunk = 0; chunk < table->chunk_rows.size(); ++chunk) {
    const auto& dictionary = table->string_dictionaries[chunk * columns + column];
    const uint32_t size = dictionary.offsets.empty() ? 0 : static_cast<uint32_t>(dictionary.offsets.size() - 1);
    // chars.data() is NULL for a dictionary that holds only the empty string
    dictionaries[chunk] = LikeDictionary{dictionary.chars.data(), dictionary.offsets.data(), size};
    words += (size_t{size} + 31) / 32;
  }
  HYB_CHECK(words <= UINT32_MAX, HYB_ERR_INVALID, "bitmap exceeds 2^32 words");
  if (!out_words) {
    *inout_word_count = static_cast<uint32_t>(words);
    return HYB_OK;
  }
  HYB_CHECK(*inout_word_count >= words, HYB_ERR_INVALID, "out_words holds fewer words than the bitmaps need");
  HYB_TRY(in_match_dictionaries(condition, LikeDictionary{element_chars, element_offsets, element_count},
                                dictionaries.data(), dictionaries.size(), out_words, nullptr));
  *inout_word_count = static_cast<uint32_t>(words);
  return HYB_OK;
}

int hyb_binary_table_column_translation(const hyb_binary_table* table, uint32_t left_column, uint32_t right_column,
                                        uint32_t* out_words, uint32_t* inout_count) {
  HYB_CHECK(table && inout_count, HYB_ERR_INVALID, "NULL argument");
  const size_t columns = table->column_types.size();
  HYB_CHECK(left_column < columns && table->column_types[left_column] == HYB_TYPE_STRING && right_column < columns &&
                table->column_types[right_column] == HYB_TYPE_STRING,
            HYB_ERR_INVALID, "not two string columns");
  const auto view = [&](size_t chunk, uint32_t column) {
    const auto& dictionary = table->string_dictionaries[chunk * columns + column];
    const uint32_t size = dictionary.offsets.empty() ? 0 : static_cast<uint32_t>(dictionary.offsets.size() - 1);
    // chars.data() is NULL for a dictionary that holds only the empty string
    return LikeDictionary{dictionary.chars.data(), dictionary.offsets.data(), size};
  };
  uint64_t words = 0;
  for (size_t chunk = 0; chunk < table->chunk_rows.size(); ++chunk) words += view(chunk, right_column).count;
  HYB_CHECK(words <= UINT32_MAX, HYB_ERR_INVALID, "translation exceeds 2^32 words");
  if (!out_words) {
    *inout_count = static_cast<uint32_t>(words);
    return HYB_OK;
  }
  HYB_CHECK(*inout_count >= words, HYB_ERR_INVALID, "out_words holds fewer words than the translation needs");
  uint32_t* at = out_words;
  for (size_t chunk = 0; chunk < table->chunk_rows.size(); ++chunk) {
    const LikeDictionary right = view(chunk, right_column);
    HYB_TRY(translate_dictionary(view(chunk, left_column), right, at));
    at += right.count;
  }
  *inout_count = static_cast<uint32_t>(words);
  return HYB_OK;
}

int hyb_binary_table_string_order_ranks(const hyb_binary_table* table, uint32_t column, uint32_t* out_ranks,
                                        uint32_t* inout_count) {
  HYB_CHECK(table && inout_count, HYB_ERR_INVALID, "NULL argument");
  const size_t columns = table->column_types.size();
  HYB_CHECK(column < columns && table->column_types[column] == HYB_TYPE_STRING, HYB_ERR_INVALID, "not a string column");
  std::vector<LikeDictionary> dictionaries(table->chunk_rows.size());
  uint64_t words = 0;
  for (size_t chunk = 0; chunk < table->chunk_rows.size(); ++chunk) {
    const auto& dictionary = table->string_dictionaries[chunk * columns + column];
    const uint32_t size = dictionary.offsets.empty() ? 0 : static_cast<uint32_t>(dictionary.offsets.size() - 1);
    // chars.data() is NULL for a dictionary that holds only the empty string
    dictionaries[chunk] = LikeDictionary{dictionary.chars.data(), dictionary.offsets.data(), size};
    words += size;
  }
  HYB_CHECK(words <= UINT32_MAX, HYB_ERR_INVALID, "ranks exceed 2^32 words");
  if (!out_ranks) {
    *inout_count = static_cast<uint32_t>(words);
    return HYB_OK;
  }
  HYB_CHECK(*inout_count >= words, HYB_ERR_INVALID, "out_ranks holds fewer words than the ranks need");
  HYB_TRY(order_rank_dictionaries(dictionaries.data(), dictionaries.size(), out_ranks, nullptr));
  *inout_count = static_cast<uint32_t>(words);
  return HYB_OK;
}

int hyb_table_upload_binary(hyb_context* context, const hyb_binary_table* table, hyb_table_t* out_table) {
  HYB_CHECK(context && table && out_table, HYB_ERR_INVALID, "NULL argument");
  hyb_block_set_t block_set = 0;
  HYB_TRY(hyb_blocks_upload(context, table->blocks.data(), static_cast<uint32_t>(table->blocks.size()), &block_set));
  hyb_table_view view{};
  hyb_binary_table_view(table, &view);
  const int status = hyb_table_upload_from_blocks(context, &view, block_set, out_table);
  hyb_blocks_free(context, block_set);  // the table keeps the device copies alive
  return status;
}

}  // extern "C"
