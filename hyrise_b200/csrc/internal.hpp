// Internal host-side structures of libhyrise_b200 (not part of the C-ABI).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/hyrise_b200.h"

struct hyb_context;

namespace hyb {

// ---------------------------------------------------------------------------------------------------------------------
// Device-visible segment descriptor. One per (chunk, column); arrays of these are what every kernel indexes, so a single
// launch covers all chunks of a column (9 157 chunks at SF100) instead of one launch per chunk.
// ---------------------------------------------------------------------------------------------------------------------
struct DevSegment {
  const void* values;           // unencoded values | dictionary | FoR block minima
  const void* av;               // attribute vector (value-IDs) | FoR offsets, in vector_type layout
  const uint8_t* nulls;         // 1 byte per row or nullptr
  const uint64_t* dict_codes;   // chunk-independent group-by codes per dictionary entry or nullptr
  uint32_t row_count;
  uint32_t dict_size;           // == NULL value-ID for dictionary segments
  uint8_t encoding;
  uint8_t data_type;
  uint8_t vector_type;
  uint8_t bit_width;
  uint32_t pad;                 // flags: kSegmentMayContainNulls
};
constexpr uint32_t kSegmentMayContainNulls = 1u;  // set at upload (null vector present / NULL value-ID found)
static_assert(sizeof(DevSegment) == 48, "DevSegment layout");

// Bump allocator over large device slabs: one table = a handful of cudaMalloc calls instead of one per segment.
class Arena {
 public:
  static constexpr size_t kAlign = 256;
  static constexpr size_t kTailPad = 64;  // kernels may read one 16-byte vector past the last row
  ~Arena() { release(); }
  void* alloc(size_t bytes);
  hyb_context* owner = nullptr;  // set: a failed slab allocation releases the owner's idle cache blocks and retries once
  void release();
  size_t bytes_reserved() const { return _reserved; }
  size_t bytes_used() const { return _used; }

 private:
  struct Slab {
    char* base;
    size_t size;
    size_t offset;
  };
  std::vector<Slab> _slabs;
  size_t _reserved = 0;
  size_t _used = 0;
};

// Device copies of host arena blocks (hyb_blocks_upload): tables created from them hold a reference.
struct BlockSet {
  struct Block {
    const char* host_base;
    uint64_t bytes;
    char* device_base;
  };
  std::vector<Block> blocks;
  hyb_context* owner = nullptr;  // device blocks come from / go back to owner's DeviceCache: re-uploading the same arena
                                 // every step (an end-to-end pipeline) must not cost a cudaMalloc / cudaFree per block
  ~BlockSet();
  // Device address of a host buffer that lies inside one of the blocks, or nullptr.
  const void* translate(const void* host, size_t bytes) const;
};

struct Table {
  hyb_context* owner = nullptr;             // descriptor arrays and tile maps come from / go back to its DeviceCache: creating
                                            // and dropping tables in a loop (an end-to-end pipeline) never calls the driver
  std::shared_ptr<BlockSet> block_set;      // set when the segment buffers live in uploaded arena blocks
  bool adopting_device_buffers = false;     // hyb_table_append_chunk_device in progress: pointers are device pointers
  uint32_t column_count = 0;
  std::vector<uint32_t> chunk_rows;         // rows per chunk
  std::vector<uint64_t> chunk_row_start;    // exclusive prefix, chunk_count + 1 entries
  std::vector<DevSegment> segments;         // host copy, chunk-major: [chunk * column_count + column]
  std::vector<int32_t> column_types;        // hyb_data_type per column (from the first chunk)
  Arena arena;

  // Device mirrors, rebuilt lazily when `dirty`.
  DevSegment* d_segments = nullptr;         // column-major: [column * chunk_count + chunk]
  uint64_t* d_chunk_row_start = nullptr;    // chunk_count + 1
  uint32_t d_chunk_capacity = 0;
  bool dirty = true;
  std::map<uint32_t, std::pair<uint2*, uint32_t>> d_tile_maps;  // tile_rows -> (device {chunk,row0} per tile, count)
  // Integer key bounds per column {min, max, has_values}, computed on first use by JoinHash (the device-side analogue of
  // the MinMaxFilter pruning statistics, statistics/generate_pruning_statistics.cpp); cleared when chunks are appended.
  struct KeyBounds {
    long long min = 0, max = 0;
    bool has_values = false;
    uint32_t constant_low_bits = 0;  // every non-NULL key has the same value in these low bits (capped at 16)
    bool strictly_increasing = false;  // no NULLs and key[i] > key[i - 1] for every row position i
  };
  std::map<uint32_t, KeyBounds> key_bounds;
  // What an operator derived from a pass over all segment descriptors for one query shape (vector widths, dictionary sizes,
  // bytes per launch ...), keyed by the shape's signature: like the reference's physical-plan cache it spares a repeated
  // query the O(chunks x columns) analysis. Dropped with the key bounds whenever chunks change.
  std::map<std::string, std::shared_ptr<void>> plan_memo;
  // A string dictionary column seen by AggregateHash as an INT32 dictionary column: same attribute vectors, vector types,
  // bit widths and NULL value-IDs, with per-entry words as dictionaries. `ordered`: the words are the column's order ranks
  // (hyb_table_set_string_order) and `d_first_entry[rank]` = chunk_id << 32 | value_id of the first entry (in chunk order)
  // that holds the rank. Otherwise the words are zeros, which is all COUNT needs. Dropped with the key bounds.
  struct StringColumnView {
    hyb_context* owner = nullptr;
    DevSegment* d_segments = nullptr;           // chunk_count descriptors
    uint32_t* d_words = nullptr;
    unsigned long long* d_first_entry = nullptr;
    uint64_t word_count = 0;                    // rank words: the sum of the dictionary sizes
    bool ordered = false;
    ~StringColumnView();
  };
  std::map<uint32_t, std::shared_ptr<StringColumnView>> string_views;

  uint32_t chunk_count() const { return static_cast<uint32_t>(chunk_rows.size()); }
  uint64_t row_count() const { return chunk_row_start.empty() ? 0 : chunk_row_start.back(); }
  // Largest chunk and whether all chunks but the last share one size (lets kernels divide instead of search).
  uint32_t max_chunk_rows = 0;
  bool uniform_chunks = true;
  // > 0: a one-chunk table over a fixed device buffer whose row count changes between calls (the receive regions of a peer
  // group): descriptors are patched in place and tile maps are built once, for this many rows.
  uint32_t fixed_single_chunk_capacity = 0;
  // != nullptr: operators that emit RowIDs of this table emit position_payload[row position] instead (JoinHash only; the
  // tuples a rank received in a radix exchange stand for rows of the global table)
  const hyb_row_id* position_payload = nullptr;
  ~Table();
};

struct PosList {
  hyb_table_t table = 0;
  uint32_t chunk_count = 0;
  hyb_row_id* d_row_ids = nullptr;      // flat, chunk-major, ascending offsets inside a chunk
  uint64_t capacity = 0;
  uint64_t* d_chunk_end = nullptr;      // inclusive prefix per chunk (chunk_count entries) + total at [chunk_count]
  std::vector<uint64_t> h_chunk_offsets;  // chunk_count + 1, filled on first query
  bool host_valid = false;
  bool ascending = true;                // RowIDs in table order (what every TableScan of a table or of an ascending list produces)
  bool may_hold_null_rows = false;      // NULL_ROW_ID entries possible (one side of an outer join's result)
  cudaStream_t stream = nullptr;
  hyb_context* owner = nullptr;         // buffers go back to owner's DeviceCache
  ~PosList();
};

struct JoinResult {
  hyb_table_t build_table = 0, probe_table = 0;
  int32_t mode = 0;
  int32_t radix_bits = 0;
  uint32_t partition_count = 1;
  hyb_row_id* d_build = nullptr;
  hyb_row_id* d_probe = nullptr;
  uint64_t* d_partition_offsets = nullptr;  // partition_count + 1
  uint64_t capacity = 0;
  bool secondary = false;                   // joined with secondary predicates (hyb_join_hash_predicates)
  std::vector<uint64_t> h_partition_offsets;
  bool host_valid = false;
  cudaStream_t stream = nullptr;
  hyb_context* owner = nullptr;
  ~JoinResult();
};

struct AggregateColumn {
  int32_t value_type = 0;             // hyb_data_type of the result
  std::vector<uint8_t> values;        // group_count * element size
  std::vector<uint8_t> nulls;         // group_count
  bool is_any = false;                // ANY: no values; the column at the representative RowIDs (value_type = its type)
};

struct AggregateResult {
  hyb_table_t table = 0;              // the aggregated table: what row_ids point into (sort keys on its columns)
  uint64_t group_count = 0;
  int32_t used_immediate_keys = 0;
  std::vector<hyb_row_id> row_ids;
  std::vector<AggregateColumn> columns;
};

struct OperatorTiming {
  static constexpr int kMaxKernelSpans = 8;
  cudaEvent_t op_begin = nullptr, op_end = nullptr;
  // Device time of the bandwidth-bound kernel(s) only: up to kMaxKernelSpans begin/end pairs, summed (host round
  // trips between two kernels of one operator are not kernel time).
  cudaEvent_t kernel_begin[kMaxKernelSpans] = {}, kernel_end[kMaxKernelSpans] = {};
  int kernel_spans = 0;
  cudaEvent_t count_ready = nullptr;
  bool valid = false;
  hyb_operator_stats stats{};
  // Output cardinality is only known on the device when the operator returns: it is copied into this pinned slot.
  const uint64_t* d_output_count = nullptr;
  uint64_t* h_output_count = nullptr;
  uint32_t output_bytes_each = 0;
};

}  // namespace hyb

namespace hyb {
// Size-binned cache of device blocks for operator scratch and result buffers. All work of a context is queued on ONE
// stream, so a block can be handed out again as soon as it has been returned: later kernels are ordered after earlier
// ones. The CUDA stream-ordered pool (cudaMallocAsync) was measured to re-map physical memory inside the stream when the
// allocation pattern of consecutive operators differs (+9 ms per JoinHash at SF 10); this cache never calls the driver
// in steady state.
struct DeviceCache {
  std::multimap<size_t, void*> free_blocks;      // rounded size -> block
  std::unordered_map<void*, size_t> block_size;  // every block obtained from cudaMalloc that is still alive
  size_t free_bytes = 0;
};
}  // namespace hyb

namespace hyb {
// Tuning / test knobs. Read from the environment ONCE, when the context is created (never on an operator's hot path);
// hyb_context_set_option changes them afterwards (the parity tests force every join table kind that way).
struct ContextOptions {
  enum JoinTable : int { kAuto = 0, kHash, kDirect, kRank };
  int join_table = kAuto;      // HYB_JOIN_TABLE = hash | direct | rank
  bool join_colocated = true;  // HYB_JOIN_COLOCATED = 0: the distributed join always exchanges, even when the shards are co-located
  bool join_span = true;       // HYB_JOIN_SPAN = 0: keep the 4096-row tile kernels for the Inner/unique fast path
  bool join_ballot_rank = false;  // HYB_JOIN_RANK = ballot: one ballot per radix bit instead of MATCH.ANY (measured slower)
  bool scan_two_pass = true;   // HYB_SCAN_TWO_PASS = 1: match bits + tile counts, prefix, expansion (no look-back chain)
  bool scan_bulk = false;      // HYB_SCAN_BULK = 0: scan without the cp.async.bulk + mbarrier input pipeline
  bool aggregate_stream = true;  // HYB_AGG_STREAM = 0: keep the register-tile fast kernel for low-cardinality group-bys
  uint32_t aggregate_stages = 3;        // HYB_AGG_STAGES: depth of the streaming kernel's shared-memory ring (2..8, as far as it
                                        // fits); on an H100 a shallower ring leaves more L1 to the dictionary gathers
  bool aggregate_static_shapes = true;  // HYB_AGG_SHAPES = 0: always the layout-generic row loop of the streaming kernel
  bool trace = false;                   // HYB_TRACE = 1: one stderr line per kernel-variant decision
};
}  // namespace hyb

namespace hyb {
struct PeerGroup;
}

struct hyb_context {
  int device = 0;
  hyb::ContextOptions options;
  std::unordered_map<uint64_t, std::shared_ptr<hyb::PeerGroup>> peer_groups;
  cudaStream_t stream = nullptr;
  int sm_count = 132;  // H100 SXM; replaced by the device's count when the context is created
  std::mutex mutex;  // serialises enqueue + registry access; device work itself is asynchronous
  uint64_t next_handle = 1;
  std::unordered_map<uint64_t, std::unique_ptr<hyb::Table>> tables;
  std::unordered_map<uint64_t, std::unique_ptr<hyb::PosList>> pos_lists;
  std::unordered_map<uint64_t, std::unique_ptr<hyb::JoinResult>> join_results;
  std::unordered_map<uint64_t, std::unique_ptr<hyb::AggregateResult>> aggregate_results;
  std::unordered_map<uint64_t, std::shared_ptr<hyb::BlockSet>> block_sets;
  hyb::OperatorTiming timing;
  hyb::DeviceCache cache;
};

namespace hyb {

// Error plumbing -------------------------------------------------------------------------------------------------------
void set_error(const std::string& message);
int fail(int status, const std::string& message);

#define HYB_CUDA(expr)                                                                                      \
  do {                                                                                                      \
    cudaError_t _e = (expr);                                                                                \
    if (_e != cudaSuccess) {                                                                                \
      return ::hyb::fail(_e == cudaErrorMemoryAllocation ? HYB_ERR_OOM : HYB_ERR_CUDA,                      \
                         std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" + __FILE__ + ":" +       \
                             std::to_string(__LINE__) + ")");                                               \
    }                                                                                                       \
  } while (0)

#define HYB_CHECK(cond, status, message)        \
  do {                                          \
    if (!(cond)) {                              \
      return ::hyb::fail((status), (message));  \
    }                                           \
  } while (0)

#define HYB_TRY(expr)            \
  do {                           \
    int _s = (expr);             \
    if (_s != HYB_OK) return _s; \
  } while (0)

// LIKE over host string dictionaries (like.cu) -------------------------------------------------------------------------
// Entry i of a dictionary = chars[offsets[i] .. offsets[i + 1]); `chars` may be NULL when every entry is empty.
struct LikeDictionary {
  const char* chars;
  const uint64_t* offsets;
  uint32_t count;
};
// Compiles the pattern once and writes ceil(count / 32) match words per dictionary, the dictionaries' words one after
// another into out_words (hyb_like_dictionary_matches is the one-dictionary case).
int like_match_dictionaries(const char* pattern, uint64_t pattern_length, int32_t condition,
                            const LikeDictionary* dictionaries, size_t dictionary_count, uint32_t* out_words,
                            uint64_t* out_match_count);
// hyb_dictionary_translate (translate.cu): right_in_left of one chunk, right.count words, for two sorted unique
// dictionaries in the layout above.
int translate_dictionary(const LikeDictionary& left, const LikeDictionary& right, uint32_t* out_words);
// hyb_dictionary_order_ranks (translate.cu): dense ranks of every entry among the distinct strings of all dictionaries,
// in dictionary order.
int order_rank_dictionaries(const LikeDictionary* dictionaries, size_t dictionary_count, uint32_t* out_ranks,
                            uint32_t* out_distinct_count);
// hyb_in_dictionary_matches (in_list.cu) over several dictionaries, their bitmaps concatenated in out_words.
int in_match_dictionaries(int32_t condition, const LikeDictionary& elements, const LikeDictionary* dictionaries,
                          size_t dictionary_count, uint32_t* out_words, uint64_t* out_match_count);
// hyb_in_list_normalize (in_list.cu): [lo, hi] pairs in the column type's member of hyb_value.
int normalize_in_list(int32_t column_type, const hyb_literal* elements, uint32_t count, std::vector<hyb_value>& out_bounds);

// Helpers implemented in context.cu ---------------------------------------------------------------------------------
class DeviceGuard {
 public:
  explicit DeviceGuard(int device) {
    cudaGetDevice(&_previous);
    if (_previous != device) cudaSetDevice(device);
    _device = device;
  }
  ~DeviceGuard() {
    if (_previous != _device) cudaSetDevice(_previous);
  }

 private:
  int _previous = 0, _device = 0;
};

Table* find_table(hyb_context* context, hyb_table_t handle);
PosList* find_pos_list(hyb_context* context, hyb_pos_list_t handle);
// Rows in the list (synchronises the stream): d_chunk_end[chunk_count], with the "unset" fill of an empty scan read as 0.
int pos_list_total(hyb_context* context, const PosList* list, uint64_t* out_rows);
// Make the table's device descriptor arrays current (call with context->mutex held).
int sync_table_descriptors(hyb_context* context, Table* table);
// Device tile map: tiles of `tile_rows` rows never straddle a chunk; entry t = {chunk, first row | last-in-chunk << 31}.
int get_tile_map(hyb_context* context, Table* table, uint32_t tile_rows, const uint2** out_device,
                 uint32_t* out_tile_count);
// Stream-ordered scratch/result memory.
int device_alloc(hyb_context* context, size_t bytes, void** out);
cudaError_t device_malloc_retry(hyb_context* context, void** out, size_t bytes);
void device_free(hyb_context* context, void* ptr);
void device_cache_destroy(hyb_context* context);

// Scratch memory of one operator call: everything taken through it goes back to the context's block cache when the
// call returns, on EVERY path (the HYB_TRY / HYB_CUDA / HYB_CHECK early returns included).
class DeviceScratch {
 public:
  explicit DeviceScratch(hyb_context* context) : _context(context) {}
  DeviceScratch(const DeviceScratch&) = delete;
  DeviceScratch& operator=(const DeviceScratch&) = delete;
  ~DeviceScratch() {
    for (void* block : _blocks) device_free(_context, block);
  }
  int alloc(size_t bytes, void** out) {
    const int status = device_alloc(_context, bytes, out);
    if (status == HYB_OK) _blocks.push_back(*out);
    return status;
  }
  template <typename T>
  int alloc_array(size_t count, T** out) {
    void* block = nullptr;
    const int status = alloc(sizeof(T) * (count ? count : 1), &block);
    *out = static_cast<T*>(block);
    return status;
  }
  // Release a block taken with device_alloc together with this scope's blocks (nullptr: nothing to do).
  void adopt(void* block) {
    if (block) _blocks.push_back(block);
  }
  // Hand a block over to a result object (it is no longer released by this scope).
  void* release(void* block) {
    for (auto& entry : _blocks) {
      if (entry == block) {
        entry = nullptr;
        break;
      }
    }
    return block;
  }

 private:
  hyb_context* _context;
  std::vector<void*> _blocks;
};

void timing_begin(hyb_context* context);
void timing_kernel_begin(hyb_context* context);
void timing_kernel_end(hyb_context* context);
void timing_end(hyb_context* context, uint32_t launches, uint64_t algorithmic_bytes, uint64_t input_rows,
                uint64_t output_rows);
void timing_output_count(hyb_context* context, const uint64_t* d_count, uint32_t bytes_each);

inline size_t data_type_size(int32_t data_type) {
  switch (data_type) {
    case HYB_TYPE_INT32:
    case HYB_TYPE_FLOAT32:
      return 4;
    case HYB_TYPE_INT64:
    case HYB_TYPE_FLOAT64:
      return 8;
    default:
      return 0;
  }
}

inline size_t vector_bytes(int32_t vector_type, int32_t bit_width, uint32_t rows) {
  switch (vector_type) {
    case HYB_VEC_FIXED_1B:
      return rows;
    case HYB_VEC_FIXED_2B:
      return size_t{rows} * 2;
    case HYB_VEC_FIXED_4B:
      return size_t{rows} * 4;
    case HYB_VEC_BITPACKED:
      return ((size_t{rows} * bit_width + 63) / 64) * 8;
    default:
      return 0;
  }
}

}  // namespace hyb
