// JoinHash on the device: equi-join on one int32/int64 key column per side.
//
// Replaces JoinHashImpl::_on_execute (src/lib/operators/join_hash.cpp:270-572) and its steps materialize_input /
// partition_by_radix / build / probe / probe_semi_anti (src/lib/operators/join_hash/join_hash_steps.hpp:274-922).
// The reference radix-partitions both inputs so that every partition's hash table fits a CPU L2; that buys nothing on a
// GPU whose L2 is 50 MB (H100), so the device path keeps ONE hash table for the whole build side and never materialises
// {RowID, value} tuples. What the reference's partitioning does fix is the ORDER of the output — pairs come out grouped
// by hash(key) & (2^radix_bits - 1) (std::hash<int> is the identity), inside a partition in probe-row order, for one
// probe row in build-row order — and that order is reproduced exactly by ranking the matches instead of moving tuples:
//
//   join_build_kernel      every build row inserts {key, build position} into a bucketised open-addressing table
//                          (32-byte buckets of four {key:32, value:32} slots; bucket = mix(key >> 2), so four consecutive
//                          keys — the TPC-H orderkey pattern — share one sector). Duplicate keys keep the smallest
//                          position and raise a flag; if it is raised the CSR of positions per key is built (count,
//                          scan, fill, sort) so matches can be emitted in build-row order (PosHashTable, :97-236).
//   join_probe_count_kernel  per 4096-position tile of the probe side: 128-bit loads of the key column (8 keys per
//                          thread), in-register FoR / dictionary decode, one table lookup per run of equal keys, the
//                          match (4 bytes) and the radix partition (1 byte) of every probe row, and the emitted-row
//                          counts added to a per-(partition, tile) histogram.
//   exclusive scan         over the histogram laid out partition-major: the start of every (partition, tile) run.
//   join_probe_write_kernel  stable multi-split over the matches: each tile ranks its rows per partition (warp
//                          match_any + shared counters) and writes (build RowID, probe RowID) pairs straight to their
//                          final position. It never touches the key column again.
//
// Semi / Anti modes emit probe RowIDs only (probe_semi_anti); Left/Right emit NULL_ROW_ID partners for unmatched or
// NULL probe keys (probe<keep_null_values = true>). NULL build keys are never inserted (join_hash.cpp:271-286).
// Secondary predicates (hyb_join_hash_predicates) run a variant of the two tile kernels that evaluates them per candidate
// (join_probe_secondary_count_kernel / join_probe_secondary_write_kernel).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "column_pair.cuh"
#include "device_utils.cuh"
#include "internal.hpp"
#include "peer.hpp"

namespace hyb {

constexpr int kJoinThreads = 256;
constexpr int kJoinWarps = kJoinThreads / 32;
constexpr int kJoinTileRows = 4096;
constexpr int kJoinRowsPerWarp = kJoinTileRows / kJoinWarps;  // 512 contiguous positions per warp
constexpr uint32_t kNoMatch = 0xFFFFFFFFu;
constexpr unsigned long long kEmptySlot = ~0ull;
constexpr int kMaxPartitions = 256;
constexpr uint32_t kEmitWithoutPartner = 0xFFFFFFFEu;  // output row with a NULL build partner / Semi-Anti output row
constexpr int kMaxPeers = 16;            // ranks of one NVSwitch domain addressed by hyb_join_partition_push
constexpr int32_t kModePartition = 100;  // not a JoinMode: hyb_join_partition's stable split of {key, RowID} tuples by owner

struct KeySource {
  const DevSegment* segments;        // key column descriptors, one per chunk
  const uint2* tile_map;             // unfiltered input: per tile {chunk, row0 | last << 31}
  const hyb_row_id* filter;          // filtered input: flat pos list (then tile_map == nullptr)
  const unsigned long long* chunk_row_start;  // chunk_count + 1 (unfiltered)
  unsigned long long position_count;
  uint32_t tile_count;
  uint32_t chunk_count;
  const hyb_row_id* payload;         // != nullptr: position -> the RowID to emit (received tuples of a peer group carry the
                                     // global RowIDs of the rows they came from); else RowIDs of this table are emitted
  uint32_t uniform_chunk_rows;       // > 0: all chunks but the last have this many rows
  uint32_t uniform_magic;            // ceil(2^(32 + shift) / uniform_chunk_rows) - 2^32  (position / rows by multiply-shift)
  uint32_t uniform_shift;
  uint32_t chunk_id_base;            // added to the chunk id of every RowID of this table that is emitted (a rank's shard of a
                                     // global table: hyb_join_hash_distributed on co-located shards); 0 otherwise
  uint32_t null_key_zero;            // 1: the filter is one list over many chunks (a join's output, or a scan of it); the
                                     // reference reads it through MultipleChunkIterator, which yields T{} for every NULL
                                     // row (reference_segment_iterable.hpp:200-220)
};

struct KeyAt {
  long long key;
  bool valid;
  bool is_null;
  hyb_row_id row_id;
  unsigned long long position;
};

// Value at one position of an integer key column. NULL positions yield what the reference iterators yield: the stored
// value for ValueSegments, minimum + offset for FrameOfReference, T{} for dictionaries (dictionary_segment_iterable.hpp
// :116, frame_of_reference_segment_iterable.hpp:131-139) — it decides the partition a NULL probe row is emitted in. A
// PosList over many chunks yields 0 instead (KeySource::null_key_zero, applied where a probe row's partition is taken).
__device__ __forceinline__ long long decode_int_key(const DevSegment& segment, uint32_t row, bool& is_null) {
  switch (segment.encoding) {
    case HYB_ENC_UNENCODED:
      is_null = segment.nulls && segment.nulls[row];
      return segment.data_type == HYB_TYPE_INT32 ? static_cast<long long>(__ldg(static_cast<const int32_t*>(segment.values) + row))
                                                 : __ldg(static_cast<const long long*>(segment.values) + row);
    case HYB_ENC_DICTIONARY: {
      const uint32_t value_id = load_code1(segment.av, segment.vector_type, segment.bit_width, row);
      is_null = value_id >= segment.dict_size;
      if (is_null) return 0;
      return segment.data_type == HYB_TYPE_INT32
                 ? static_cast<long long>(__ldg(static_cast<const int32_t*>(segment.values) + value_id))
                 : __ldg(static_cast<const long long*>(segment.values) + value_id);
    }
    default: {
      is_null = segment.nulls && segment.nulls[row];
      const uint32_t code = load_code1(segment.av, segment.vector_type, segment.bit_width, row);
      const int32_t minimum = __ldg(static_cast<const int32_t*>(segment.values) + row / HYB_FOR_BLOCK_SIZE);
      return static_cast<long long>(static_cast<int32_t>(static_cast<uint32_t>(minimum) + code));
    }
  }
}

__device__ __forceinline__ KeyAt key_at(const KeySource& source, uint32_t tile, uint32_t index_in_tile) {
  KeyAt result{};
  if (source.tile_map) {
    const uint2 info = __ldg(source.tile_map + tile);
    const uint32_t chunk = info.x;
    const uint32_t row = (info.y & 0x7FFFFFFFu) + index_in_tile;
    const DevSegment& segment = source.segments[chunk];
    result.valid = row < segment.row_count;
    if (result.valid) {
      result.key = decode_int_key(segment, row, result.is_null);
      result.row_id = hyb_row_id{chunk, row};
      result.position = __ldg(source.chunk_row_start + chunk) + row;
    }
  } else {
    const unsigned long long position = static_cast<unsigned long long>(tile) * kJoinTileRows + index_in_tile;
    result.valid = position < source.position_count;
    if (result.valid) {
      result.row_id = source.filter[position];
      if (result.row_id.chunk_id == HYB_INVALID_CHUNK_ID) {
        result.is_null = true;
      } else {
        result.key = decode_int_key(source.segments[result.row_id.chunk_id], result.row_id.chunk_offset, result.is_null);
      }
      result.position = position;
    }
  }
  return result;
}

__device__ __forceinline__ hyb_row_id position_to_row_id(const KeySource& source, unsigned long long position) {
  if (source.payload) return source.payload[position];
  if (source.filter) {
    hyb_row_id row = source.filter[position];
    if (row.chunk_id != HYB_INVALID_CHUNK_ID) row.chunk_id += source.chunk_id_base;
    return row;
  }
  if (source.uniform_chunk_rows) {
    // positions are < 2^32 here (checked by the host): exact division by an invariant via multiply-high
    // (Granlund & Montgomery; q = (mulhi(n, m') + ((n - mulhi(n, m')) >> 1)) >> (shift - 1))
    const uint32_t n = static_cast<uint32_t>(position);
    const uint32_t t = __umulhi(n, source.uniform_magic);
    const uint32_t chunk = source.uniform_shift == 0 ? n : (t + ((n - t) >> 1)) >> (source.uniform_shift - 1);
    return hyb_row_id{chunk + source.chunk_id_base, n - chunk * source.uniform_chunk_rows};
  }
  uint32_t lo = 0, hi = source.chunk_count;  // chunk_row_start[lo] <= position < chunk_row_start[hi]
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(source.chunk_row_start + mid) <= position) {
      lo = mid;
    } else {
      hi = mid;
    }
  }
  return hyb_row_id{lo + source.chunk_id_base, static_cast<uint32_t>(position - __ldg(source.chunk_row_start + lo))};
}

struct TileRef {
  uint32_t chunk;       // unfiltered
  uint32_t row0;        // first row of the tile inside the chunk (unfiltered) / unused
  unsigned long long first_position;  // position of index 0 of this tile
};

__device__ __forceinline__ TileRef tile_ref(const KeySource& source, uint32_t tile) {
  TileRef ref{};
  if (source.tile_map) {
    const uint2 info = __ldg(source.tile_map + tile);
    ref.chunk = info.x;
    ref.row0 = info.y & 0x7FFFFFFFu;
    ref.first_position = __ldg(source.chunk_row_start + info.x) + ref.row0;
  } else {
    ref.first_position = static_cast<unsigned long long>(tile) * kJoinTileRows;
  }
  return ref;
}

// ---------------------------------------------------------------------------------------------------------------------
// Hash table: buckets of four 64-bit slots {key (low 32 bits of the int64 key... see below), value}.
// Keys are compared as 32-bit patterns when both columns are int32 (kWide == false). For int64 keys (kWide == true) a
// slot holds the low 32 key bits and the value indexes `wide_keys`, where the full key is verified.
// ---------------------------------------------------------------------------------------------------------------------
struct HashTable {
  unsigned long long* slots;      // bucket_count * 4
  uint32_t bucket_mask;           // bucket_count - 1 (power of two)
  const long long* wide_keys;     // per build position (int64 joins only), else nullptr
  // Direct-address mode (dense key domains): direct[key - direct_min] = smallest build position with that key, or
  // kNoMatch. std::hash<int> is the identity in the reference (join_hash_steps.hpp:52-60), so "hashing" a dense domain is
  // an array index; neighbouring keys share sectors and sorted inputs probe the table sequentially.
  // When all build keys agree in their `direct_shift` low bits (keys received by one rank of a radix exchange do), the
  // table is indexed by (key - direct_min) >> direct_shift and keys with other low bits cannot match.
  uint32_t* direct;
  long long direct_min;
  unsigned long long direct_range;
  uint32_t direct_shift;
  // Rank mode (dense key domain AND a build side whose keys strictly increase with the build position — primary keys
  // as dbgen and most loaders store them, also behind an order-preserving PosList): one {presence bits, ~(smallest
  // position)} pair per block of 32 key values. position(key) = smallest position of the block + number of present
  // keys below it in the block. 2 bits per key value instead of 32: the table of config 3 (60 M key values) shrinks
  // from 240 MB to 15 MB and stays in L2 for both probe passes, whatever the probe order. Indexed by key - direct_min.
  uint2* rank_blocks;
};

__device__ __forceinline__ uint32_t rank_block_position(const uint2 block, uint32_t bit) {
  return ~block.y + __popc(block.x & ((1u << bit) - 1u));
}

__device__ __forceinline__ uint32_t mix32(uint32_t h) {
  h ^= h >> 16;
  h *= 0x85EBCA6Bu;
  h ^= h >> 13;
  h *= 0xC2B2AE35u;
  h ^= h >> 16;
  return h;
}

__device__ __forceinline__ uint32_t bucket_of(long long key, uint32_t mask) {
  const unsigned long long bits = static_cast<unsigned long long>(key);
  return mix32(static_cast<uint32_t>(bits >> 2) ^ static_cast<uint32_t>(bits >> 34) * 0x9E3779B1u) & mask;
}

__device__ __forceinline__ unsigned long long pack_slot(uint32_t key_bits, uint32_t value) {
  return (static_cast<unsigned long long>(value) << 32) | key_bits;
}

// Looks `key` up. Returns the slot index (kNoMatch if absent) and the slot's value. A bucket with a free slot ends the
// search (there are no deletions). Written for few instructions: the probe kernel is issue-bound, not bandwidth-bound.
__device__ __forceinline__ uint32_t table_find(const HashTable& table, long long key, uint32_t& value) {
  if (table.rank_blocks) {
    const unsigned long long offset = static_cast<unsigned long long>(key) - static_cast<unsigned long long>(table.direct_min);
    if (offset >= table.direct_range) return kNoMatch;
    const uint2 block = __ldg(table.rank_blocks + (offset >> 5));
    const uint32_t bit = static_cast<uint32_t>(offset) & 31u;
    if (!((block.x >> bit) & 1u)) return kNoMatch;
    value = rank_block_position(block, bit);
    return static_cast<uint32_t>(offset);
  }
  if (table.direct) {
    const unsigned long long offset = static_cast<unsigned long long>(key) - static_cast<unsigned long long>(table.direct_min);
    const unsigned long long index = offset >> table.direct_shift;
    if (index >= table.direct_range || (offset & ((1ull << table.direct_shift) - 1ull))) return kNoMatch;
    value = __ldg(table.direct + index);
    return value == kNoMatch ? kNoMatch : static_cast<uint32_t>(index);
  }
  const uint32_t key_bits = static_cast<uint32_t>(key);
  uint32_t bucket = bucket_of(key, table.bucket_mask);
  while (true) {
    const uint4* base = reinterpret_cast<const uint4*>(table.slots + static_cast<size_t>(bucket) * 4);
    const uint4 a = __ldg(base);      // {key0, value0, key1, value1}
    const uint4 b = __ldg(base + 1);  // {key2, value2, key3, value3}
    // an empty slot has value 0xFFFFFFFF (no entry ever does): 1 bit per slot
    const uint32_t empty = (a.y == 0xFFFFFFFFu ? 1u : 0u) | (a.w == 0xFFFFFFFFu ? 2u : 0u) | (b.y == 0xFFFFFFFFu ? 4u : 0u) |
                           (b.w == 0xFFFFFFFFu ? 8u : 0u);
    uint32_t hits = ((a.x == key_bits ? 1u : 0u) | (a.z == key_bits ? 2u : 0u) | (b.x == key_bits ? 4u : 0u) |
                     (b.z == key_bits ? 8u : 0u)) & ~empty;
    while (hits) {
      const uint32_t e = __ffs(hits) - 1;
      hits &= hits - 1;
      value = e == 0 ? a.y : e == 1 ? a.w : e == 2 ? b.y : b.w;
      if (!table.wide_keys || table.wide_keys[value] == key) return bucket * 4 + e;
    }
    if (empty) return kNoMatch;
    bucket = (bucket + 1) & table.bucket_mask;
  }
}

__device__ __forceinline__ uint32_t table_find(const HashTable& table, long long key) {
  uint32_t value;
  return table_find(table, key, value);
}

struct BuildParams {
  KeySource source;
  HashTable table;
  long long* wide_keys_out;        // int64 hash tables: full key per build position, written by join_wide_keys_kernel
  uint32_t* flags;                 // [0] duplicate keys seen, [1] NULL keys seen, [2] inserted rows
};

__device__ __forceinline__ void table_insert(const BuildParams& params, long long key, uint32_t value) {
  if (params.table.rank_blocks) {
    // keys are unique here (strictly increasing build side): no return value needed, both updates are fire-and-forget
    const unsigned long long offset = static_cast<unsigned long long>(key) - static_cast<unsigned long long>(params.table.direct_min);
    uint2* block = params.table.rank_blocks + (offset >> 5);
    atomicOr(&block->x, 1u << (static_cast<uint32_t>(offset) & 31u));
    atomicMax(&block->y, ~value);
    return;
  }
  if (params.table.direct) {
    // every key lies inside [direct_min, direct_min + direct_range): the bounds cover the whole column
    const unsigned long long index =
        (static_cast<unsigned long long>(key) - static_cast<unsigned long long>(params.table.direct_min)) >> params.table.direct_shift;
    if (atomicMin(params.table.direct + index, value) != kNoMatch) params.flags[0] = 1;
    return;
  }
  const uint32_t key_bits = static_cast<uint32_t>(key);
  const unsigned long long desired = pack_slot(key_bits, value);
  uint32_t bucket = bucket_of(key, params.table.bucket_mask);
  while (true) {
    unsigned long long* slots = params.table.slots + static_cast<size_t>(bucket) * 4;
    const uint32_t start = key_bits & 3u;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      unsigned long long* slot = slots + ((start + j) & 3u);
      unsigned long long current = *reinterpret_cast<volatile unsigned long long*>(slot);
      if (current == kEmptySlot) {
        current = atomicCAS(slot, kEmptySlot, desired);
        if (current == kEmptySlot) return;
      }
      if (static_cast<uint32_t>(current) == key_bits) {
        // int64 keys: the owner's full key was stored by join_wide_keys_kernel, which finished before this kernel began.
        // No key value serves as an "unset" marker, so every key compares the same way.
        if (!params.wide_keys_out || params.wide_keys_out[static_cast<uint32_t>(current >> 32)] == key) {
          // Equal key already present: keep the smallest build position in the slot (deterministic) and flag it.
          atomicMin(reinterpret_cast<uint32_t*>(slot) + 1, value);
          params.flags[0] = 1;
          return;
        }
      }
    }
    bucket = (bucket + 1) & params.table.bucket_mask;
  }
}

// One key of a tile, lane-consecutive (thread t handles index t, t + 256, ...): neighbouring lanes hold neighbouring
// keys, so their hash-table accesses fall into the same 32-byte buckets — measured 4x faster than giving each thread 8
// consecutive rows, although that needs fewer load instructions.
__device__ __forceinline__ bool load_key1(const KeySource& source, const TileRef& ref, const DevSegment& segment,
                                          uint32_t index, long long& key, bool& is_null) {
  if (source.tile_map) {
    const uint32_t row = ref.row0 + index;
    if (row >= segment.row_count) return false;
    key = decode_int_key(segment, row, is_null);
    return true;
  }
  const unsigned long long position = ref.first_position + index;
  if (position >= source.position_count) return false;
  const hyb_row_id row_id = source.filter[position];
  if (row_id.chunk_id == HYB_INVALID_CHUNK_ID) {  // NULL_ROW_ID (an outer join's unmatched side): a NULL key
    key = 0;
    is_null = true;
    return true;
  }
  key = decode_int_key(source.segments[row_id.chunk_id], row_id.chunk_offset, is_null);
  return true;
}

__global__ void __launch_bounds__(kJoinThreads) join_build_kernel(const BuildParams params) {
  for (uint32_t tile = blockIdx.x; tile < params.source.tile_count; tile += gridDim.x) {
    const TileRef ref = tile_ref(params.source, tile);
    const DevSegment segment = params.source.tile_map ? params.source.segments[ref.chunk] : DevSegment{};
    for (uint32_t index = threadIdx.x; index < kJoinTileRows; index += kJoinThreads) {
      long long key;
      bool is_null;
      if (!load_key1(params.source, ref, segment, index, key, is_null)) continue;
      if (is_null) {
        params.flags[1] = 1;
        continue;
      }
      table_insert(params, key, static_cast<uint32_t>(ref.first_position + index));
    }
  }
}

// int64 hash tables: the full key of every non-NULL build position, stored before join_build_kernel runs so that an
// insert that meets a slot with equal low 32 bits can compare the owner's full key without waiting for it.
__global__ void __launch_bounds__(kJoinThreads) join_wide_keys_kernel(const BuildParams params) {
  for (uint32_t tile = blockIdx.x; tile < params.source.tile_count; tile += gridDim.x) {
    const TileRef ref = tile_ref(params.source, tile);
    const DevSegment segment = params.source.tile_map ? params.source.segments[ref.chunk] : DevSegment{};
    for (uint32_t index = threadIdx.x; index < kJoinTileRows; index += kJoinThreads) {
      long long key;
      bool is_null;
      if (!load_key1(params.source, ref, segment, index, key, is_null) || is_null) continue;
      params.wide_keys_out[ref.first_position + index] = key;
    }
  }
}

// ---- per-tile key codecs ---------------------------------------------------------------------------------------------
// The inner loops are specialised for the layouts that dominate (plain int32/int64 values, FrameOfReference offsets in a
// FixedWidthIntegerVector, no NULL vector); everything else — dictionaries, bit-packed vectors, nullable segments, PosList
// inputs — takes the generic decoder. The choice is uniform per tile (tiles never straddle chunks).
enum : uint32_t { kCodecGeneric = 0, kCodecPlain32, kCodecPlain64, kCodecFor8, kCodecFor16, kCodecFor32 };

__device__ __forceinline__ uint32_t tile_codec(const KeySource& source, const DevSegment& segment) {
  if (!source.tile_map || segment.nulls) return kCodecGeneric;
  if (segment.encoding == HYB_ENC_UNENCODED) return segment.data_type == HYB_TYPE_INT32 ? kCodecPlain32 : kCodecPlain64;
  if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) {
    if (segment.vector_type == HYB_VEC_FIXED_1B) return kCodecFor8;
    if (segment.vector_type == HYB_VEC_FIXED_2B) return kCodecFor16;
    if (segment.vector_type == HYB_VEC_FIXED_4B) return kCodecFor32;
  }
  return kCodecGeneric;
}

// Rank-table build. Keys arrive in rising order (that is what qualifies a build side for the rank table), so neighbouring
// rows fall into the same 32-key block: a thread combines the presence bits and the smallest position of its 4
// consecutive keys (one 128-bit load) before it touches the table — ONE atomicOr + ONE atomicMax per run of equal block
// ids instead of two atomics per key on the same 8 bytes (8 keys per block for dbgen's sparse order keys). Unique key
// columns are stored as plain ValueSegment<int32> by the reference's encoder (benchmark_table_encoder.cpp:119-120), which
// is the vectorised path; every other layout (FrameOfReference, dictionaries, int64, PosList inputs) inserts row by row.
// An input that is not sorted after all is still inserted correctly, only with more atomics.
__global__ void __launch_bounds__(kJoinThreads) join_build_rank_kernel(const BuildParams params) {
  const unsigned long long minimum = static_cast<unsigned long long>(params.table.direct_min);
  uint2* __restrict__ blocks = params.table.rank_blocks;
  for (uint32_t tile = blockIdx.x; tile < params.source.tile_count; tile += gridDim.x) {
    const TileRef ref = tile_ref(params.source, tile);
    const DevSegment segment = params.source.tile_map ? params.source.segments[ref.chunk] : DevSegment{};
    const uint32_t codec = tile_codec(params.source, segment);
    if (codec == kCodecPlain32 && ref.row0 + kJoinTileRows <= segment.row_count) {
      constexpr int kVectors = kJoinTileRows / (4 * kJoinThreads);  // 4 x 128-bit loads per thread, all in flight
      const uint4* keys4 = reinterpret_cast<const uint4*>(static_cast<const uint32_t*>(segment.values) + ref.row0);
      uint4 loaded[kVectors];
#pragma unroll
      for (int v = 0; v < kVectors; ++v) loaded[v] = ld_stream_v4(keys4 + v * kJoinThreads + threadIdx.x);
#pragma unroll
      for (int v = 0; v < kVectors; ++v) {
        const uint32_t first_position = static_cast<uint32_t>(ref.first_position) + (v * kJoinThreads + threadIdx.x) * 4;
        const uint32_t keys[4] = {loaded[v].x, loaded[v].y, loaded[v].z, loaded[v].w};
        uint32_t run_block = 0, run_bits = 0, run_position = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const unsigned long long offset = static_cast<unsigned long long>(static_cast<long long>(static_cast<int32_t>(keys[j]))) - minimum;
          const uint32_t block = static_cast<uint32_t>(offset >> 5);
          const uint32_t bit = 1u << (static_cast<uint32_t>(offset) & 31u);
          if (j > 0 && block == run_block) {
            run_bits |= bit;
          } else {
            if (j > 0) {
              atomicOr(&blocks[run_block].x, run_bits);
              atomicMax(&blocks[run_block].y, ~run_position);
            }
            run_block = block;
            run_bits = bit;
            run_position = first_position + j;
          }
        }
        atomicOr(&blocks[run_block].x, run_bits);
        atomicMax(&blocks[run_block].y, ~run_position);
      }
      continue;
    }
    constexpr int kSteps = kJoinTileRows / kJoinThreads;
    long long key[kSteps];
    uint32_t usable = 0;
#pragma unroll
    for (int s = 0; s < kSteps; ++s) {
      bool is_null = false;
      key[s] = 0;
      const bool valid = load_key1(params.source, ref, segment, s * kJoinThreads + threadIdx.x, key[s], is_null);
      if (valid && is_null) params.flags[1] = 1;
      usable |= (valid && !is_null) ? (1u << s) : 0u;
    }
#pragma unroll
    for (int s = 0; s < kSteps; ++s) {
      if ((usable >> s) & 1u) table_insert(params, key[s], static_cast<uint32_t>(ref.first_position + s * kJoinThreads + threadIdx.x));
    }
  }
}

// Smallest / largest non-NULL key of a column: out = {min, max, count of non-NULL rows, AND of keys, OR of keys, order
// violations}. Decides direct-address mode; bits where AND == OR are the same in every key; zero violations (no NULL, every
// key greater than the key one position earlier) means the column strictly increases in row order (rank mode).
__global__ void __launch_bounds__(kJoinThreads) join_key_bounds_kernel(const KeySource source, long long* __restrict__ out) {
  long long low = 0x7FFFFFFFFFFFFFFFll, high = -0x7FFFFFFFFFFFFFFFll - 1;
  unsigned long long count = 0, all_and = ~0ull, all_or = 0ull, violations = 0;
  for (uint32_t tile = blockIdx.x; tile < source.tile_count; tile += gridDim.x) {
    const TileRef ref = tile_ref(source, tile);
    const DevSegment segment = source.tile_map ? source.segments[ref.chunk] : DevSegment{};
    for (uint32_t index = threadIdx.x; index < kJoinTileRows; index += kJoinThreads) {
      long long key;
      bool is_null;
      if (!load_key1(source, ref, segment, index, key, is_null)) continue;
      if (is_null) {
        ++violations;
        continue;
      }
      // the key one position earlier: same tile, or the last row of the previous tile (possibly another chunk)
      long long previous = 0;
      bool previous_null = false, has_previous = false;
      if (index > 0) {
        has_previous = load_key1(source, ref, segment, index - 1, previous, previous_null);
      } else if (tile > 0 && source.tile_map) {
        const TileRef before = tile_ref(source, tile - 1);
        const DevSegment& before_segment = source.segments[before.chunk];
        const uint32_t last = min(static_cast<uint32_t>(kJoinTileRows), before_segment.row_count - before.row0) - 1;
        has_previous = load_key1(source, before, before_segment, last, previous, previous_null);
      }
      if (has_previous && !previous_null && previous >= key) ++violations;
      low = key < low ? key : low;
      high = key > high ? key : high;
      all_and &= static_cast<unsigned long long>(key);
      all_or |= static_cast<unsigned long long>(key);
      ++count;
    }
  }
#pragma unroll
  for (int delta = 16; delta > 0; delta >>= 1) {
    const long long other_low = __shfl_xor_sync(kFullMask, low, delta);
    const long long other_high = __shfl_xor_sync(kFullMask, high, delta);
    low = other_low < low ? other_low : low;
    high = other_high > high ? other_high : high;
    count += __shfl_xor_sync(kFullMask, count, delta);
    violations += __shfl_xor_sync(kFullMask, violations, delta);
    all_and &= __shfl_xor_sync(kFullMask, all_and, delta);
    all_or |= __shfl_xor_sync(kFullMask, all_or, delta);
  }
  if ((threadIdx.x & 31) == 0) {
    if (count) {
      atomicMin(out, low);
      atomicMax(out + 1, high);
      atomicAdd(reinterpret_cast<unsigned long long*>(out + 2), count);
      atomicAnd(reinterpret_cast<unsigned long long*>(out + 3), all_and);
      atomicOr(reinterpret_cast<unsigned long long*>(out + 4), all_or);
    }
    if (violations) atomicAdd(reinterpret_cast<unsigned long long*>(out + 5), violations);
  }
}

// ---- duplicate build keys: CSR of build positions per slot ----------------------------------------------------------
__global__ void join_count_duplicates_kernel(const KeySource source, const HashTable table, uint32_t* __restrict__ counts) {
  for (uint32_t tile = blockIdx.x; tile < source.tile_count; tile += gridDim.x) {
    for (uint32_t index = threadIdx.x; index < kJoinTileRows; index += kJoinThreads) {
      const KeyAt row = key_at(source, tile, index);
      if (!row.valid || row.is_null) continue;
      const uint32_t slot = table_find(table, row.key);
      if (slot != kNoMatch) atomicAdd(counts + slot, 1u);
    }
  }
}

__global__ void join_fill_positions_kernel(const KeySource source, const HashTable table,
                                           const unsigned long long* __restrict__ offsets, uint32_t* __restrict__ cursors,
                                           uint32_t* __restrict__ positions) {
  for (uint32_t tile = blockIdx.x; tile < source.tile_count; tile += gridDim.x) {
    for (uint32_t index = threadIdx.x; index < kJoinTileRows; index += kJoinThreads) {
      const KeyAt row = key_at(source, tile, index);
      if (!row.valid || row.is_null) continue;
      const uint32_t slot = table_find(table, row.key);
      if (slot == kNoMatch) continue;
      const uint32_t at = atomicAdd(cursors + slot, 1u);
      positions[offsets[slot] + at] = static_cast<uint32_t>(row.position);
    }
  }
}

// Build-row order inside a key's position list (insertion order of PosHashTable::emplace): heap sort, one thread per key.
__global__ void join_sort_positions_kernel(const uint32_t* __restrict__ counts, const unsigned long long* __restrict__ offsets,
                                           uint32_t slot_count, uint32_t* __restrict__ positions) {
  const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= slot_count) return;
  const uint32_t n = counts[slot];
  if (n < 2) return;
  uint32_t* a = positions + offsets[slot];
  const auto sift_down = [&](uint32_t start, uint32_t end) {
    uint32_t root = start;
    while (2 * root + 1 < end) {
      uint32_t child = 2 * root + 1;
      if (child + 1 < end && a[child] < a[child + 1]) ++child;
      if (a[root] >= a[child]) return;
      const uint32_t t = a[root];
      a[root] = a[child];
      a[child] = t;
      root = child;
    }
  };
  for (uint32_t start = n / 2; start-- > 0;) sift_down(start, n);
  for (uint32_t end = n; end-- > 1;) {
    const uint32_t t = a[0];
    a[0] = a[end];
    a[end] = t;
    sift_down(0, end);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Generic single-pass exclusive scan uint32 -> uint64 (decoupled look-back), used for the (partition, tile) histogram and
// the duplicate-key CSR.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kScanItems = 8;
constexpr int kScanTile = kJoinThreads * kScanItems;

__global__ void __launch_bounds__(kJoinThreads) exclusive_scan_kernel(const uint32_t* __restrict__ in,
                                                                      unsigned long long* __restrict__ out,
                                                                      unsigned long long count, unsigned long long* status,
                                                                      uint32_t* ticket, unsigned long long* total_out) {
  __shared__ unsigned long long s_warp[kJoinWarps];
  __shared__ unsigned long long s_base;
  __shared__ uint32_t s_tile;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t tile_count = static_cast<uint32_t>((count + kScanTile - 1) / kScanTile);
  while (true) {
    if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
    __syncthreads();
    const uint32_t tile = s_tile;
    if (tile >= tile_count) return;
    const unsigned long long first = static_cast<unsigned long long>(tile) * kScanTile + threadIdx.x * kScanItems;
    uint32_t items[kScanItems];
    unsigned long long sum = 0;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
      items[j] = first + j < count ? in[first + j] : 0u;
      sum += items[j];
    }
    unsigned long long inclusive = sum;
#pragma unroll
    for (int delta = 1; delta < 32; delta <<= 1) {
      const unsigned long long other = __shfl_up_sync(kFullMask, inclusive, delta);
      if (lane >= static_cast<uint32_t>(delta)) inclusive += other;
    }
    if (lane == 31) s_warp[warp] = inclusive;
    __syncthreads();
    unsigned long long warp_base = 0, tile_total = 0;
#pragma unroll
    for (int w = 0; w < kJoinWarps; ++w) {
      if (w < static_cast<int>(warp)) warp_base += s_warp[w];
      tile_total += s_warp[w];
    }
    if (warp == 0) {
      const unsigned long long base = lookback_exclusive_prefix(status, tile, tile_total, lane);
      if (lane == 0) {
        s_base = base;
        if (tile + 1 == tile_count && total_out) *total_out = base + tile_total;
      }
    }
    __syncthreads();
    unsigned long long running = s_base + warp_base + inclusive - sum;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
      if (first + j < count) out[first + j] = running;
      running += items[j];
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Probe
// ---------------------------------------------------------------------------------------------------------------------
// One secondary predicate of hyb_join_hash_predicates: `build value <condition> probe value` in the common type of the
// two columns.
struct JoinPredicate {
  const DevSegment* build;  // the build column's descriptors, one per chunk
  const DevSegment* probe;  // the probe column's descriptors
  int32_t condition;        // HYB_PRED_EQUALS .. HYB_PRED_GREATER_THAN_EQUALS
  uint32_t compare;         // PairCompare
};

// The second argument of the *_secondary_* probe kernels (ProbeParams stays the other kernels' layout).
struct SecondaryPredicates {
  const JoinPredicate* predicates;  // device copy
  uint32_t count;
};

struct ProbeParams {
  KeySource probe;
  KeySource build;                        // for position -> RowID of the build side
  HashTable table;
  int32_t mode;
  uint32_t partition_mask;                // 2^radix_bits - 1
  uint32_t partition_count;
  uint32_t unique_build;                  // 1: slot value is the build position; 0: use counts/offsets/positions
  uint32_t build_is_empty;
  const uint32_t* flags;                  // [0] duplicate build keys, [1] NULL build keys (written by the build kernel)
  const uint32_t* dup_counts;             // per slot
  const unsigned long long* dup_offsets;  // per slot
  const uint32_t* dup_positions;
  uint32_t* matches;                      // per probe slot (tile * 4096 + index): build position | slot | kEmit... | kNoMatch
  uint8_t* partitions;                    // per probe slot: hash(key) & partition_mask
  uint32_t* histogram;                    // [partition][tile]
  const unsigned long long* run_starts;   // exclusive scan of histogram
  hyb_row_id* out_build;
  hyb_row_id* out_probe;
  unsigned long long out_capacity;
  uint32_t* overflow;                     // set when the output does not fit out_capacity (optimistic sizing)
  uint32_t chunk_id_base;                 // kModePartition: added to chunk ids (RowIDs of the global table)
  uint32_t fast;                          // Inner join, int32 keys on both sides, direct-address table without shift
  // kModePartition with peer destinations (hyb_join_partition_push): group p is written to peer_keys[p] / peer_rows[p]
  // (device memory of rank p, mapped through CUDA IPC — NVLink P2P stores) at the group-relative index.
  long long* peer_keys[kMaxPeers];
  long long* peer_rows[kMaxPeers];
  uint32_t push_to_peers;
  // hyb_join_hash_distributed: the LAST CTA of the push kernels (both sides share the arrival counter) raises this rank's
  // done flag in every peer's control block, after a system-scope fence that orders it behind all tuple stores.
  unsigned int* signal_arrivals;
  uint32_t signal_expected;
  uint32_t signal_world;
  unsigned long long signal_epoch;
  unsigned long long* signal_flags[kMaxPeers];
};

__device__ __forceinline__ void peer_signal_when_last(const ProbeParams& params) {
  if (!params.signal_arrivals) return;
  __threadfence_system();  // this thread's peer stores are performed system-wide before the CTA counts itself in
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int ticket = atomicAdd(params.signal_arrivals, 1u);
    if (ticket + 1 == params.signal_expected) {
      __threadfence_system();
      for (uint32_t peer = 0; peer < params.signal_world; ++peer) st_volatile_u64(params.signal_flags[peer], params.signal_epoch);
    }
  }
}

__global__ void peer_signal_kernel(const ProbeParams params) { peer_signal_when_last(params); }

// What one probe row contributes. Returns the match word: a build position (unique build side), a table slot
// (duplicate build keys), kEmitWithoutPartner (one output row without a build partner) or kNoMatch (no output row).
// Inner/Semi drop NULL probe keys during materialisation; Left/Right and AntiNullAsFalse emit them; AntiNullAsTrue emits
// them only when the build table is empty, and nothing at all once the build side holds a NULL
// (join_hash_steps.hpp:711-758, 848-913; join_hash.cpp:471-483).
__device__ __forceinline__ uint32_t probe_match_resolved(const ProbeParams& params, uint32_t slot, uint32_t value,
                                                         bool is_null, bool build_has_nulls) {
  const int32_t mode = params.mode;
  if (mode == HYB_JOIN_INNER) {  // the common case first: NULL probe keys were never looked up (slot == kNoMatch)
    return slot == kNoMatch ? kNoMatch : (params.unique_build ? value : slot);
  }
  if (mode == kModePartition) return is_null ? kNoMatch : kEmitWithoutPartner;
  if (mode == HYB_JOIN_ANTI_NULL_AS_TRUE && build_has_nulls) return kNoMatch;
  if (is_null) {
    if (mode == HYB_JOIN_LEFT || mode == HYB_JOIN_RIGHT || mode == HYB_JOIN_ANTI_NULL_AS_FALSE) return kEmitWithoutPartner;
    if (mode == HYB_JOIN_ANTI_NULL_AS_TRUE) return params.build_is_empty ? kEmitWithoutPartner : kNoMatch;
    return kNoMatch;
  }
  const bool found = slot != kNoMatch;
  switch (mode) {
    case HYB_JOIN_SEMI:
      return found ? kEmitWithoutPartner : kNoMatch;
    case HYB_JOIN_ANTI_NULL_AS_TRUE:
    case HYB_JOIN_ANTI_NULL_AS_FALSE:
      return found ? kNoMatch : kEmitWithoutPartner;
    default:
      break;
  }
  if (!found) return (mode == HYB_JOIN_LEFT || mode == HYB_JOIN_RIGHT) ? kEmitWithoutPartner : kNoMatch;
  return params.unique_build ? value : slot;
}

__device__ __forceinline__ uint32_t emitted_rows(const ProbeParams& params, uint32_t match) {
  if (match == kNoMatch) return 0;
  if (match == kEmitWithoutPartner || params.unique_build) return 1;
  return params.dup_counts[match];
}

// ---- secondary predicates (hyb_join_hash_predicates) -----------------------------------------------------------------
// probe / probe_semi_anti with a MultiPredicateJoinEvaluator (join_hash_steps.hpp:690-748, :844-883): every candidate of
// a probe row — a build row with its key — is tested against every predicate, one FieldComparator::compare each
// (multi_predicate_join_evaluator.cpp): a NULL on either side fails, otherwise the comparator in the common type.
// Candidates are never materialised: the count pass counts the passing ones; the write pass evaluates them again to
// rank the row and, for Inner / Left / Right rows with passing candidates, a third time to store exactly those pairs.

// One side's value of every predicate at one row, as the bits of each predicate's common type; bit i of `nulls`: NULL.
struct PredicateValues {
  unsigned long long bits[HYB_MAX_JOIN_PREDICATES];
  uint32_t nulls;
};

// Returns true for NULL (a NULL_ROW_ID of a filter is NULL in every column).
__device__ __forceinline__ bool predicate_value(const DevSegment* segments, uint32_t compare, hyb_row_id row,
                                                unsigned long long& bits) {
  if (row.chunk_id == HYB_INVALID_CHUNK_ID) return true;
  const DevSegment& segment = segments[row.chunk_id];
  if (compare == kCompareInt64) {
    long long value;
    if (decode1<AsInt64>(segment, row.chunk_offset, value)) return true;
    bits = static_cast<unsigned long long>(value);
  } else if (compare == kCompareFloat) {
    float value;
    if (decode1<AsFloat>(segment, row.chunk_offset, value)) return true;
    bits = __float_as_uint(value);
  } else {
    double value;
    if (decode1<AsDouble>(segment, row.chunk_offset, value)) return true;
    bits = static_cast<unsigned long long>(__double_as_longlong(value));
  }
  return false;
}

// The probe row's values: decoded once per probe row and evaluation (secondary_resolved, write_passing_candidates). Not
// inlined: the probe loops are unrolled 16 times.
__device__ __noinline__ PredicateValues probe_predicate_values(const JoinPredicate* predicates, uint32_t count, hyb_row_id row) {
  PredicateValues values{};
#pragma unroll
  for (uint32_t i = 0; i < HYB_MAX_JOIN_PREDICATES; ++i) {
    if (i < count && predicate_value(predicates[i].probe, predicates[i].compare, row, values.bits[i])) values.nulls |= 1u << i;
  }
  return values;
}

// Whether the build row `row` passes every predicate against the probe row's values.
__device__ __noinline__ bool candidate_passes(const JoinPredicate* predicates, uint32_t count, const PredicateValues probe,
                                              hyb_row_id row) {
#pragma unroll
  for (uint32_t i = 0; i < HYB_MAX_JOIN_PREDICATES; ++i) {
    if (i >= count) break;
    if ((probe.nulls >> i) & 1u) return false;
    const JoinPredicate predicate = predicates[i];
    unsigned long long bits = 0;
    if (predicate_value(predicate.build, predicate.compare, row, bits)) return false;
    bool holds;
    if (predicate.compare == kCompareInt64) {
      holds = compare1(predicate.condition, static_cast<long long>(bits), static_cast<long long>(probe.bits[i]));
    } else if (predicate.compare == kCompareFloat) {
      holds = compare1(predicate.condition, __uint_as_float(static_cast<uint32_t>(bits)),
                       __uint_as_float(static_cast<uint32_t>(probe.bits[i])));
    } else {
      holds = compare1(predicate.condition, __longlong_as_double(static_cast<long long>(bits)),
                       __longlong_as_double(static_cast<long long>(probe.bits[i])));
    }
    if (!holds) return false;
  }
  return true;
}

// The word a probe row's key lookup leaves for the predicates: its candidates (the build position of a unique build
// side, else the table slot whose position list holds them), or — no key match, or a NULL key — kEmitWithoutPartner for
// the modes that keep such rows and kNoMatch for the others.
__device__ __forceinline__ uint32_t secondary_candidates(const ProbeParams& params, uint32_t slot, uint32_t value, bool is_null) {
  if (!is_null && slot != kNoMatch) return params.unique_build ? value : slot;
  const int32_t mode = params.mode;
  return (mode == HYB_JOIN_LEFT || mode == HYB_JOIN_RIGHT || mode == HYB_JOIN_ANTI_NULL_AS_FALSE) ? kEmitWithoutPartner : kNoMatch;
}

// RowID of a probe side's tile index `index` in its own table (a NULL_ROW_ID of a filter stays one).
__device__ __forceinline__ hyb_row_id probe_row_id(const KeySource& source, const TileRef& ref, uint32_t index) {
  if (source.tile_map) return hyb_row_id{ref.chunk, ref.row0 + index};
  return source.filter[ref.first_position + index];
}

// Evaluates the candidates of one probe row. Returns the match word the write pass acts on — kNoMatch, kEmitWithoutPartner
// (one row without a build partner; Semi / Anti: the probe row) or, when candidates pass in an Inner / Left / Right join,
// the candidates themselves — and the probe row's output rows in `emit`.
__device__ __forceinline__ uint32_t secondary_resolved(const ProbeParams& params, const SecondaryPredicates& secondary,
                                                       uint32_t candidates, const TileRef& ref, uint32_t index, uint32_t& emit) {
  emit = candidates == kEmitWithoutPartner ? 1u : 0u;
  if (candidates == kNoMatch || candidates == kEmitWithoutPartner) return candidates;
  const int32_t mode = params.mode;
  const bool existence = mode == HYB_JOIN_SEMI || mode == HYB_JOIN_ANTI_NULL_AS_FALSE;  // the first passing one decides
  const PredicateValues probe = probe_predicate_values(secondary.predicates, secondary.count, probe_row_id(params.probe, ref, index));
  const bool unique = params.unique_build != 0;
  const uint32_t count = unique ? 1u : params.dup_counts[candidates];
  const unsigned long long first = unique ? 0ull : params.dup_offsets[candidates];
  uint32_t passing = 0;
  for (uint32_t j = 0; j < count; ++j) {
    const uint32_t position = unique ? candidates : params.dup_positions[first + j];
    if (candidate_passes(secondary.predicates, secondary.count, probe, position_to_row_id(params.build, position))) {
      ++passing;
      if (existence) break;
    }
  }
  if (mode == HYB_JOIN_SEMI || mode == HYB_JOIN_ANTI_NULL_AS_FALSE) {
    const bool kept = (passing != 0) == (mode == HYB_JOIN_SEMI);
    emit = kept ? 1u : 0u;
    return kept ? kEmitWithoutPartner : kNoMatch;
  }
  if (passing) {
    emit = passing;
    return candidates;
  }
  if (mode == HYB_JOIN_INNER) return kNoMatch;
  emit = 1;  // Left / Right: one row with a NULL build partner where the pairs would have been
  return kEmitWithoutPartner;
}

// The write pass of a probe row with passing candidates: those candidates, in build-row order, from `at` on.
__device__ __forceinline__ void write_passing_candidates(const ProbeParams& params, const SecondaryPredicates& secondary,
                                                         uint32_t candidates, hyb_row_id probe_row, unsigned long long at) {
  const PredicateValues probe = probe_predicate_values(secondary.predicates, secondary.count, probe_row);
  const bool unique = params.unique_build != 0;
  const uint32_t count = unique ? 1u : params.dup_counts[candidates];
  const unsigned long long first = unique ? 0ull : params.dup_offsets[candidates];
  for (uint32_t j = 0; j < count; ++j) {
    const hyb_row_id build_row = position_to_row_id(params.build, unique ? candidates : params.dup_positions[first + j]);
    if (!candidate_passes(secondary.predicates, secondary.count, probe, build_row)) continue;
    if (at >= params.out_capacity) {
      *params.overflow = 1;
      return;
    }
    st_stream_v2(params.out_build + at, build_row.chunk_id, build_row.chunk_offset);
    st_stream_v2(params.out_probe + at, probe_row.chunk_id, probe_row.chunk_offset);
    ++at;
  }
}

template <uint32_t kCodec>
__device__ __forceinline__ bool codec_key(const KeySource& source, const TileRef& ref, const DevSegment& segment, uint32_t index,
                                          uint32_t for_minimum, long long& key, bool& is_null) {
  if constexpr (kCodec == kCodecGeneric) {
    return load_key1(source, ref, segment, index, key, is_null);
  } else {
    const uint32_t row = ref.row0 + index;
    is_null = false;
    if (row >= segment.row_count) return false;
    if constexpr (kCodec == kCodecPlain32) {
      key = static_cast<int32_t>(ld_stream_u32(static_cast<const uint32_t*>(segment.values) + row));
    } else if constexpr (kCodec == kCodecPlain64) {
      key = __ldg(static_cast<const long long*>(segment.values) + row);
    } else if constexpr (kCodec == kCodecFor8) {
      key = static_cast<int32_t>(for_minimum + __ldg(static_cast<const uint8_t*>(segment.av) + row));
    } else if constexpr (kCodec == kCodecFor16) {
      key = static_cast<int32_t>(for_minimum + __ldg(static_cast<const uint16_t*>(segment.av) + row));
    } else {
      key = static_cast<int32_t>(for_minimum + ld_stream_u32(static_cast<const uint32_t*>(segment.av) + row));
    }
    return true;
  }
}

constexpr int kProbeSteps = kJoinRowsPerWarp / 32;  // 16 rows per lane, lane-consecutive: step s, lane l -> chunk0 + 32 s + l

// The rows of one warp chunk (512 consecutive tile indexes) held in registers between the two passes of the write kernel.
struct ChunkRows {
  uint32_t match[kProbeSteps];
  uint32_t rank[kProbeSteps];            // output row of this probe row, relative to its (warp chunk, partition) run
  uint32_t partitions[kProbeSteps / 4];  // one byte per step
};

// Pass 1 over one warp chunk: key -> table lookup -> match word and radix partition of every row, emitted-row counts
// added to histogram[partition] (one shared-memory atomic per distinct partition and step). With kRank the value the
// histogram held before the add — the number of rows this warp chunk emitted into the partition in earlier steps — plus
// the emitting peers in lower lanes is the row's rank: lane order is probe order, so ranks reproduce the reference order.
// kSource: 0 = decode + look up, storing nothing; 1 = decode + look up and store match/partition per probe slot (hash
// tables: the write kernel must not repeat the random accesses); 2 = load what mode 1 stored. kSecondary: the match
// word is secondary_candidates' (stored as such) and the row's output comes from evaluating them.
template <bool kRank, int kSource, uint32_t kCodec, bool kSecondary = false>
__device__ __forceinline__ void probe_chunk(const ProbeParams& params, const TileRef& ref, const DevSegment& segment,
                                            uint32_t chunk0, size_t tile_slot0, uint32_t lane, bool build_has_nulls,
                                            uint32_t* histogram, ChunkRows& rows,
                                            const SecondaryPredicates& secondary = SecondaryPredicates{}) {
  const bool unique = params.unique_build != 0;
  const uint32_t lanes_below = (1u << lane) - 1u;
  uint32_t for_minimum = 0;
  if constexpr (kSource != 2 && kCodec >= kCodecFor8) {
    // chunk0 is a multiple of 512 and tiles start at multiples of 4096 rows: the warp chunk lies inside one 2048-row block
    const uint32_t first_row = ref.row0 + chunk0;
    if (first_row < segment.row_count) {
      for_minimum = static_cast<uint32_t>(__ldg(static_cast<const int32_t*>(segment.values) + first_row / HYB_FOR_BLOCK_SIZE));
    }
  }
#pragma unroll
  for (int q = 0; q < kProbeSteps / 4; ++q) rows.partitions[q] = 0;
#pragma unroll
  for (int step = 0; step < kProbeSteps; ++step) {
    const uint32_t index = chunk0 + step * 32 + lane;
    uint32_t match, partition;
    if constexpr (kSource == 2) {
      match = __ldg(params.matches + tile_slot0 + index);
      partition = __ldg(params.partitions + tile_slot0 + index);
    } else {
      long long key = 0;
      bool is_null = false;
      const bool valid = codec_key<kCodec>(params.probe, ref, segment, index, for_minimum, key, is_null);
      if constexpr (kCodec == kCodecGeneric) {
        if (is_null && params.probe.null_key_zero) key = 0;  // only PosList inputs set it; they take the generic codec
      }
      match = kNoMatch;
      if (valid) {
        uint32_t value = 0;
        const uint32_t slot = (!is_null && params.table.slots) ? table_find(params.table, key, value) : kNoMatch;
        if constexpr (kSecondary) {
          match = secondary_candidates(params, slot, value, is_null);
        } else {
          match = probe_match_resolved(params, slot, value, is_null, build_has_nulls);
        }
      }
      partition = static_cast<uint32_t>(static_cast<unsigned long long>(key)) & params.partition_mask;
      if constexpr (kSource == 1) {
        params.matches[tile_slot0 + index] = match;
        params.partitions[tile_slot0 + index] = static_cast<uint8_t>(partition);
      }
    }
    uint32_t emit;
    if constexpr (kSecondary) {
      match = secondary_resolved(params, secondary, match, ref, index, emit);
    } else {
      emit = emitted_rows(params, match);
    }
    if constexpr (!kRank) {
      if (emit) atomicAdd(histogram + partition, emit);  // counting needs no order
      continue;
    }
    const uint32_t peers = __match_any_sync(kFullMask, partition);
    uint32_t before = 0, total = 0;
    if (unique) {
      const uint32_t emitting = __ballot_sync(kFullMask, emit != 0) & peers;
      total = __popc(emitting);
      before = __popc(emitting & lanes_below);
    } else {
      uint32_t remaining = peers;
      while (remaining) {
        const int source_lane = __ffs(remaining) - 1;
        const uint32_t value = __shfl_sync(peers, emit, source_lane);
        if (static_cast<uint32_t>(source_lane) < lane) before += value;
        total += value;
        remaining &= remaining - 1;
      }
    }
    const int leader = __ffs(peers) - 1;
    uint32_t earlier = 0;
    if (lane == static_cast<uint32_t>(leader) && total) earlier = atomicAdd(histogram + partition, total);
    if constexpr (kRank) {
      earlier = __shfl_sync(kFullMask, earlier, leader);
      rows.match[step] = match;
      rows.rank[step] = earlier + before;
      rows.partitions[step >> 2] |= partition << (8 * (step & 3));
    }
  }
}

// The same pass for the case that dominates (Inner join, unique build side, int32 keys, direct-address table, plain or
// FrameOfReference probe segment without NULLs), stripped to ~20 instructions per probe row: 32-bit key arithmetic, no mode
// or NULL handling, the row-count check only in a chunk's last tile.
template <bool kRank, uint32_t kCodec, bool kFull>
__device__ __forceinline__ void probe_chunk_fast(const ProbeParams& params, const TileRef& ref, const DevSegment& segment,
                                                 uint32_t chunk0, uint32_t lane, uint32_t* histogram, ChunkRows& rows) {
  constexpr bool kWide = kCodec == kCodecPlain64;  // int64 keys (the tuples of a radix exchange): 64-bit index arithmetic
  const uint32_t lanes_below = (1u << lane) - 1u;
  const uint32_t partition_mask = params.partition_mask;
  const uint32_t* __restrict__ direct = params.table.direct;
  const uint32_t direct_min = static_cast<uint32_t>(params.table.direct_min);
  const uint32_t direct_range = static_cast<uint32_t>(params.table.direct_range);
  const unsigned long long wide_min = static_cast<unsigned long long>(params.table.direct_min);
  const uint32_t shift = params.table.direct_shift;
  const unsigned long long low_bits = (1ull << shift) - 1ull;
  const uint32_t row_count = segment.row_count;
  const uint32_t row_base = ref.row0 + chunk0 + lane;
  uint32_t for_minimum = 0;
  if constexpr (kCodec >= kCodecFor8 && kCodec != kCodecPlain64) {
    if (kFull || ref.row0 + chunk0 < row_count) {
      for_minimum = static_cast<uint32_t>(__ldg(static_cast<const int32_t*>(segment.values) + (ref.row0 + chunk0) / HYB_FOR_BLOCK_SIZE));
    }
  }
#pragma unroll
  for (int q = 0; q < kProbeSteps / 4; ++q) rows.partitions[q] = 0;
#pragma unroll
  for (int step = 0; step < kProbeSteps; ++step) {
    const uint32_t row = row_base + step * 32;
    const bool valid = kFull || row < row_count;
    uint32_t key = 0;
    uint32_t match = kNoMatch;
    if constexpr (kWide) {
      if (valid) {
        const uint2 bits = ld_stream_v2(static_cast<const long long*>(segment.values) + row);
        key = bits.x;  // the partition only needs the low bits
        const unsigned long long offset = ((static_cast<unsigned long long>(bits.y) << 32) | bits.x) - wide_min;
        const unsigned long long index = offset >> shift;
        if (index < direct_range && !(offset & low_bits)) match = __ldg(direct + index);
      }
    } else {
      if (valid) {
        if constexpr (kCodec == kCodecPlain32) {
          key = ld_stream_u32(static_cast<const uint32_t*>(segment.values) + row);
        } else if constexpr (kCodec == kCodecFor8) {
          key = for_minimum + __ldg(static_cast<const uint8_t*>(segment.av) + row);
        } else if constexpr (kCodec == kCodecFor16) {
          key = for_minimum + __ldg(static_cast<const uint16_t*>(segment.av) + row);
        } else {
          key = for_minimum + ld_stream_u32(static_cast<const uint32_t*>(segment.av) + row);
        }
      }
      const uint32_t index = key - direct_min;  // wraps above the range for keys below the minimum
      if (valid && index < direct_range) match = __ldg(direct + index);
    }
    const uint32_t partition = key & partition_mask;
    if constexpr (!kRank) {
      // Counting needs no order: one shared-memory reduction per emitting lane (measured 1.3 cycles per warp instruction
      // and SM with 4-way address conflicts, against 16 for MATCH.ANY alone — tools/micro/warp_ops.cu).
      if (match != kNoMatch) atomicAdd(histogram + partition, 1u);
    } else {
      const uint32_t peers = __match_any_sync(kFullMask, partition);
      const uint32_t emitting = __ballot_sync(kFullMask, match != kNoMatch) & peers;
      const int leader = __ffs(peers) - 1;
      uint32_t earlier = 0;
      if (lane == static_cast<uint32_t>(leader) && emitting) earlier = atomicAdd(histogram + partition, __popc(emitting));
      earlier = __shfl_sync(kFullMask, earlier, leader);
      rows.match[step] = match;
      rows.rank[step] = earlier + __popc(emitting & lanes_below);
      rows.partitions[step >> 2] |= partition << (8 * (step & 3));
    }
  }
}

template <bool kRank, bool kFull>
__device__ __forceinline__ void probe_chunk_fast_any_codec(const ProbeParams& params, const TileRef& ref, const DevSegment& segment,
                                                           uint32_t codec, uint32_t chunk0, uint32_t lane, uint32_t* histogram,
                                                           ChunkRows& rows) {
  switch (codec) {
    case kCodecPlain32:
      return probe_chunk_fast<kRank, kCodecPlain32, kFull>(params, ref, segment, chunk0, lane, histogram, rows);
    case kCodecFor8:
      return probe_chunk_fast<kRank, kCodecFor8, kFull>(params, ref, segment, chunk0, lane, histogram, rows);
    case kCodecFor16:
      return probe_chunk_fast<kRank, kCodecFor16, kFull>(params, ref, segment, chunk0, lane, histogram, rows);
    case kCodecPlain64:
      return probe_chunk_fast<kRank, kCodecPlain64, kFull>(params, ref, segment, chunk0, lane, histogram, rows);
    default:
      return probe_chunk_fast<kRank, kCodecFor32, kFull>(params, ref, segment, chunk0, lane, histogram, rows);
  }
}

// params.fast: 1 = int32 keys on both sides, unshifted direct table (32-bit arithmetic for every plain / FoR codec);
// 2 = int64 probe keys against a (possibly shifted) direct table: plain int64 segments only.
__device__ __forceinline__ bool fast_tile(const ProbeParams& params, uint32_t codec) {
  if (!params.unique_build || codec == kCodecGeneric) return false;
  return params.fast == 1 ? codec != kCodecPlain64 : (params.fast == 2 && codec == kCodecPlain64);
}

template <bool kRank, int kSource>
__device__ __forceinline__ void probe_chunk_any_codec(const ProbeParams& params, const TileRef& ref, const DevSegment& segment,
                                                      uint32_t codec, uint32_t chunk0, size_t tile_slot0, uint32_t lane,
                                                      bool build_has_nulls, uint32_t* histogram, ChunkRows& rows) {
  switch (codec) {
    case kCodecPlain32:
      return probe_chunk<kRank, kSource, kCodecPlain32>(params, ref, segment, chunk0, tile_slot0, lane, build_has_nulls, histogram, rows);
    case kCodecPlain64:
      return probe_chunk<kRank, kSource, kCodecPlain64>(params, ref, segment, chunk0, tile_slot0, lane, build_has_nulls, histogram, rows);
    case kCodecFor8:
      return probe_chunk<kRank, kSource, kCodecFor8>(params, ref, segment, chunk0, tile_slot0, lane, build_has_nulls, histogram, rows);
    case kCodecFor16:
      return probe_chunk<kRank, kSource, kCodecFor16>(params, ref, segment, chunk0, tile_slot0, lane, build_has_nulls, histogram, rows);
    case kCodecFor32:
      return probe_chunk<kRank, kSource, kCodecFor32>(params, ref, segment, chunk0, tile_slot0, lane, build_has_nulls, histogram, rows);
    default:
      return probe_chunk<kRank, kSource, kCodecGeneric>(params, ref, segment, chunk0, tile_slot0, lane, build_has_nulls, histogram, rows);
  }
}

// Emitted rows per (partition, tile). kStore: also keep match/partition per probe slot for the write kernel.
// kSecondary: the secondary predicates' variant (generic decoder, candidates evaluated per probe row).
template <bool kStore, bool kSecondary>
__device__ __forceinline__ void probe_count_tiles(const ProbeParams& params, const SecondaryPredicates& secondary) {
  __shared__ uint32_t s_histogram[kMaxPartitions];
  const bool build_has_nulls = params.flags[1] != 0;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t tile = blockIdx.x; tile < params.probe.tile_count; tile += gridDim.x) {
    for (uint32_t p = threadIdx.x; p < params.partition_count; p += kJoinThreads) s_histogram[p] = 0;
    __syncthreads();
    const TileRef ref = tile_ref(params.probe, tile);
    const DevSegment segment = params.probe.tile_map ? params.probe.segments[ref.chunk] : DevSegment{};
    const size_t tile_slot0 = static_cast<size_t>(tile) * kJoinTileRows;
    ChunkRows rows;
    if constexpr (kSecondary) {
      probe_chunk<false, kStore ? 1 : 0, kCodecGeneric, true>(params, ref, segment, warp * kJoinRowsPerWarp, tile_slot0, lane,
                                                             build_has_nulls, s_histogram, rows, secondary);
    } else {
      const uint32_t codec = tile_codec(params.probe, segment);
      if (!kStore && fast_tile(params, codec)) {
        if (ref.row0 + kJoinTileRows <= segment.row_count) {
          probe_chunk_fast_any_codec<false, true>(params, ref, segment, codec, warp * kJoinRowsPerWarp, lane, s_histogram, rows);
        } else {
          probe_chunk_fast_any_codec<false, false>(params, ref, segment, codec, warp * kJoinRowsPerWarp, lane, s_histogram, rows);
        }
      } else {
        probe_chunk_any_codec<false, kStore ? 1 : 0>(params, ref, segment, codec, warp * kJoinRowsPerWarp, tile_slot0, lane,
                                                     build_has_nulls, s_histogram, rows);
      }
    }
    __syncthreads();
    for (uint32_t p = threadIdx.x; p < params.partition_count; p += kJoinThreads) {
      params.histogram[static_cast<size_t>(p) * params.probe.tile_count + tile] = s_histogram[p];
    }
    __syncthreads();
  }
}

template <bool kStore>
__global__ void __launch_bounds__(kJoinThreads, 5) join_probe_count_kernel(const ProbeParams params) {
  probe_count_tiles<kStore, false>(params, SecondaryPredicates{});
}

template <bool kStore>
__global__ void __launch_bounds__(kJoinThreads, 3) join_probe_secondary_count_kernel(const ProbeParams params,
                                                                                     const SecondaryPredicates secondary) {
  probe_count_tiles<kStore, true>(params, secondary);
}

// Stable multi-split: every probe row's output position = start of its (partition, tile) run (exclusive scan of the
// histogram) + rows of lower warp chunks of the tile in that partition + its rank inside the warp chunk.
template <bool kStored, bool kSecondary>
__device__ __forceinline__ void probe_write_tiles(const ProbeParams& params, const SecondaryPredicates& secondary) {
  __shared__ uint32_t s_warp_histogram[kJoinWarps][kMaxPartitions];
  __shared__ unsigned long long s_start[kJoinWarps][kMaxPartitions];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool emit_build = params.out_build != nullptr;
  const bool unique = params.unique_build != 0;
  const bool build_has_nulls = params.flags[1] != 0;

  // Blocked tile assignment: a CTA's consecutive tiles extend the same 256 (partition) output runs, so the partly
  // written 32-byte sectors at the run boundaries are completed while they are still in L2.
  const uint32_t tiles_per_cta = (params.probe.tile_count + gridDim.x - 1) / gridDim.x;
  const uint32_t tile_end = min(params.probe.tile_count, (blockIdx.x + 1) * tiles_per_cta);
  for (uint32_t tile = blockIdx.x * tiles_per_cta; tile < tile_end; ++tile) {
    for (uint32_t p = lane; p < params.partition_count; p += 32) s_warp_histogram[warp][p] = 0;
    __syncwarp();
    const TileRef ref = tile_ref(params.probe, tile);
    const DevSegment segment = params.probe.tile_map ? params.probe.segments[ref.chunk] : DevSegment{};
    const size_t tile_slot0 = static_cast<size_t>(tile) * kJoinTileRows;
    ChunkRows rows;
    const uint32_t codec = (kStored || kSecondary) ? kCodecGeneric : tile_codec(params.probe, segment);
    const bool fast = !kStored && !kSecondary && fast_tile(params, codec);
    if (fast) {
      if (ref.row0 + kJoinTileRows <= segment.row_count) {
        probe_chunk_fast_any_codec<true, true>(params, ref, segment, codec, warp * kJoinRowsPerWarp, lane, s_warp_histogram[warp], rows);
      } else {
        probe_chunk_fast_any_codec<true, false>(params, ref, segment, codec, warp * kJoinRowsPerWarp, lane, s_warp_histogram[warp], rows);
      }
    } else if constexpr (kSecondary) {
      probe_chunk<true, kStored ? 2 : 0, kCodecGeneric, true>(params, ref, segment, warp * kJoinRowsPerWarp, tile_slot0, lane,
                                                             build_has_nulls, s_warp_histogram[warp], rows, secondary);
    } else {
      probe_chunk_any_codec<true, kStored ? 2 : 0>(params, ref, segment, codec, warp * kJoinRowsPerWarp, tile_slot0, lane,
                                                   build_has_nulls, s_warp_histogram[warp], rows);
    }
    __syncthreads();
    for (uint32_t p = threadIdx.x; p < params.partition_count; p += kJoinThreads) {
      unsigned long long running = params.run_starts[static_cast<size_t>(p) * params.probe.tile_count + tile];
#pragma unroll
      for (int w = 0; w < kJoinWarps; ++w) {
        s_start[w][p] = running;
        running += s_warp_histogram[w][p];
      }
    }
    __syncthreads();
    if (fast) {
      // unique build side: one output row per match, `match` is the build position; capacity == probe positions suffices
      const uint32_t row_base = ref.row0 + warp * kJoinRowsPerWarp + lane;
#pragma unroll
      for (int step = 0; step < kProbeSteps; ++step) {
        const uint32_t match = rows.match[step];
        if (match == kNoMatch) continue;
        const uint32_t partition = (rows.partitions[step >> 2] >> (8 * (step & 3))) & 0xFFu;
        const unsigned long long at = s_start[warp][partition] + rows.rank[step];
        const hyb_row_id build_row = position_to_row_id(params.build, match);
        st_stream_v2(params.out_build + at, build_row.chunk_id, build_row.chunk_offset);
        if (params.probe.payload) {
          const hyb_row_id probe_row = params.probe.payload[ref.first_position + (row_base - ref.row0) + step * 32];
          st_stream_v2(params.out_probe + at, probe_row.chunk_id, probe_row.chunk_offset);
        } else {
          st_stream_v2(params.out_probe + at, ref.chunk + params.probe.chunk_id_base, row_base + step * 32);
        }
      }
      __syncthreads();
      continue;
    }
#pragma unroll
    for (int step = 0; step < kProbeSteps; ++step) {
      const uint32_t match = rows.match[step];
      // secondary predicates: the candidate loop below checks the capacity row by row
      const uint32_t emit = kSecondary ? (match == kNoMatch ? 0u : 1u) : emitted_rows(params, match);
      if (emit == 0) continue;
      const uint32_t index = warp * kJoinRowsPerWarp + step * 32 + lane;
      const uint32_t partition = (rows.partitions[step >> 2] >> (8 * (step & 3))) & 0xFFu;
      const unsigned long long at = s_start[warp][partition] + rows.rank[step];
      if (at + emit > params.out_capacity) {
        *params.overflow = 1;
        continue;
      }
      hyb_row_id probe_row;
      if (params.probe.tile_map) {
        probe_row = params.probe.payload ? params.probe.payload[ref.first_position + index]
                                         : hyb_row_id{ref.chunk + params.probe.chunk_id_base, ref.row0 + index};
      } else {
        probe_row = params.probe.filter[ref.first_position + index];
        if (probe_row.chunk_id != HYB_INVALID_CHUNK_ID) probe_row.chunk_id += params.probe.chunk_id_base;
      }
      if (match == kEmitWithoutPartner) {
        if (emit_build) st_stream_v2(params.out_build + at, HYB_INVALID_CHUNK_ID, HYB_INVALID_CHUNK_OFFSET);
        st_stream_v2(params.out_probe + at, probe_row.chunk_id, probe_row.chunk_offset);
      } else if constexpr (kSecondary) {
        write_passing_candidates(params, secondary, match, probe_row, at);
      } else if (unique) {
        const hyb_row_id build_row = position_to_row_id(params.build, match);
        st_stream_v2(params.out_build + at, build_row.chunk_id, build_row.chunk_offset);
        st_stream_v2(params.out_probe + at, probe_row.chunk_id, probe_row.chunk_offset);
      } else {
        const unsigned long long first = params.dup_offsets[match];
        for (uint32_t j = 0; j < emit; ++j) {
          const hyb_row_id build_row = position_to_row_id(params.build, params.dup_positions[first + j]);
          st_stream_v2(params.out_build + at + j, build_row.chunk_id, build_row.chunk_offset);
          st_stream_v2(params.out_probe + at + j, probe_row.chunk_id, probe_row.chunk_offset);
        }
      }
    }
    __syncthreads();
  }
}

template <bool kStored>
__global__ void __launch_bounds__(kJoinThreads, 3) join_probe_write_kernel(const ProbeParams params) {
  probe_write_tiles<kStored, false>(params, SecondaryPredicates{});
}

// (two CTAs per SM: at the 80 registers of three the candidate loops spilled 104-184 bytes; at 128 the direct-table
// variant does not spill and the hash-table variant, kStored, still spills 24 bytes)
template <bool kStored>
__global__ void __launch_bounds__(kJoinThreads, 2) join_probe_secondary_write_kernel(const ProbeParams params,
                                                                                     const SecondaryPredicates secondary) {
  probe_write_tiles<kStored, true>(params, secondary);
}

// ---------------------------------------------------------------------------------------------------------------------
// Span kernels: the Inner / unique-build / direct-or-rank-table path (TPC-H's PK-FK joins) over 8192-row spans.
//
// What bounded the 4096-row tile kernels was not DRAM but the store path: every probe row wrote its two RowIDs with two
// 8-byte stores into ~256-byte runs (a tile's 32 rows per partition), 32 different sectors per warp instruction. Here a
// CTA owns 8192 consecutive probe rows and scatters {build position, row index | partition} into SHARED memory at the
// row's position inside the span's partition-ordered output; the span's output then leaves in one flat loop in which
// consecutive threads hold consecutive output rows of a run, so every warp store is 256 contiguous bytes per PosList.
//
//   join_span_count_kernel   matches per (span, 512-row warp chunk, partition) as uint16 + per (partition, span) totals.
//                            The fine counts are what lets the write pass be a SINGLE sweep: a warp knows where its rows
//                            of a partition start inside the staged span before it has ranked anything, so a row is
//                            looked up, ranked (lane order = probe order) and scattered at once — no per-row state in
//                            registers, no barrier between ranking and scattering.
//   exclusive scan           over the (partition, span) totals: the run starts in the output.
//   join_span_write_kernel   the sweep + the flat coalesced write-out.
// All 16 key loads of a lane are issued before the first use; table lookups follow in groups of kSpanGroup.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kSpanThreads = 512;
constexpr int kSpanWarps = kSpanThreads / 32;
constexpr int kSpanRows = kSpanWarps * kJoinRowsPerWarp;  // 8192
constexpr int kSpanGroup = 4;                             // table lookups in flight together
enum : int { kTableDirect = 0, kTableRank = 1 };

struct SpanKeys {
  uint32_t low[kProbeSteps];
  uint32_t valid_mask;
};

// Keys of all 16 probe steps of a lane: step s, lane l -> row row_base + 32 s.
template <uint32_t kCodec, bool kFull>
__device__ __forceinline__ void span_load_keys(const DevSegment& segment, uint32_t row_base, uint32_t for_minimum, SpanKeys& keys,
                                               uint32_t (&high)[kCodec == kCodecPlain64 ? kProbeSteps : 1]) {
  const uint32_t row_count = segment.row_count;
  keys.valid_mask = 0;
#pragma unroll
  for (int s = 0; s < kProbeSteps; ++s) {
    const uint32_t row = row_base + s * 32;
    const bool valid = kFull || row < row_count;
    keys.valid_mask |= valid ? (1u << s) : 0u;
    keys.low[s] = 0;
    if constexpr (kCodec == kCodecPlain64) high[s] = 0;
    if (valid) {
      if constexpr (kCodec == kCodecPlain32) {
        keys.low[s] = ld_stream_u32(static_cast<const uint32_t*>(segment.values) + row);
      } else if constexpr (kCodec == kCodecPlain64) {
        const uint2 bits = ld_stream_v2(static_cast<const long long*>(segment.values) + row);
        keys.low[s] = bits.x;
        high[s] = bits.y;
      } else if constexpr (kCodec == kCodecFor8) {
        keys.low[s] = for_minimum + __ldg(static_cast<const uint8_t*>(segment.av) + row);
      } else if constexpr (kCodec == kCodecFor16) {
        keys.low[s] = for_minimum + __ldg(static_cast<const uint16_t*>(segment.av) + row);
      } else {
        keys.low[s] = for_minimum + ld_stream_u32(static_cast<const uint32_t*>(segment.av) + row);
      }
    }
  }
}

// Matches (build position or kNoMatch) of steps first .. first + kSpanGroup - 1.
template <uint32_t kCodec, int kTable>
__device__ __forceinline__ void span_match(const ProbeParams& params, const SpanKeys& keys,
                                           const uint32_t (&high)[kCodec == kCodecPlain64 ? kProbeSteps : 1], int first,
                                           uint32_t (&match)[kSpanGroup]) {
  constexpr bool kWide = kCodec == kCodecPlain64;
  static_assert(!(kWide && kTable == kTableRank), "rank tables are probed with int32 keys");
  if constexpr (kTable == kTableRank) {
    const uint2* __restrict__ blocks = params.table.rank_blocks;
    const uint32_t minimum = static_cast<uint32_t>(params.table.direct_min);
    const uint32_t range = static_cast<uint32_t>(params.table.direct_range);
    uint2 block[kSpanGroup];
#pragma unroll
    for (int s = 0; s < kSpanGroup; ++s) {
      const uint32_t offset = keys.low[first + s] - minimum;  // wraps above the range for keys below the minimum
      block[s] = make_uint2(0u, 0u);
      if (((keys.valid_mask >> (first + s)) & 1u) && offset < range) block[s] = __ldg(blocks + (offset >> 5));
    }
#pragma unroll
    for (int s = 0; s < kSpanGroup; ++s) {
      const uint32_t bit = (keys.low[first + s] - minimum) & 31u;
      match[s] = ((block[s].x >> bit) & 1u) ? rank_block_position(block[s], bit) : kNoMatch;
    }
  } else if constexpr (!kWide) {
    const uint32_t* __restrict__ direct = params.table.direct;
    const uint32_t minimum = static_cast<uint32_t>(params.table.direct_min);
    const uint32_t range = static_cast<uint32_t>(params.table.direct_range);
#pragma unroll
    for (int s = 0; s < kSpanGroup; ++s) {
      const uint32_t index = keys.low[first + s] - minimum;
      match[s] = kNoMatch;
      if (((keys.valid_mask >> (first + s)) & 1u) && index < range) match[s] = __ldg(direct + index);
    }
  } else {
    const uint32_t* __restrict__ direct = params.table.direct;
    const unsigned long long minimum = static_cast<unsigned long long>(params.table.direct_min);
    const unsigned long long range = params.table.direct_range;
    const uint32_t shift = params.table.direct_shift;
    const unsigned long long low_bits = (1ull << shift) - 1ull;
#pragma unroll
    for (int s = 0; s < kSpanGroup; ++s) {
      const unsigned long long offset = ((static_cast<unsigned long long>(high[first + s]) << 32) | keys.low[first + s]) - minimum;
      const unsigned long long index = offset >> shift;
      match[s] = kNoMatch;
      if (((keys.valid_mask >> (first + s)) & 1u) && index < range && !(offset & low_bits)) match[s] = __ldg(direct + index);
    }
  }
}

__device__ __forceinline__ uint32_t span_for_minimum(const DevSegment& segment, uint32_t codec, uint32_t first_row) {
  // first_row is a multiple of 512 and spans start at multiples of 8192: a warp chunk lies inside one 2048-row block
  if (codec < kCodecFor8 || first_row >= segment.row_count) return 0;
  return static_cast<uint32_t>(__ldg(static_cast<const int32_t*>(segment.values) + first_row / HYB_FOR_BLOCK_SIZE));
}

// Lanes of the warp whose row falls into the same radix partition: MATCH.ANY (the default), or one ballot per radix bit
// (selectable, option join_rank).
template <bool kBallot>
__device__ __forceinline__ uint32_t partition_peers(uint32_t partition, uint32_t radix_bits) {
  if constexpr (kBallot) {
    uint32_t peers = kFullMask;
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      if (static_cast<uint32_t>(b) < radix_bits) {  // uniform
        const bool set = (partition >> b) & 1u;
        const uint32_t vote = __ballot_sync(kFullMask, set);
        peers &= set ? vote : ~vote;
      }
    }
    return peers;
  } else {
    return __match_any_sync(kFullMask, partition);
  }
}

// One warp chunk (512 rows) of a span. kScatter == false: count matches per partition into `counters` (this warp's
// histogram). kScatter == true: `counters[p]` holds the staged position of the chunk's next row of partition p; every
// matching row is ranked in lane order and stored at once.
template <uint32_t kCodec, bool kFull, int kTable, bool kScatter, bool kBallot>
__device__ __forceinline__ void span_warp_chunk(const ProbeParams& params, const TileRef& ref, const DevSegment& segment,
                                                uint32_t warp, uint32_t lane, uint32_t* counters, uint2* stage) {
  const uint32_t chunk0 = warp * kJoinRowsPerWarp;
  const uint32_t for_minimum = span_for_minimum(segment, kCodec, ref.row0 + chunk0);
  const uint32_t lanes_below = (1u << lane) - 1u;
  const uint32_t radix_bits = __popc(params.partition_mask);
  SpanKeys keys;
  uint32_t high[kCodec == kCodecPlain64 ? kProbeSteps : 1];
  span_load_keys<kCodec, kFull>(segment, ref.row0 + chunk0 + lane, for_minimum, keys, high);
#pragma unroll
  for (int group = 0; group < kProbeSteps / kSpanGroup; ++group) {
    uint32_t match[kSpanGroup];
    span_match<kCodec, kTable>(params, keys, high, group * kSpanGroup, match);
#pragma unroll
    for (int s = 0; s < kSpanGroup; ++s) {
      const int step = group * kSpanGroup + s;
      const uint32_t partition = keys.low[step] & params.partition_mask;
      if constexpr (!kScatter) {
        if (match[s] != kNoMatch) atomicAdd(counters + partition, 1u);  // counting needs no order
      } else {
        // (run detection for sorted probe keys — equal keys adjacent, one shuffle + two votes instead of MATCH.ANY — was
        //  measured: 5.57 vs 5.65 ms at SF 100, within noise; the ranking primitive is not what bounds this kernel)
        const uint32_t peers = partition_peers<kBallot>(partition, radix_bits);
        const uint32_t emitting = __ballot_sync(kFullMask, match[s] != kNoMatch) & peers;
        const int leader = __ffs(peers) - 1;
        uint32_t base = 0;
        if (lane == static_cast<uint32_t>(leader) && emitting) base = atomicAdd(counters + partition, __popc(emitting));
        base = __shfl_sync(kFullMask, base, leader);
        if (match[s] != kNoMatch) {
          stage[base + __popc(emitting & lanes_below)] = make_uint2(match[s], (chunk0 + step * 32 + lane) | (partition << 16));
        }
      }
    }
  }
}

// Codec and span fullness are uniform per span: one switch per CTA in front of fully specialised loops.
#define HYB_SPAN_DISPATCH(CALL)                                                    \
  do {                                                                             \
    const bool span_full = ref.row0 + kSpanRows <= segment.row_count;              \
    if constexpr (kTable == kTableRank) {                                          \
      switch (codec) {                                                             \
        case kCodecPlain32:                                                        \
          if (span_full) CALL(kCodecPlain32, true) else CALL(kCodecPlain32, false) \
          break;                                                                   \
        case kCodecFor8:                                                           \
          if (span_full) CALL(kCodecFor8, true) else CALL(kCodecFor8, false)       \
          break;                                                                   \
        case kCodecFor16:                                                          \
          if (span_full) CALL(kCodecFor16, true) else CALL(kCodecFor16, false)     \
          break;                                                                   \
        default:                                                                   \
          if (span_full) CALL(kCodecFor32, true) else CALL(kCodecFor32, false)     \
          break;                                                                   \
      }                                                                            \
    } else {                                                                       \
      switch (codec) {                                                             \
        case kCodecPlain32:                                                        \
          if (span_full) CALL(kCodecPlain32, true) else CALL(kCodecPlain32, false) \
          break;                                                                   \
        case kCodecPlain64:                                                        \
          if (span_full) CALL(kCodecPlain64, true) else CALL(kCodecPlain64, false) \
          break;                                                                   \
        case kCodecFor8:                                                           \
          if (span_full) CALL(kCodecFor8, true) else CALL(kCodecFor8, false)       \
          break;                                                                   \
        case kCodecFor16:                                                          \
          if (span_full) CALL(kCodecFor16, true) else CALL(kCodecFor16, false)     \
          break;                                                                   \
        default:                                                                   \
          if (span_full) CALL(kCodecFor32, true) else CALL(kCodecFor32, false)     \
          break;                                                                   \
      }                                                                            \
    }                                                                              \
  } while (0)

// params.probe is the span-granular source (tile map of kSpanRows-row tiles). Dynamic shared memory (both kernels):
// uint32 counters[kSpanWarps][partition_count] (the write kernel: behind its kSpanRows staged rows).
// params.histogram[p * spans + span] = matches of partition p in the span; fine_counts[(span * kSpanWarps + w) *
// partition_count + p] = those of warp chunk w.
template <int kTable>
__global__ void __launch_bounds__(kSpanThreads, 2) join_span_count_kernel(const ProbeParams params, uint16_t* __restrict__ fine_counts) {
  extern __shared__ uint32_t s_counters[];  // [kSpanWarps][partition_count]
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t span = blockIdx.x;
  const uint32_t partition_count = params.partition_count;
  uint32_t* mine = s_counters + warp * partition_count;
  for (uint32_t p = lane; p < partition_count; p += 32) mine[p] = 0;
  __syncwarp();
  const TileRef ref = tile_ref(params.probe, span);
  const DevSegment segment = params.probe.segments[ref.chunk];
  const uint32_t codec = tile_codec(params.probe, segment);
#define HYB_SPAN_COUNT(CODEC, FULL) span_warp_chunk<CODEC, FULL, kTable, false, false>(params, ref, segment, warp, lane, mine, nullptr);
  HYB_SPAN_DISPATCH(HYB_SPAN_COUNT);
#undef HYB_SPAN_COUNT
  __syncthreads();
  uint16_t* out = fine_counts + static_cast<size_t>(span) * kSpanWarps * partition_count;
  for (uint32_t i = threadIdx.x; i < kSpanWarps * partition_count; i += kSpanThreads) out[i] = static_cast<uint16_t>(s_counters[i]);
  if (threadIdx.x < partition_count) {
    uint32_t total = 0;
#pragma unroll
    for (int w = 0; w < kSpanWarps; ++w) total += s_counters[w * partition_count + threadIdx.x];
    params.histogram[static_cast<size_t>(threadIdx.x) * params.probe.tile_count + span] = total;
  }
}

template <int kTable, bool kBallot>
__global__ void __launch_bounds__(kSpanThreads, 2) join_span_write_kernel(const ProbeParams params,
                                                                          const uint16_t* __restrict__ fine_counts) {
  extern __shared__ __align__(16) unsigned char s_dynamic[];
  uint2* s_stage = reinterpret_cast<uint2*>(s_dynamic);  // kSpanRows x {build position, row index in the span | partition << 16}
  uint32_t* s_position = reinterpret_cast<uint32_t*>(s_dynamic + sizeof(uint2) * kSpanRows);  // [kSpanWarps][partition_count]
  __shared__ uint32_t s_destination[kMaxPartitions];  // output index of staged row i of partition p = this + i (mod 2^32)
  __shared__ uint32_t s_scan[8];
  __shared__ uint32_t s_total;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t span = blockIdx.x;
  const uint32_t partition_count = params.partition_count;
  const TileRef ref = tile_ref(params.probe, span);
  const DevSegment segment = params.probe.segments[ref.chunk];
  const uint32_t codec = tile_codec(params.probe, segment);

  // ---- where every warp chunk's rows of every partition go inside the staged span (from the count pass) ----------------
  uint32_t partition_total = 0;
  unsigned long long run_start = 0;
  if (threadIdx.x < partition_count) {
    run_start = __ldg(params.run_starts + static_cast<size_t>(threadIdx.x) * params.probe.tile_count + span);
    const uint16_t* counts = fine_counts + static_cast<size_t>(span) * kSpanWarps * partition_count + threadIdx.x;
    uint32_t count[kSpanWarps];
#pragma unroll
    for (int w = 0; w < kSpanWarps; ++w) count[w] = __ldg(counts + w * partition_count);
#pragma unroll
    for (int w = 0; w < kSpanWarps; ++w) {
      s_position[w * partition_count + threadIdx.x] = partition_total;  // relative to the partition's first staged row
      partition_total += count[w];
    }
  }
  const uint32_t inclusive = warp_inclusive_scan(partition_total, lane);
  if (warp < 8 && lane == 31) s_scan[warp] = inclusive;
  __syncthreads();
  if (threadIdx.x < partition_count) {
    uint32_t before = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) before += w < static_cast<int>(warp) ? s_scan[w] : 0u;
    const uint32_t exclusive = before + inclusive - partition_total;
#pragma unroll
    for (int w = 0; w < kSpanWarps; ++w) s_position[w * partition_count + threadIdx.x] += exclusive;
    s_destination[threadIdx.x] = static_cast<uint32_t>(run_start) - exclusive;  // run_start + (i - exclusive) for staged row i
    if (threadIdx.x + 1 == partition_count) s_total = exclusive + partition_total;
  }
  __syncthreads();

  // ---- one sweep: look up, rank, scatter --------------------------------------------------------------------------------
  uint32_t* mine = s_position + warp * partition_count;
#define HYB_SPAN_SCATTER(CODEC, FULL) \
  span_warp_chunk<CODEC, FULL, kTable, true, kBallot>(params, ref, segment, warp, lane, mine, s_stage);
  HYB_SPAN_DISPATCH(HYB_SPAN_SCATTER);
#undef HYB_SPAN_SCATTER
  __syncthreads();

  // ---- flat write-out: consecutive threads, consecutive output rows of a run ---------------------------------------------
  // (output positions fit 32 bits: the output holds at most one row per probe position, and those are < 2^32)
  const uint32_t total = s_total;
  hyb_row_id* __restrict__ out_build = params.out_build;
  hyb_row_id* __restrict__ out_probe = params.out_probe;
  const uint32_t build_base = params.build.chunk_id_base, probe_chunk = ref.chunk + params.probe.chunk_id_base;
  if (!params.build.filter && !params.build.payload && !params.probe.payload && params.build.uniform_chunk_rows) {
    // build position -> RowID by an exact multiply-shift division (all chunks but the last have uniform_chunk_rows rows)
    const uint32_t magic = params.build.uniform_magic, shift = params.build.uniform_shift;
    const uint32_t chunk_rows = params.build.uniform_chunk_rows;
    for (uint32_t i = threadIdx.x; i < total; i += kSpanThreads) {
      const uint2 staged = s_stage[i];
      const uint32_t at = s_destination[staged.y >> 16] + i;
      const uint32_t n = staged.x;
      const uint32_t t = __umulhi(n, magic);
      const uint32_t chunk = shift == 0 ? n : (t + ((n - t) >> 1)) >> (shift - 1);
      st_stream_v2(out_build + at, chunk + build_base, n - chunk * chunk_rows);
      st_stream_v2(out_probe + at, probe_chunk, ref.row0 + (staged.y & 0xFFFFu));
    }
  } else if (params.probe.payload) {
    // received tuples: both sides emit the RowIDs that travelled with the keys; the probe side's lie in this span's slice
    const hyb_row_id* __restrict__ probe_payload = params.probe.payload + ref.first_position;
    for (uint32_t i = threadIdx.x; i < total; i += kSpanThreads) {
      const uint2 staged = s_stage[i];
      const uint32_t at = s_destination[staged.y >> 16] + i;
      const hyb_row_id build_row = position_to_row_id(params.build, staged.x);
      const hyb_row_id probe_row = probe_payload[staged.y & 0xFFFFu];
      st_stream_v2(out_build + at, build_row.chunk_id, build_row.chunk_offset);
      st_stream_v2(out_probe + at, probe_row.chunk_id, probe_row.chunk_offset);
    }
  } else {
    for (uint32_t i = threadIdx.x; i < total; i += kSpanThreads) {
      const uint2 staged = s_stage[i];
      const uint32_t at = s_destination[staged.y >> 16] + i;
      const hyb_row_id build_row = position_to_row_id(params.build, staged.x);
      st_stream_v2(out_build + at, build_row.chunk_id, build_row.chunk_offset);
      st_stream_v2(out_probe + at, probe_chunk, ref.row0 + (staged.y & 0xFFFFu));
    }
  }
}
#undef HYB_SPAN_DISPATCH

// hyb_join_partition / hyb_join_partition_push / hyb_join_hash_distributed, ranked-write pass: the stable split of one
// side's non-NULL {key, global RowID} tuples by owner rank. Same ranking as join_probe_write_kernel, nothing is looked up,
// the keys stay in registers between the passes. The tile's tuples are first scattered into SHARED memory in destination
// order and then leave in one flat loop, so every warp store is 256 contiguous bytes per array INSIDE ONE DESTINATION —
// what NVLink wants (8-byte stores into 32-byte runs, as the direct scatter produced at world = 8, waste most of every
// packet). Destinations are local buffers, or (push_to_peers) the owners' memory over NVLink.
constexpr size_t kPartitionStageBytes = sizeof(uint4) * kJoinTileRows;  // dynamic shared memory of the kernel

__global__ void __launch_bounds__(kJoinThreads, 3) join_partition_write_kernel(const ProbeParams params) {
  extern __shared__ uint4 s_tuples[];  // kJoinTileRows x {key low, key high, RowID chunk, RowID offset}, destination-major
  __shared__ uint32_t s_warp_histogram[kJoinWarps][kMaxPartitions];  // counts, then exclusive prefixes over the warps
  __shared__ uint32_t s_local_start[kMaxPartitions];
  __shared__ unsigned long long s_destination[kMaxPartitions];  // index in the destination array of staged tuple i = this + i
  __shared__ long long* s_keys_out[kMaxPeers];
  __shared__ long long* s_rows_out[kMaxPeers];
  __shared__ uint32_t s_scan[kJoinWarps];
  __shared__ uint32_t s_total;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lanes_below = (1u << lane) - 1u;
  const uint32_t partition_count = params.partition_count;
  const bool push = params.push_to_peers != 0;
  if (threadIdx.x < kMaxPeers) {
    s_keys_out[threadIdx.x] = push ? params.peer_keys[threadIdx.x] : reinterpret_cast<long long*>(params.out_build);
    s_rows_out[threadIdx.x] = push ? params.peer_rows[threadIdx.x] : reinterpret_cast<long long*>(params.out_probe);
  }
  const uint32_t tiles_per_cta = (params.probe.tile_count + gridDim.x - 1) / gridDim.x;
  const uint32_t tile_end = min(params.probe.tile_count, (blockIdx.x + 1) * tiles_per_cta);
  for (uint32_t tile = blockIdx.x * tiles_per_cta; tile < tile_end; ++tile) {
    for (uint32_t p = lane; p < partition_count; p += 32) s_warp_histogram[warp][p] = 0;
    __syncwarp();
    const TileRef ref = tile_ref(params.probe, tile);
    const DevSegment segment = params.probe.tile_map ? params.probe.segments[ref.chunk] : DevSegment{};
    const uint32_t codec = tile_codec(params.probe, segment);
    const uint32_t chunk0 = warp * kJoinRowsPerWarp;
    uint32_t for_minimum = 0;
    if (codec >= kCodecFor8 && ref.row0 + chunk0 < segment.row_count) {
      for_minimum = static_cast<uint32_t>(__ldg(static_cast<const int32_t*>(segment.values) + (ref.row0 + chunk0) / HYB_FOR_BLOCK_SIZE));
    }
    // this tile's run starts (exclusive scan of the count pass), in flight while the rows are ranked
    unsigned long long run_start = 0;
    if (threadIdx.x < partition_count) {
      const size_t first = static_cast<size_t>(threadIdx.x) * params.probe.tile_count;
      run_start = __ldg(params.run_starts + first + tile);
      if (push) run_start -= __ldg(params.run_starts + first);  // peers receive a pointer to the start of their group
    }
    uint32_t key_low[kProbeSteps], key_high[kProbeSteps], rank[kProbeSteps];
    uint32_t emit_mask = 0;
#pragma unroll
    for (int step = 0; step < kProbeSteps; ++step) {
      const uint32_t index = chunk0 + step * 32 + lane;
      long long key = 0;
      bool is_null = false;
      bool valid;
      // uniform per tile: the specialised decoders of the probe for the layouts that dominate, the generic one otherwise
      switch (codec) {
        case kCodecPlain32:
          valid = codec_key<kCodecPlain32>(params.probe, ref, segment, index, for_minimum, key, is_null);
          break;
        case kCodecFor8:
          valid = codec_key<kCodecFor8>(params.probe, ref, segment, index, for_minimum, key, is_null);
          break;
        case kCodecFor16:
          valid = codec_key<kCodecFor16>(params.probe, ref, segment, index, for_minimum, key, is_null);
          break;
        case kCodecFor32:
          valid = codec_key<kCodecFor32>(params.probe, ref, segment, index, for_minimum, key, is_null);
          break;
        default:
          valid = load_key1(params.probe, ref, segment, index, key, is_null);
          break;
      }
      const bool emit = valid && !is_null;
      const uint32_t partition = static_cast<uint32_t>(static_cast<unsigned long long>(key)) & params.partition_mask;
      const uint32_t peers = __match_any_sync(kFullMask, partition);
      const uint32_t emitting = __ballot_sync(kFullMask, emit) & peers;
      const int leader = __ffs(peers) - 1;
      uint32_t earlier = 0;
      if (lane == static_cast<uint32_t>(leader) && emitting) earlier = atomicAdd(&s_warp_histogram[warp][partition], __popc(emitting));
      earlier = __shfl_sync(kFullMask, earlier, leader);
      key_low[step] = static_cast<uint32_t>(static_cast<unsigned long long>(key));
      key_high[step] = static_cast<uint32_t>(static_cast<unsigned long long>(key) >> 32);
      rank[step] = earlier + __popc(emitting & lanes_below);
      emit_mask |= emit ? (1u << step) : 0u;
    }
    __syncthreads();
    // per destination: exclusive prefix over the warp chunks, then over the destinations
    uint32_t partition_total = 0;
    if (threadIdx.x < partition_count) {
#pragma unroll
      for (int w = 0; w < kJoinWarps; ++w) {
        const uint32_t count = s_warp_histogram[w][threadIdx.x];
        s_warp_histogram[w][threadIdx.x] = partition_total;
        partition_total += count;
      }
    }
    const uint32_t inclusive = warp_inclusive_scan(partition_total, lane);
    if (lane == 31) s_scan[warp] = inclusive;
    __syncthreads();
    if (threadIdx.x < partition_count) {
      uint32_t before = 0;
#pragma unroll
      for (int w = 0; w < kJoinWarps; ++w) before += w < static_cast<int>(warp) ? s_scan[w] : 0u;
      const uint32_t exclusive = before + inclusive - partition_total;
      s_local_start[threadIdx.x] = exclusive;
      s_destination[threadIdx.x] = run_start - exclusive;  // modulo 2^64
      if (threadIdx.x + 1 == partition_count) s_total = exclusive + partition_total;
    }
    __syncthreads();
#pragma unroll
    for (int step = 0; step < kProbeSteps; ++step) {
      if (!((emit_mask >> step) & 1u)) continue;
      const uint32_t index = chunk0 + step * 32 + lane;
      const uint32_t partition = key_low[step] & params.partition_mask;
      hyb_row_id row;
      if (params.probe.tile_map) {
        row = hyb_row_id{ref.chunk, ref.row0 + index};
      } else {
        row = params.probe.filter[ref.first_position + index];
      }
      s_tuples[s_local_start[partition] + s_warp_histogram[warp][partition] + rank[step]] =
          make_uint4(key_low[step], key_high[step], row.chunk_id + params.chunk_id_base, row.chunk_offset);
    }
    __syncthreads();
    const uint32_t total = s_total;
    for (uint32_t i = threadIdx.x; i < total; i += kJoinThreads) {
      const uint4 tuple = s_tuples[i];
      const uint32_t partition = tuple.x & params.partition_mask;
      const unsigned long long at = s_destination[partition] + i;
      const uint32_t owner = push ? partition : 0u;
      st_stream_v2(s_keys_out[owner] + at, tuple.x, tuple.y);
      st_stream_v2(s_rows_out[owner] + at, tuple.z, tuple.w);
    }
    __syncthreads();
  }
  peer_signal_when_last(params);
}

// Multi-GPU exchange payload: {key, packed global RowID} per position; NULL keys are marked with RowID -1.
__global__ void __launch_bounds__(kJoinThreads) join_materialize_kernel(const KeySource source, uint32_t chunk_id_base,
                                                                        long long* __restrict__ out_keys,
                                                                        long long* __restrict__ out_row_ids) {
  for (uint32_t tile = blockIdx.x; tile < source.tile_count; tile += gridDim.x) {
    const TileRef ref = tile_ref(source, tile);
    const DevSegment segment = source.tile_map ? source.segments[ref.chunk] : DevSegment{};
    for (uint32_t index = threadIdx.x; index < kJoinTileRows; index += kJoinThreads) {
      long long key;
      bool is_null;
      if (!load_key1(source, ref, segment, index, key, is_null)) continue;
      const unsigned long long position = ref.first_position + index;
      hyb_row_id row_id;
      if (source.tile_map) {
        row_id = hyb_row_id{ref.chunk, ref.row0 + index};
      } else {
        row_id = source.filter[position];
      }
      out_keys[position] = key;
      out_row_ids[position] = is_null ? -1ll
                                      : static_cast<long long>(static_cast<unsigned long long>(row_id.chunk_id + chunk_id_base) |
                                                               (static_cast<unsigned long long>(row_id.chunk_offset) << 32));
    }
  }
}

__global__ void join_partition_offsets_kernel(const unsigned long long* __restrict__ run_starts,
                                              const unsigned long long* __restrict__ total, uint32_t partition_count,
                                              uint32_t tile_count, unsigned long long* __restrict__ out) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > partition_count) return;
  out[p] = (p == partition_count || tile_count == 0) ? *total : run_starts[static_cast<size_t>(p) * tile_count];
}

// ---------------------------------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------------------------------
// JoinHash::calculate_radix_bits (join_hash.cpp:70-114)
static int32_t calculate_radix_bits(uint64_t build_side_size) {
  constexpr double kL2CacheMaxUsable = 1'024'000 * 0.75;
  const double complete_hash_map_size = static_cast<double>(build_side_size) * static_cast<double>(sizeof(uint32_t)) / 0.8;
  const double cluster_count = std::max(1.0, complete_hash_map_size / kL2CacheMaxUsable);
  return static_cast<int32_t>(std::min<size_t>(8, static_cast<size_t>(std::ceil(std::log2(cluster_count)))));
}

// Grid of a kernel that strides over `tiles` tiles: at most `blocks_per_sm` CTAs per SM, and at least one CTA.
static uint32_t tile_grid(const hyb_context* context, uint32_t tiles, int blocks_per_sm) {
  return std::max<uint32_t>(1, std::min<uint32_t>(tiles, context->sm_count * std::max(blocks_per_sm, 1)));
}

struct SideInfo {
  Table* table = nullptr;
  PosList* filter = nullptr;
  KeySource source{};
  uint32_t column_id = 0;
  int32_t data_type = 0;
  uint64_t positions = 0;
};

// A column's type on a join side (a table without chunks has none: its columns read as int32).
static int32_t side_column_type(const SideInfo& side, uint32_t column_id) {
  return side.table->chunk_count() ? side.table->column_types[column_id] : HYB_TYPE_INT32;
}

static int prepare_side(hyb_context* context, const hyb_join_side* side, SideInfo* out) {
  out->table = find_table(context, side->table);
  HYB_CHECK(out->table, HYB_ERR_NOT_FOUND, "unknown table handle");
  HYB_CHECK(side->column_id < out->table->column_count, HYB_ERR_INVALID, "join column out of range");
  out->column_id = side->column_id;
  out->data_type = side_column_type(*out, side->column_id);
  HYB_CHECK(out->data_type == HYB_TYPE_INT32 || out->data_type == HYB_TYPE_INT64, HYB_ERR_UNSUPPORTED,
            "JoinHash on the device supports int32/int64 key columns; other key types run on the CPU operator");
  HYB_TRY(sync_table_descriptors(context, out->table));
  KeySource& source = out->source;
  const uint32_t chunk_count = out->table->chunk_count();
  source.segments = out->table->d_segments + size_t{side->column_id} * chunk_count;
  source.chunk_row_start = reinterpret_cast<const unsigned long long*>(out->table->d_chunk_row_start);
  source.chunk_count = chunk_count;
  source.payload = out->table->position_payload;
  source.uniform_chunk_rows = (out->table->uniform_chunks && chunk_count) ? out->table->chunk_rows[0] : 0;
  if (source.uniform_chunk_rows) {
    // d = rows: shift = ceil(log2 d); magic = floor(2^32 * (2^shift - d) / d) + 1
    const uint64_t d = source.uniform_chunk_rows;
    uint32_t shift = 0;
    while ((uint64_t{1} << shift) < d) ++shift;
    source.uniform_shift = shift;
    source.uniform_magic = shift == 0 ? 0 : static_cast<uint32_t>(((uint64_t{1} << 32) * ((uint64_t{1} << shift) - d)) / d + 1);
  }
  if (side->filter) {
    out->filter = find_pos_list(context, side->filter);
    HYB_CHECK(out->filter, HYB_ERR_NOT_FOUND, "unknown filter handle");
    HYB_CHECK(out->filter->table == side->table, HYB_ERR_INVALID, "filter belongs to a different table");
    uint64_t count = 0;
    HYB_TRY(pos_list_total(context, out->filter, &count));
    out->positions = count;
    source.filter = out->filter->d_row_ids;
    source.null_key_zero = out->filter->ascending ? 0u : 1u;  // per-chunk scan lists are single-chunk PosLists
    source.tile_map = nullptr;
    source.tile_count = static_cast<uint32_t>((count + kJoinTileRows - 1) / kJoinTileRows);
  } else {
    out->positions = out->table->row_count();
    HYB_TRY(get_tile_map(context, out->table, kJoinTileRows, &source.tile_map, &source.tile_count));
  }
  source.position_count = out->positions;
  return HYB_OK;
}

// Key bounds of the (whole) key column of a join side, cached on the table. A filtered side uses the same bounds: they
// cover a superset of its keys.
static int column_key_bounds(hyb_context* context, const SideInfo& side, Table::KeyBounds* out, uint32_t* launches) {
  Table* table = side.table;
  const auto cached = table->key_bounds.find(side.column_id);
  if (cached != table->key_bounds.end()) {
    *out = cached->second;
    return HYB_OK;
  }
  Table::KeyBounds bounds{};
  if (table->row_count()) {
    KeySource whole = side.source;
    whole.filter = nullptr;
    HYB_TRY(get_tile_map(context, table, kJoinTileRows, &whole.tile_map, &whole.tile_count));
    whole.position_count = table->row_count();
    DeviceScratch scratch(context);
    long long* device_bounds = nullptr;
    HYB_TRY(scratch.alloc_array(6, &device_bounds));
    const long long initial[6] = {0x7FFFFFFFFFFFFFFFll, -0x7FFFFFFFFFFFFFFFll - 1, 0, -1ll, 0, 0};
    HYB_CUDA(cudaMemcpyAsync(device_bounds, initial, sizeof(initial), cudaMemcpyHostToDevice, context->stream));
    join_key_bounds_kernel<<<tile_grid(context, whole.tile_count, 8), kJoinThreads, 0, context->stream>>>(whole, device_bounds);
    HYB_CUDA(cudaGetLastError());
    ++*launches;
    long long host_bounds[6] = {};
    HYB_CUDA(cudaMemcpyAsync(host_bounds, device_bounds, sizeof(host_bounds), cudaMemcpyDeviceToHost, context->stream));
    HYB_CUDA(cudaStreamSynchronize(context->stream));
    bounds.has_values = host_bounds[2] != 0;
    bounds.min = host_bounds[0];
    bounds.max = host_bounds[1];
    bounds.strictly_increasing = bounds.has_values && host_bounds[5] == 0;
    if (bounds.has_values) {
      const unsigned long long varying = static_cast<unsigned long long>(host_bounds[3]) ^ static_cast<unsigned long long>(host_bounds[4]);
      while (bounds.constant_low_bits < 16 && !((varying >> bounds.constant_low_bits) & 1ull)) ++bounds.constant_low_bits;
    }
  }
  table->key_bounds.emplace(side.column_id, bounds);
  *out = bounds;
  return HYB_OK;
}

static int run_exclusive_scan(hyb_context* context, const uint32_t* in, unsigned long long* out, uint64_t count,
                              unsigned long long* total_out) {
  const uint32_t tile_count = static_cast<uint32_t>((count + kScanTile - 1) / kScanTile);
  if (tile_count == 0) {
    if (total_out) HYB_CUDA(cudaMemsetAsync(total_out, 0, sizeof(unsigned long long), context->stream));
    return HYB_OK;
  }
  DeviceScratch scratch(context);  // the look-back status words; the next user of the block is queued after the scan
  unsigned long long* status = nullptr;
  HYB_TRY(scratch.alloc_array(size_t{tile_count} + 1, &status));
  HYB_CUDA(cudaMemsetAsync(status, 0, sizeof(uint64_t) * (size_t{tile_count} + 1), context->stream));
  exclusive_scan_kernel<<<tile_grid(context, tile_count, 4), kJoinThreads, 0, context->stream>>>(
      in, out, count, status, reinterpret_cast<uint32_t*>(status + tile_count), total_out);
  HYB_CUDA(cudaGetLastError());
  return HYB_OK;
}

// The partition-count sequence of every probe pass and every partitioning: `count` launches the kernel that fills
// params.histogram ([partition][tile] over `tiles` tiles), the exclusive scan turns it into params.run_starts and *total,
// and join_partition_offsets_kernel writes the partition_count + 1 offsets. `write` runs between the scan and the offsets:
// a probe's write kernel. A partitioning writes once it has read the offsets and passes nothing.
template <typename Count, typename Write>
static int count_partitions(hyb_context* context, const ProbeParams& params, uint32_t tiles, unsigned long long* total,
                            unsigned long long* offsets, Count&& count, Write&& write) {
  HYB_TRY(count());
  // the kernels read run_starts through ProbeParams, hence const there; the scan is what fills it
  HYB_TRY(run_exclusive_scan(context, params.histogram, const_cast<unsigned long long*>(params.run_starts),
                             size_t{params.partition_count} * tiles, total));
  HYB_TRY(write());
  join_partition_offsets_kernel<<<(params.partition_count + 1 + 127) / 128, 128, 0, context->stream>>>(
      params.run_starts, total, params.partition_count, tiles, offsets);
  HYB_CUDA(cudaGetLastError());
  return HYB_OK;
}

static int no_write() { return HYB_OK; }

// ---- JoinHash stages (join_hash_locked) --------------------------------------------------------------------------------

// The table over the build side. Dense key domain (range of the build column <= 8x its rows): direct-address table, one
// uint32 per key value — or, when the build keys strictly increase with the build position, the 2-bits-per-key-value
// rank table. Otherwise: bucketised open addressing at load factor <= 0.5.
struct JoinTablePlan {
  uint32_t kind = HYB_JOIN_PATH_TABLE_HASH;  // HYB_JOIN_PATH_TABLE_*
  bool direct = false;                       // a direct-address table (shifted or not) or the rank table
  bool rank = false;
  bool wide = false;                         // int64 keys on either side
  uint32_t direct_shift = 0;                 // the build keys agree in these low bits (one rank's share of an exchange)
  unsigned long long key_span = 0, direct_span = 0;
  uint64_t bucket_count = 1, slot_count = 0;
  size_t slot_bytes = 0;
};

static int plan_join_table(const Table::KeyBounds& bounds, const SideInfo& build, const SideInfo& probe,
                           const ContextOptions& options, JoinTablePlan* out) {
  JoinTablePlan& plan = *out;
  plan.wide = build.data_type == HYB_TYPE_INT64 || probe.data_type == HYB_TYPE_INT64;
  plan.key_span = static_cast<unsigned long long>(bounds.max) - static_cast<unsigned long long>(bounds.min);
  // options.join_table overrides the choice (the parity tests run every case with every table kind).
  const bool force_hash = options.join_table == ContextOptions::kHash;
  const bool force_direct = options.join_table == ContextOptions::kDirect;
  plan.direct_shift = bounds.constant_low_bits;
  plan.direct_span = plan.key_span >> plan.direct_shift;
  plan.direct = bounds.has_values && build.positions > 0 && plan.direct_span < 0xFFFFFFE0ull && !force_hash &&
                (plan.direct_span < 8 * build.positions + 65'536 ||
                 (options.join_table != ContextOptions::kAuto && plan.direct_span < (1ull << 28)));
  // Rank table: positions must grow with the keys — the column does (cached with the key bounds) and a PosList on top of
  // it keeps the table order.
  plan.rank = plan.direct && !force_direct && bounds.strictly_increasing && plan.key_span < 0xFFFFFFE0ull &&
              (!build.filter || build.filter->ascending);
  while (plan.bucket_count * 2 < build.positions) plan.bucket_count <<= 1;  // >= positions / 2 buckets -> load factor <= 0.5
  HYB_CHECK(plan.bucket_count * 4 < 0xFFFFFFF0ull, HYB_ERR_UNSUPPORTED, "build side too large for 32-bit slot indexes");
  plan.slot_count = plan.rank ? (plan.key_span >> 5) + 1 : plan.direct ? plan.direct_span + 1 : plan.bucket_count * 4;
  plan.slot_bytes = plan.direct && !plan.rank ? sizeof(uint32_t) : sizeof(uint64_t);
  plan.kind = plan.rank     ? HYB_JOIN_PATH_TABLE_RANK
              : plan.direct ? (plan.direct_shift ? HYB_JOIN_PATH_TABLE_DIRECT_SHIFTED : HYB_JOIN_PATH_TABLE_DIRECT)
              : plan.wide   ? HYB_JOIN_PATH_TABLE_HASH_WIDE
                            : HYB_JOIN_PATH_TABLE_HASH;
  return HYB_OK;
}

// Allocates the table's slots, the control words ([0] duplicate keys, [1] NULL build keys, [2] output overflow, [4..5] the
// probe's total, u64) and an int64 hash table's keys, and queues the build kernels. Kernel time starts with them.
static int build_join_table(hyb_context* context, DeviceScratch& scratch, const JoinTablePlan& plan,
                            const Table::KeyBounds& bounds, const SideInfo& build, HashTable* out_table, uint32_t** out_control,
                            uint32_t* launches) {
  cudaStream_t stream = context->stream;
  void* slots = nullptr;
  uint32_t* control = nullptr;
  long long* wide_keys = nullptr;
  HYB_TRY(scratch.alloc(plan.slot_bytes * plan.slot_count, &slots));
  HYB_CUDA(cudaMemsetAsync(slots, plan.rank ? 0x00 : 0xFF, plan.slot_bytes * plan.slot_count, stream));
  HYB_TRY(scratch.alloc_array(16, &control));
  HYB_CUDA(cudaMemsetAsync(control, 0, 64, stream));
  if (plan.kind == HYB_JOIN_PATH_TABLE_HASH_WIDE) {
    // every position a slot can name is written by join_wide_keys_kernel: no initialisation needed
    HYB_TRY(scratch.alloc_array(std::max<uint64_t>(build.positions, 1), &wide_keys));
  }
  HashTable& table = *out_table;
  table = HashTable{};
  table.slots = static_cast<unsigned long long*>(slots);  // non-NULL also in direct / rank mode: "a table exists"
  table.bucket_mask = static_cast<uint32_t>(plan.bucket_count - 1);
  table.wide_keys = wide_keys;
  if (plan.rank) {
    table.rank_blocks = static_cast<uint2*>(slots);
    table.direct_min = bounds.min;
    table.direct_range = plan.key_span + 1;
  } else if (plan.direct) {
    table.direct = static_cast<uint32_t*>(slots);
    table.direct_min = bounds.min;
    table.direct_range = plan.direct_span + 1;
    table.direct_shift = plan.direct_shift;
  }
  *out_control = control;
  const uint32_t build_grid = tile_grid(context, build.source.tile_count, 8);
  timing_kernel_begin(context);
  if (build.source.tile_count) {
    BuildParams params{};
    params.source = build.source;
    params.table = table;
    params.wide_keys_out = wide_keys;
    params.flags = control;
    if (wide_keys) {
      join_wide_keys_kernel<<<build_grid, kJoinThreads, 0, stream>>>(params);
      HYB_CUDA(cudaGetLastError());
      ++*launches;
    }
    if (plan.rank) {
      join_build_rank_kernel<<<build_grid, kJoinThreads, 0, stream>>>(params);
    } else {
      join_build_kernel<<<build_grid, kJoinThreads, 0, stream>>>(params);
    }
    HYB_CUDA(cudaGetLastError());
    ++*launches;
  }
  return HYB_OK;
}

// Which probe kernels run.
struct ProbePlan {
  bool span = false;       // the 8192-row span kernels (else the 4096-row tile kernels)
  uint32_t tile_fast = 0;  // ProbeParams::fast of the tile kernels, whose lean path knows the direct table only
};

static ProbePlan plan_probe(const JoinTablePlan& table, const SideInfo& probe, int32_t mode, bool secondary,
                            const ContextOptions& options) {
  // Lean path of the case that dominates (Inner, dense unique build side): 1 = int32 keys on both sides, 2 = int64 probe
  // keys against a (possibly shifted) direct table. Secondary predicates take the generic loop only.
  const uint32_t fast =
      (mode == HYB_JOIN_INNER && table.direct && !secondary)
          ? ((table.direct_shift == 0 && !table.wide) ? 1u : ((!table.rank && probe.data_type == HYB_TYPE_INT64) ? 2u : 0u))
          : 0u;
  ProbePlan plan;
  plan.tile_fast = table.rank ? 0u : fast;
  // Span kernels: every probe segment must decode with a lean codec (plain values or FrameOfReference in a
  // FixedWidthIntegerVector, no NULL vector); anything else keeps the tile kernels, which pick a decoder per tile.
  plan.span = options.join_span && fast != 0 && !probe.filter && probe.source.tile_count > 0;
  const Table* source = probe.table;
  for (uint32_t chunk = 0; chunk < source->chunk_count() && plan.span; ++chunk) {
    const DevSegment& segment = source->segments[size_t{chunk} * source->column_count + probe.column_id];
    const bool plain64 = segment.encoding == HYB_ENC_UNENCODED && segment.data_type == HYB_TYPE_INT64;
    plan.span = !segment.nulls && segment.encoding != HYB_ENC_DICTIONARY &&
                !(segment.encoding == HYB_ENC_FRAME_OF_REFERENCE && segment.vector_type == HYB_VEC_BITPACKED) &&
                (fast == 2) == plain64;
  }
  return plan;
}

// Compulsory traffic of one column of a join side (SURVEY.md §8d): the column once, or a PosList's rows of it.
static uint64_t join_column_bytes(const SideInfo& side, uint32_t column_id) {
  if (side.filter) return side.positions * data_type_size(side_column_type(side, column_id));
  uint64_t bytes = 0;
  for (uint32_t chunk = 0; chunk < side.table->chunk_count(); ++chunk) {
    const auto& segment = side.table->segments[size_t{chunk} * side.table->column_count + column_id];
    bytes += segment.encoding == HYB_ENC_UNENCODED ? data_type_size(segment.data_type) * segment.row_count
                                                   : vector_bytes(segment.vector_type, segment.bit_width, segment.row_count);
    if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) {
      bytes += sizeof(int32_t) * ((segment.row_count + HYB_FOR_BLOCK_SIZE - 1) / HYB_FOR_BLOCK_SIZE);
    }
  }
  return bytes;
}

// ... of one side's keys: the key column once, or a PosList's RowIDs and keys.
static uint64_t join_key_bytes(const SideInfo& side) {
  return join_column_bytes(side, side.column_id) + (side.filter ? side.positions * sizeof(hyb_row_id) : 0);
}

// The secondary predicates of a call (hyb_join_hash_predicates): checked, typed and copied to the device.
struct SecondaryPlan {
  SecondaryPredicates device{};     // count == 0: none
  uint64_t algorithmic_bytes = 0;   // every distinct secondary column of both sides once
};

static int prepare_secondary(hyb_context* context, DeviceScratch& scratch, const SideInfo& build, const SideInfo& probe,
                             const hyb_join_predicate* predicates, uint32_t count, SecondaryPlan* out) {
  if (count == 0) return HYB_OK;
  HYB_CHECK(!build.table->position_payload && !probe.table->position_payload, HYB_ERR_UNSUPPORTED,
            "secondary join predicates read the columns of the rows they join; received exchange tuples stand for "
            "another table's rows");
  std::vector<JoinPredicate> host(count);
  std::vector<uint32_t> build_columns, probe_columns;
  for (uint32_t i = 0; i < count; ++i) {
    const hyb_join_predicate& predicate = predicates[i];
    HYB_CHECK(predicate.reserved == 0, HYB_ERR_INVALID, "hyb_join_predicate.reserved must be 0");
    HYB_CHECK(predicate.build_column_id < build.table->column_count && predicate.probe_column_id < probe.table->column_count,
              HYB_ERR_INVALID, "secondary join predicate column out of range");
    HYB_CHECK(predicate.condition >= HYB_PRED_EQUALS && predicate.condition <= HYB_PRED_GREATER_THAN_EQUALS, HYB_ERR_INVALID,
              "secondary join predicates take =, !=, <, <=, >, >= (condition " + std::to_string(predicate.condition) + ")");
    const int32_t build_type = side_column_type(build, predicate.build_column_id);
    const int32_t probe_type = side_column_type(probe, predicate.probe_column_id);
    const bool strings = build_type == HYB_TYPE_STRING;
    // multi_predicate_join_evaluator.cpp: Fail("Types of columns cannot be compared")
    HYB_CHECK(strings == (probe_type == HYB_TYPE_STRING), HYB_ERR_INVALID, "Types of columns cannot be compared");
    HYB_CHECK(!strings, HYB_ERR_UNSUPPORTED,
              "string secondary join predicates need a dictionary translation per chunk pair; they run on the CPU operator");
    host[i].build = build.table->d_segments + size_t{predicate.build_column_id} * build.table->chunk_count();
    host[i].probe = probe.table->d_segments + size_t{predicate.probe_column_id} * probe.table->chunk_count();
    host[i].condition = predicate.condition;
    host[i].compare = pair_compare(build_type, probe_type);
    const auto count_column = [&](std::vector<uint32_t>& seen, const SideInfo& side, uint32_t column) {
      if (std::find(seen.begin(), seen.end(), column) != seen.end()) return;
      seen.push_back(column);
      out->algorithmic_bytes += join_column_bytes(side, column);
    };
    count_column(build_columns, build, predicate.build_column_id);
    count_column(probe_columns, probe, predicate.probe_column_id);
  }
  JoinPredicate* device = nullptr;
  HYB_TRY(scratch.alloc_array(count, &device));
  // pageable source: the copy is staged before cudaMemcpyAsync returns
  HYB_CUDA(cudaMemcpyAsync(device, host.data(), sizeof(JoinPredicate) * count, cudaMemcpyHostToDevice, context->stream));
  out->device = SecondaryPredicates{device, count};
  return HYB_OK;
}

// What every probe pass of one join shares.
struct ProbeSetup {
  ProbeParams params{};  // the tile kernels' parameters; each pass fills in its output blocks
  void (*count_kernel)(const ProbeParams) = nullptr;
  void (*write_kernel)(const ProbeParams) = nullptr;
  // secondary predicates: these tile kernels run instead, with `secondary` as their second argument
  SecondaryPredicates secondary{};
  void (*secondary_count_kernel)(const ProbeParams, const SecondaryPredicates) = nullptr;
  void (*secondary_write_kernel)(const ProbeParams, const SecondaryPredicates) = nullptr;
  uint32_t count_grid = 1, write_grid = 1;
  KeySource span_source{};  // the span kernels: the probe side in kSpanRows-row spans
  bool rank = false;        // span kernel variants
  bool ballot = false;
  unsigned long long* total = nullptr;  // output rows of the pass (device)
};

static int prepare_probe(hyb_context* context, DeviceScratch& scratch, const JoinTablePlan& plan, const ProbePlan& probe_plan,
                         const SecondaryPlan& secondary, const SideInfo& build, const SideInfo& probe, int32_t mode,
                         uint32_t partition_count, const HashTable& table, uint32_t* control, ProbeSetup* out) {
  out->span_source = probe.source;
  if (probe_plan.span) HYB_TRY(get_tile_map(context, probe.table, kSpanRows, &out->span_source.tile_map, &out->span_source.tile_count));
  // Hash tables: the count kernel keeps match + partition per probe slot so that the write kernel does not repeat the
  // random table accesses. Direct-address / rank tables are probed sequentially or from L2; looking up twice is cheaper
  // than 10 bytes/row.
  const bool store_matches = !plan.direct;
  out->count_kernel = store_matches ? join_probe_count_kernel<true> : join_probe_count_kernel<false>;
  out->write_kernel = store_matches ? join_probe_write_kernel<true> : join_probe_write_kernel<false>;
  int count_blocks = 1, write_blocks = 1;
  out->secondary = secondary.device;
  if (secondary.device.count) {
    out->secondary_count_kernel = store_matches ? join_probe_secondary_count_kernel<true> : join_probe_secondary_count_kernel<false>;
    out->secondary_write_kernel = store_matches ? join_probe_secondary_write_kernel<true> : join_probe_secondary_write_kernel<false>;
    HYB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&count_blocks, out->secondary_count_kernel, kJoinThreads, 0));
    HYB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&write_blocks, out->secondary_write_kernel, kJoinThreads, 0));
  } else {
    HYB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&count_blocks, out->count_kernel, kJoinThreads, 0));
    HYB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&write_blocks, out->write_kernel, kJoinThreads, 0));
  }
  const uint32_t probe_tiles = probe.source.tile_count;
  out->count_grid = tile_grid(context, probe_tiles, count_blocks);
  out->write_grid = tile_grid(context, probe_tiles, write_blocks);
  out->rank = plan.rank;
  out->ballot = context->options.join_ballot_rank;
  out->total = reinterpret_cast<unsigned long long*>(control + 4);
  if (!probe_tiles) return HYB_OK;
  ProbeParams& params = out->params;
  const size_t probe_slots = size_t{probe_tiles} * kJoinTileRows;
  if (store_matches) {
    HYB_TRY(scratch.alloc_array(probe_slots, &params.matches));
    HYB_TRY(scratch.alloc_array(probe_slots, &params.partitions));
  }
  // sized for the tile kernels as well: a duplicate build key sends a span-path call back to them
  unsigned long long* run_starts = nullptr;
  HYB_TRY(scratch.alloc_array(size_t{partition_count} * probe_tiles, &params.histogram));
  HYB_TRY(scratch.alloc_array(size_t{partition_count} * probe_tiles, &run_starts));
  params.probe = probe.source;
  params.build = build.source;
  params.table = table;
  if (build.source.tile_count == 0) params.table.slots = nullptr;
  params.mode = mode;
  params.partition_mask = partition_count - 1;
  params.partition_count = partition_count;
  params.unique_build = 1;  // optimistic: a flag raised by the build kernel sends us to rerun_with_duplicates
  params.fast = probe_plan.tile_fast;
  params.build_is_empty = build.positions == 0;
  params.flags = control;
  params.run_starts = run_starts;
  params.overflow = control + 2;
  return HYB_OK;
}

// One pass of the tile kernels (count or write) over setup.params: the secondary predicates' variant when there are any.
static int launch_tile_pass(hyb_context* context, const ProbeSetup& setup, bool write) {
  const uint32_t grid = write ? setup.write_grid : setup.count_grid;
  if (setup.secondary.count) {
    (write ? setup.secondary_write_kernel : setup.secondary_count_kernel)<<<grid, kJoinThreads, 0, context->stream>>>(
        setup.params, setup.secondary);
  } else {
    (write ? setup.write_kernel : setup.count_kernel)<<<grid, kJoinThreads, 0, context->stream>>>(setup.params);
  }
  HYB_CUDA(cudaGetLastError());
  return HYB_OK;
}

// The result's output blocks for `capacity` rows (the previous pass's blocks go back to the cache): the result owns them.
static int allocate_join_outputs(hyb_context* context, JoinResult* result, uint64_t capacity) {
  device_free(context, result->d_probe);
  device_free(context, result->d_build);
  result->d_probe = nullptr;
  result->d_build = nullptr;
  void* out_probe = nullptr;
  void* out_build = nullptr;
  HYB_TRY(device_alloc(context, sizeof(hyb_row_id) * std::max<uint64_t>(capacity, 1), &out_probe));
  result->d_probe = static_cast<hyb_row_id*>(out_probe);
  const int32_t mode = result->mode;
  if (mode != HYB_JOIN_SEMI && mode != HYB_JOIN_ANTI_NULL_AS_TRUE && mode != HYB_JOIN_ANTI_NULL_AS_FALSE) {
    HYB_TRY(device_alloc(context, sizeof(hyb_row_id) * std::max<uint64_t>(capacity, 1), &out_build));
    result->d_build = static_cast<hyb_row_id*>(out_build);
  }
  result->capacity = capacity;
  return HYB_OK;
}

// One probe pass: count -> scan -> output blocks of `capacity` rows -> write -> partition offsets, all queued without a
// host round trip. `span`: the span kernels over setup.span_source; otherwise the tile kernels.
static int run_probe_pass(hyb_context* context, DeviceScratch& scratch, ProbeSetup& setup, bool span, uint64_t capacity,
                          JoinResult* result, uint32_t* launches) {
  cudaStream_t stream = context->stream;
  ProbeParams& params = setup.params;
  ProbeParams span_params = params;
  span_params.probe = setup.span_source;
  const uint32_t tiles = span ? setup.span_source.tile_count : params.probe.tile_count;
  const size_t counter_bytes = sizeof(uint32_t) * kSpanWarps * params.partition_count;
  const size_t write_bytes = sizeof(uint2) * kSpanRows + counter_bytes;
  const auto count_spans = setup.rank ? join_span_count_kernel<kTableRank> : join_span_count_kernel<kTableDirect>;
  const auto write_spans =
      setup.rank ? (setup.ballot ? join_span_write_kernel<kTableRank, true> : join_span_write_kernel<kTableRank, false>)
                 : (setup.ballot ? join_span_write_kernel<kTableDirect, true> : join_span_write_kernel<kTableDirect, false>);
  uint16_t* fine_counts = nullptr;
  if (span) {
    HYB_CUDA(cudaFuncSetAttribute(write_spans, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(write_bytes)));
    HYB_TRY(scratch.alloc_array(size_t{tiles} * kSpanWarps * params.partition_count, &fine_counts));
  }
  const auto count = [&]() -> int {
    if (span) {
      count_spans<<<tiles, kSpanThreads, counter_bytes, stream>>>(span_params, fine_counts);
    } else {
      HYB_TRY(launch_tile_pass(context, setup, false));
    }
    HYB_CUDA(cudaGetLastError());
    return HYB_OK;
  };
  const auto write = [&]() -> int {
    HYB_TRY(allocate_join_outputs(context, result, capacity));
    params.out_probe = span_params.out_probe = result->d_probe;
    params.out_build = span_params.out_build = result->d_build;
    params.out_capacity = span_params.out_capacity = capacity;
    if (span) {
      write_spans<<<tiles, kSpanThreads, write_bytes, stream>>>(span_params, fine_counts);
    } else {
      HYB_TRY(launch_tile_pass(context, setup, true));
    }
    HYB_CUDA(cudaGetLastError());
    return HYB_OK;
  };
  HYB_TRY(count_partitions(context, params, tiles, setup.total,
                           reinterpret_cast<unsigned long long*>(result->d_partition_offsets), count, write));
  *launches += 4;
  return HYB_OK;
}

// Duplicate build keys: build the position lists (PosHashTable::finalize, join_hash_steps.hpp:147-175), size the output
// exactly (count + scan, read the total) and probe again with the tile kernels: the span kernels are for unique build sides.
static int rerun_with_duplicates(hyb_context* context, DeviceScratch& scratch, const JoinTablePlan& plan, const SideInfo& build,
                                 const HashTable& table, ProbeSetup& setup, JoinResult* result, uint32_t* launches) {
  cudaStream_t stream = context->stream;
  const uint64_t slot_count = plan.slot_count;
  const uint32_t build_grid = tile_grid(context, build.source.tile_count, 8);
  uint32_t* dup_counts = nullptr;  // counts | cursors
  unsigned long long* dup_offsets = nullptr;
  uint32_t* dup_positions = nullptr;
  HYB_TRY(scratch.alloc_array(slot_count * 2, &dup_counts));
  HYB_CUDA(cudaMemsetAsync(dup_counts, 0, sizeof(uint32_t) * slot_count * 2, stream));
  HYB_TRY(scratch.alloc_array(slot_count, &dup_offsets));
  HYB_TRY(scratch.alloc_array(std::max<uint64_t>(build.positions, 1), &dup_positions));
  timing_kernel_begin(context);
  join_count_duplicates_kernel<<<build_grid, kJoinThreads, 0, stream>>>(build.source, table, dup_counts);
  HYB_CUDA(cudaGetLastError());
  HYB_TRY(run_exclusive_scan(context, dup_counts, dup_offsets, slot_count, nullptr));
  join_fill_positions_kernel<<<build_grid, kJoinThreads, 0, stream>>>(build.source, table, dup_offsets, dup_counts + slot_count,
                                                                      dup_positions);
  HYB_CUDA(cudaGetLastError());
  join_sort_positions_kernel<<<static_cast<uint32_t>((slot_count + 255) / 256), 256, 0, stream>>>(
      dup_counts, dup_offsets, static_cast<uint32_t>(slot_count), dup_positions);
  HYB_CUDA(cudaGetLastError());
  *launches += 4;
  ProbeParams& params = setup.params;
  params.unique_build = 0;
  params.dup_counts = dup_counts;
  params.dup_offsets = dup_offsets;
  params.dup_positions = dup_positions;
  HYB_TRY(launch_tile_pass(context, setup, false));
  HYB_TRY(run_exclusive_scan(context, params.histogram, const_cast<unsigned long long*>(params.run_starts),
                             size_t{params.partition_count} * params.probe.tile_count, setup.total));
  *launches += 2;
  uint64_t total = 0;
  HYB_CUDA(cudaMemcpyAsync(&total, setup.total, sizeof(uint64_t), cudaMemcpyDeviceToHost, stream));
  HYB_CUDA(cudaStreamSynchronize(stream));
  HYB_CUDA(cudaMemsetAsync(params.overflow, 0, sizeof(uint32_t), stream));
  HYB_TRY(run_probe_pass(context, scratch, setup, false, total, result, launches));
  timing_kernel_end(context);
  HYB_CUDA(cudaStreamSynchronize(stream));
  return HYB_OK;
}

// The hyb_join_path code of a join: its table kind, the probe kernels (when there were probe rows) and the rerun.
static uint32_t join_path_code(const JoinTablePlan& table, const ProbePlan& probe, bool probed, bool rerun, bool secondary) {
  uint32_t path = table.kind;
  if (probed) path |= probe.span ? HYB_JOIN_PATH_PROBE_SPAN : probe.tile_fast ? HYB_JOIN_PATH_PROBE_TILE_LEAN : HYB_JOIN_PATH_PROBE_TILE;
  if (rerun) path |= HYB_JOIN_PATH_RERUN;
  if (secondary) path |= HYB_JOIN_PATH_SECONDARY;
  return path;
}

// The count kernel of a kModePartition split: the probe's count kernel without a table or stored matches.
static int launch_partition_count(hyb_context* context, const ProbeParams& params) {
  int blocks = 1;
  HYB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, join_probe_count_kernel<false>, kJoinThreads, 0));
  join_probe_count_kernel<false><<<tile_grid(context, params.probe.tile_count, blocks), kJoinThreads, 0, context->stream>>>(params);
  HYB_CUDA(cudaGetLastError());
  return HYB_OK;
}

// ProbeParams of the stable split of a side's {key, RowID} tuples by key & (partition_count - 1) (kModePartition): the
// probe machinery without a table. `control`: 16 zeroed words, the scan's total at [4..5].
static ProbeParams partition_params(const SideInfo& side, uint32_t partition_count, uint32_t chunk_id_base, uint32_t* control,
                                    uint32_t* histogram, const unsigned long long* run_starts) {
  ProbeParams params{};
  params.probe = side.source;
  params.build = side.source;
  params.mode = kModePartition;
  params.partition_mask = partition_count - 1;
  params.partition_count = partition_count;
  params.unique_build = 1;
  params.flags = control;
  params.histogram = histogram;
  params.run_starts = run_starts;
  params.overflow = control + 2;
  params.chunk_id_base = chunk_id_base;
  return params;
}

}  // namespace hyb

using namespace hyb;

// hyb_join_hash / hyb_join_hash_predicates with context->mutex held (hyb_join_hash_distributed joins the received tuples
// through it).
static int join_hash_locked(hyb_context* context, const hyb_join_side* build_side, const hyb_join_side* probe_side, int32_t mode,
                            int32_t radix_bits, hyb_join_result_t* out_result, uint32_t build_chunk_base = 0,
                            uint32_t probe_chunk_base = 0, const hyb_join_predicate* predicates = nullptr,
                            uint32_t predicate_count = 0) {
  SideInfo build, probe;
  HYB_TRY(prepare_side(context, build_side, &build));
  HYB_TRY(prepare_side(context, probe_side, &probe));
  build.source.chunk_id_base = build_chunk_base;  // emitted RowIDs only: keys are still read from this table's chunks
  probe.source.chunk_id_base = probe_chunk_base;
  HYB_CHECK(build.positions < 0xFFFFFFF0ull && probe.positions < 0xFFFFFFF0ull, HYB_ERR_UNSUPPORTED,
            "more than 2^32 - 16 rows per join side");
  if (radix_bits < 0) radix_bits = calculate_radix_bits(build.positions);
  HYB_CHECK(radix_bits <= 8, HYB_ERR_INVALID, "radix_bits must be <= 8 (join_hash.cpp:113)");
  const uint32_t partition_count = 1u << radix_bits;
  const bool semi_or_anti = mode == HYB_JOIN_SEMI || mode == HYB_JOIN_ANTI_NULL_AS_TRUE || mode == HYB_JOIN_ANTI_NULL_AS_FALSE;
  cudaStream_t stream = context->stream;
  uint32_t launches = 0;
  DeviceScratch scratch(context);  // every scratch block of this call goes back to the cache on every exit path
  SecondaryPlan secondary;
  HYB_TRY(prepare_secondary(context, scratch, build, probe, predicates, predicate_count, &secondary));
  timing_begin(context);

  Table::KeyBounds bounds{};
  HYB_TRY(column_key_bounds(context, build, &bounds, &launches));
  JoinTablePlan table_plan;
  HYB_TRY(plan_join_table(bounds, build, probe, context->options, &table_plan));
  HashTable table{};
  uint32_t* control = nullptr;
  HYB_TRY(build_join_table(context, scratch, table_plan, bounds, build, &table, &control, &launches));

  auto result = std::make_unique<JoinResult>();  // owns its output blocks and partition offsets
  result->mode = mode;
  result->build_table = build_side->table;
  result->probe_table = probe_side->table;
  result->radix_bits = radix_bits;
  result->partition_count = partition_count;
  result->secondary = secondary.device.count != 0;
  result->stream = stream;
  result->owner = context;
  void* partition_offsets = nullptr;
  HYB_TRY(device_alloc(context, sizeof(uint64_t) * (size_t{partition_count} + 2), &partition_offsets));
  result->d_partition_offsets = static_cast<uint64_t*>(partition_offsets);
  HYB_CUDA(cudaMemsetAsync(partition_offsets, 0, sizeof(uint64_t) * (size_t{partition_count} + 2), stream));

  const ProbePlan probe_plan = plan_probe(table_plan, probe, mode, secondary.device.count != 0, context->options);
  ProbeSetup setup;
  HYB_TRY(prepare_probe(context, scratch, table_plan, probe_plan, secondary, build, probe, mode, partition_count, table, control,
                        &setup));
  const bool probed = probe.source.tile_count != 0;
  // With a unique build side every probe row emits at most one output row: probe.positions rows always suffice.
  if (probed) HYB_TRY(run_probe_pass(context, scratch, setup, probe_plan.span, probe.positions, result.get(), &launches));
  timing_kernel_end(context);
  uint32_t host_control[8] = {};
  HYB_CUDA(cudaMemcpyAsync(host_control, control, sizeof(host_control), cudaMemcpyDeviceToHost, stream));
  HYB_CUDA(cudaStreamSynchronize(stream));  // the only host round trip of the operator (unique build side)
  // Semi / Anti joins need every build row of a key only when its candidates are evaluated
  const bool rerun = host_control[0] != 0 && (!semi_or_anti || secondary.device.count) && probed;
  if (rerun) HYB_TRY(rerun_with_duplicates(context, scratch, table_plan, build, table, setup, result.get(), &launches));

  timing_end(context, launches, join_key_bytes(build) + join_key_bytes(probe) + secondary.algorithmic_bytes, probe.positions, 0);
  timing_output_count(context, result->d_partition_offsets + partition_count, semi_or_anti ? 8 : 16);
  context->timing.stats.path = join_path_code(table_plan, probe_plan, probed, rerun, secondary.device.count != 0);
  const auto handle = context->next_handle++;
  context->join_results.emplace(handle, std::move(result));
  *out_result = handle;
  return HYB_OK;
}


extern "C" {

int hyb_join_hash(hyb_context* context, const hyb_join_side* build_side, const hyb_join_side* probe_side, int32_t mode,
                  int32_t radix_bits, hyb_join_result_t* out_result) {
  HYB_CHECK(context && build_side && probe_side && out_result, HYB_ERR_INVALID, "NULL argument");
  *out_result = 0;
  HYB_CHECK(mode == HYB_JOIN_INNER || mode == HYB_JOIN_LEFT || mode == HYB_JOIN_RIGHT || mode == HYB_JOIN_SEMI ||
                mode == HYB_JOIN_ANTI_NULL_AS_TRUE || mode == HYB_JOIN_ANTI_NULL_AS_FALSE,
            HYB_ERR_UNSUPPORTED, "JoinMode not supported by JoinHash");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  return join_hash_locked(context, build_side, probe_side, mode, radix_bits, out_result);
}

int hyb_join_hash_predicates(hyb_context* context, const hyb_join_side* build_side, const hyb_join_side* probe_side, int32_t mode,
                             int32_t radix_bits, const hyb_join_predicate* predicates, uint32_t predicate_count,
                             hyb_join_result_t* out_result) {
  HYB_CHECK(context && build_side && probe_side && out_result && (predicates || predicate_count == 0), HYB_ERR_INVALID,
            "NULL argument");
  *out_result = 0;
  HYB_CHECK(mode == HYB_JOIN_INNER || mode == HYB_JOIN_LEFT || mode == HYB_JOIN_RIGHT || mode == HYB_JOIN_SEMI ||
                mode == HYB_JOIN_ANTI_NULL_AS_TRUE || mode == HYB_JOIN_ANTI_NULL_AS_FALSE,
            HYB_ERR_UNSUPPORTED, "JoinMode not supported by JoinHash");
  HYB_CHECK(predicate_count <= HYB_MAX_JOIN_PREDICATES, HYB_ERR_UNSUPPORTED,
            "more than " + std::to_string(HYB_MAX_JOIN_PREDICATES) + " secondary join predicates");
  // JoinHash::supports (join_hash.cpp:36-44): no AntiNullAsTrue with secondary predicates
  HYB_CHECK(predicate_count == 0 || mode != HYB_JOIN_ANTI_NULL_AS_TRUE, HYB_ERR_UNSUPPORTED,
            "AntiNullAsTrue joins with secondary predicates are not supported by JoinHash");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  return join_hash_locked(context, build_side, probe_side, mode, radix_bits, out_result, 0, 0, predicates, predicate_count);
}

int hyb_join_side_positions(hyb_context* context, const hyb_join_side* side, uint64_t* out_positions) {
  HYB_CHECK(context && side && out_positions, HYB_ERR_INVALID, "NULL argument");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  SideInfo info;
  HYB_TRY(prepare_side(context, side, &info));
  *out_positions = info.positions;
  return HYB_OK;
}

int hyb_join_materialize(hyb_context* context, const hyb_join_side* side, uint32_t chunk_id_base, void* out_keys_device,
                         void* out_row_ids_device) {
  HYB_CHECK(context && side, HYB_ERR_INVALID, "NULL argument");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  SideInfo info;
  HYB_TRY(prepare_side(context, side, &info));
  HYB_CHECK(info.positions == 0 || (out_keys_device && out_row_ids_device), HYB_ERR_INVALID, "output buffers are NULL");
  timing_begin(context);
  timing_kernel_begin(context);
  if (info.source.tile_count) {
    join_materialize_kernel<<<tile_grid(context, info.source.tile_count, 8), kJoinThreads, 0, context->stream>>>(
        info.source, chunk_id_base, static_cast<long long*>(out_keys_device), static_cast<long long*>(out_row_ids_device));
    HYB_CUDA(cudaGetLastError());
  }
  timing_kernel_end(context);
  timing_end(context, 1, info.positions * 16, info.positions, info.positions);
  HYB_CUDA(cudaStreamSynchronize(context->stream));  // the caller hands the buffers to NCCL on another stream
  return HYB_OK;
}

// Shared by hyb_join_partition (local output buffers) and hyb_join_partition_push (peer destinations chosen by `exchange`
// after the counts are known).
static int partition_side(hyb_context* context, const hyb_join_side* side, uint32_t partition_count, uint32_t chunk_id_base,
                          void* out_keys_device, void* out_row_ids_device, uint64_t* out_partition_offsets,
                          hyb_exchange_fn exchange, void* user) {
  HYB_CHECK(partition_count >= 1 && partition_count <= kMaxPartitions && (partition_count & (partition_count - 1)) == 0,
            HYB_ERR_INVALID, "partition_count must be a power of two <= 256");
  HYB_CHECK(!exchange || partition_count <= kMaxPeers, HYB_ERR_INVALID, "at most 16 peers");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  SideInfo info;
  HYB_TRY(prepare_side(context, side, &info));
  HYB_CHECK(exchange || info.positions == 0 || (out_keys_device && out_row_ids_device), HYB_ERR_INVALID, "output buffers are NULL");
  HYB_CHECK(info.positions < 0xFFFFFFF0ull, HYB_ERR_UNSUPPORTED, "more than 2^32 - 16 rows per join side");
  cudaStream_t stream = context->stream;
  std::vector<uint64_t> offsets_host(size_t{partition_count} + 1, 0);
  timing_begin(context);
  const uint32_t tiles = info.source.tile_count;
  // Same machinery as the probe: count per (partition, tile) -> exclusive scan -> ranked write. No table, no lookups.
  const size_t histogram_entries = size_t{partition_count} * std::max<uint32_t>(tiles, 1);
  DeviceScratch scratch(context);
  uint32_t* histogram = nullptr;
  unsigned long long* run_starts = nullptr;
  uint32_t* control = nullptr;
  unsigned long long* offsets = nullptr;
  HYB_TRY(scratch.alloc_array(histogram_entries, &histogram));
  HYB_TRY(scratch.alloc_array(histogram_entries, &run_starts));
  HYB_TRY(scratch.alloc_array(16, &control));
  HYB_TRY(scratch.alloc_array(size_t{partition_count} + 1, &offsets));
  HYB_CUDA(cudaMemsetAsync(control, 0, 64, stream));
  ProbeParams params = partition_params(info, partition_count, chunk_id_base, control, histogram, run_starts);
  params.out_build = static_cast<hyb_row_id*>(out_keys_device);
  params.out_probe = static_cast<hyb_row_id*>(out_row_ids_device);
  params.out_capacity = info.positions;
  int write_blocks = 1;
  HYB_CUDA(cudaFuncSetAttribute(join_partition_write_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(kPartitionStageBytes)));
  HYB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&write_blocks, join_partition_write_kernel, kJoinThreads, kPartitionStageBytes));
  uint32_t launches = 0;
  timing_kernel_begin(context);
  if (tiles) {
    HYB_TRY(count_partitions(context, params, tiles, reinterpret_cast<unsigned long long*>(control + 4), offsets,
                             [&] { return launch_partition_count(context, params); }, no_write));
    launches += 3;
    if (exchange) {
      // The destinations depend on what every other rank sends: hand the counts to the host layer (one small
      // all-gather) and get the peer pointers this rank's groups start at.
      timing_kernel_end(context);
      HYB_CUDA(cudaMemcpyAsync(offsets_host.data(), offsets, sizeof(uint64_t) * offsets_host.size(), cudaMemcpyDeviceToHost, stream));
      HYB_CUDA(cudaStreamSynchronize(stream));
    }
  }
  if (exchange) {
    std::vector<uint64_t> counts(partition_count);
    for (uint32_t p = 0; p < partition_count; ++p) counts[p] = offsets_host[p + 1] - offsets_host[p];
    void* dest_keys[kMaxPeers] = {};
    void* dest_rows[kMaxPeers] = {};
    const int status = exchange(user, counts.data(), dest_keys, dest_rows);
    HYB_CHECK(status == 0, HYB_ERR_INVALID, "the exchange callback failed");
    for (uint32_t p = 0; p < partition_count; ++p) {
      HYB_CHECK(counts[p] == 0 || (dest_keys[p] && dest_rows[p]), HYB_ERR_INVALID, "the exchange callback left a destination NULL");
      params.peer_keys[p] = static_cast<long long*>(dest_keys[p]);
      params.peer_rows[p] = static_cast<long long*>(dest_rows[p]);
    }
    params.push_to_peers = 1;
    params.out_capacity = ~0ull;
    if (tiles) timing_kernel_begin(context);
  }
  if (tiles) {
    join_partition_write_kernel<<<tile_grid(context, tiles, write_blocks), kJoinThreads, kPartitionStageBytes, stream>>>(params);
    HYB_CUDA(cudaGetLastError());
    ++launches;
    timing_kernel_end(context);
    if (!exchange) {
      HYB_CUDA(cudaMemcpyAsync(offsets_host.data(), offsets, sizeof(uint64_t) * offsets_host.size(), cudaMemcpyDeviceToHost, stream));
    }
  } else if (!exchange) {
    timing_kernel_end(context);
  }
  timing_end(context, launches, info.positions * 16, info.positions, 0);
  HYB_CUDA(cudaStreamSynchronize(stream));  // local: the caller hands the buffers to NCCL; push: stores to peers are done
  if (out_partition_offsets) {
    for (uint32_t p = 0; p <= partition_count; ++p) out_partition_offsets[p] = offsets_host[p];
  }
  return HYB_OK;
}

int hyb_join_partition(hyb_context* context, const hyb_join_side* side, uint32_t partition_count, uint32_t chunk_id_base,
                       void* out_keys_device, void* out_row_ids_device, uint64_t* out_partition_offsets) {
  HYB_CHECK(context && side && out_partition_offsets, HYB_ERR_INVALID, "NULL argument");
  return partition_side(context, side, partition_count, chunk_id_base, out_keys_device, out_row_ids_device,
                        out_partition_offsets, nullptr, nullptr);
}

int hyb_join_partition_push(hyb_context* context, const hyb_join_side* side, uint32_t world_size, uint32_t chunk_id_base,
                            hyb_exchange_fn exchange, void* user) {
  HYB_CHECK(context && side && exchange, HYB_ERR_INVALID, "NULL argument");
  return partition_side(context, side, world_size, chunk_id_base, nullptr, nullptr, nullptr, exchange, user);
}

}  // extern "C" (reopened below)

// ---------------------------------------------------------------------------------------------------------------------
// Distributed Inner JoinHash over a peer group (peer.hpp). All of it is queued on the context stream; the host waits once,
// for the world x world count matrix.
// ---------------------------------------------------------------------------------------------------------------------
namespace hyb {

// Writes this rank's per-destination tuple counts of both sides and its build-key statistics into EVERY rank's control
// block (row `rank` of the count matrix), then — behind a system-scope fence — raises its count flag there.
__global__ void peer_publish_counts_kernel(PeerControl* const* controls, uint32_t rank, uint32_t world, unsigned long long epoch,
                                           const unsigned long long* build_offsets, const unsigned long long* probe_offsets,
                                           long long key_min, long long key_max, long long key_count) {
  const uint32_t peer = threadIdx.x / 32, lane = threadIdx.x & 31;
  if (peer < world) {
    PeerControl* control = controls[peer];
    if (lane < world) {
      control->counts[0][rank][lane] = build_offsets ? build_offsets[lane + 1] - build_offsets[lane] : 0ull;
      control->counts[1][rank][lane] = probe_offsets ? probe_offsets[lane + 1] - probe_offsets[lane] : 0ull;
    }
    if (lane == 0) {
      control->key_info[rank][0] = key_min;
      control->key_info[rank][1] = key_max;
      control->key_info[rank][2] = key_count;
    }
    __threadfence_system();
    __syncwarp();
    if (lane == 0) st_volatile_u64(&control->count_flag[rank], epoch);
  }
}

// Writes this rank's key bounds of both join sides into every rank's control block, then raises its bounds flag there.
__global__ void peer_publish_bounds_kernel(PeerControl* const* controls, uint32_t rank, uint32_t world, unsigned long long epoch,
                                           long long build_min, long long build_max, long long build_keys, long long build_rows,
                                           long long probe_min, long long probe_max, long long probe_keys, long long probe_rows) {
  const uint32_t peer = threadIdx.x;
  if (peer < world) {
    PeerControl* control = controls[peer];
    long long* row = control->side_bounds[rank];
    row[0] = build_min, row[1] = build_max, row[2] = build_keys, row[3] = build_rows;
    row[4] = probe_min, row[5] = probe_max, row[6] = probe_keys, row[7] = probe_rows;
    __threadfence_system();
    st_volatile_u64(&control->bounds_flag[rank], epoch);
  }
}

// The persistent one-chunk table over receive region `side` (ValueSegment<int64> of keys), resized to `rows`.
static int received_table(hyb_context* context, PeerGroup* group, int side, uint64_t rows, hyb_table_t* out_handle) {
  Table* table = nullptr;
  if (!group->received[side]) {
    auto created = std::make_unique<Table>();
    created->owner = context;
    created->column_count = 1;
    created->column_types.assign(1, HYB_TYPE_INT64);
    created->chunk_row_start = {0, 0};
    created->chunk_rows = {0};
    DevSegment segment{};
    segment.values = group->region(group->rank, side == 0 ? 0 : 2);
    segment.encoding = HYB_ENC_UNENCODED;
    segment.data_type = HYB_TYPE_INT64;
    segment.vector_type = HYB_VEC_NONE;
    created->segments.push_back(segment);
    created->fixed_single_chunk_capacity = static_cast<uint32_t>(std::min<uint64_t>(group->capacity, 0xFFFFFFF0ull));
    created->position_payload = reinterpret_cast<const hyb_row_id*>(group->region(group->rank, side == 0 ? 1 : 3));
    table = created.get();
    group->received[side] = context->next_handle++;
    context->tables.emplace(group->received[side], std::move(created));
  } else {
    table = find_table(context, group->received[side]);
  }
  table->segments[0].row_count = static_cast<uint32_t>(rows);
  table->chunk_rows[0] = static_cast<uint32_t>(rows);
  table->chunk_row_start[1] = rows;
  table->max_chunk_rows = static_cast<uint32_t>(rows);
  table->uniform_chunks = true;
  table->key_bounds.clear();
  table->dirty = true;
  *out_handle = group->received[side];
  return HYB_OK;
}

// Per-destination counts of one side: count kernel -> scan -> offsets (device, world + 1 entries).
static int peer_count_side(hyb_context* context, DeviceScratch& scratch, const SideInfo& info, uint32_t world, uint32_t chunk_id_base,
                           ProbeParams* params, unsigned long long** out_offsets) {
  const uint32_t tiles = info.source.tile_count;
  const size_t histogram_entries = size_t{world} * std::max<uint32_t>(tiles, 1);
  uint32_t* histogram = nullptr;
  unsigned long long* run_starts = nullptr;
  unsigned long long* offsets = nullptr;
  uint32_t* control = nullptr;
  HYB_TRY(scratch.alloc_array(histogram_entries, &histogram));
  HYB_TRY(scratch.alloc_array(histogram_entries, &run_starts));
  HYB_TRY(scratch.alloc_array(size_t{world} + 1, &offsets));
  HYB_TRY(scratch.alloc_array(16, &control));
  HYB_CUDA(cudaMemsetAsync(control, 0, 64, context->stream));
  HYB_CUDA(cudaMemsetAsync(offsets, 0, sizeof(unsigned long long) * (size_t{world} + 1), context->stream));
  *params = partition_params(info, world, chunk_id_base, control, histogram, run_starts);
  params->out_capacity = ~0ull;
  params->push_to_peers = 1;
  if (tiles) {
    HYB_TRY(count_partitions(context, *params, tiles, reinterpret_cast<unsigned long long*>(control + 4), offsets,
                             [&] { return launch_partition_count(context, *params); }, no_write));
  }
  *out_offsets = offsets;
  return HYB_OK;
}

// The radix width of a distributed join when the caller leaves it to the library: JoinHash's rule over the global build
// side, raised until every rank owns a partition. The co-located and the exchanging path share it, so their results agree.
static int32_t distributed_radix_bits(uint64_t global_build_rows, uint32_t world) {
  int32_t radix_bits = std::max<int32_t>(calculate_radix_bits(global_build_rows), 0);
  while ((1u << radix_bits) < world) ++radix_bits;
  return radix_bits;
}

// Co-located shards: no rank's probe keys [min, max] overlap another rank's build keys. `bounds`: 8 words per rank as
// peer_publish_bounds_kernel writes them (build min, max, has keys, rows; probe min, max, has keys, rows).
static bool shards_colocated(const long long* bounds, uint32_t world) {
  for (uint32_t r = 0; r < world; ++r) {
    for (uint32_t other = 0; other < world; ++other) {
      if (other == r || bounds[r * 8 + 6] == 0 || bounds[other * 8 + 2] == 0) continue;  // no probe keys / no build keys
      if (bounds[r * 8 + 5] >= bounds[other * 8 + 0] && bounds[r * 8 + 4] <= bounds[other * 8 + 1]) return false;
    }
  }
  return true;
}

// Bounds of the build keys this rank received, without another pass: they lie inside the union of the ranks' column
// bounds (`key_info`: min, max, has keys per rank) and agree in their low log2(world) bits, which is what brought them
// here. The min becomes the smallest value >= min with this rank's low bits, which keeps (key - min) a multiple of
// 2^shift: a direct table indexed by (key - min) >> shift.
static Table::KeyBounds received_key_bounds(const long long* key_info, uint32_t world, uint32_t rank) {
  Table::KeyBounds bounds{};
  for (uint32_t source = 0; source < world; ++source) {
    if (key_info[source * 4 + 2] == 0) continue;
    bounds.min = bounds.has_values ? std::min<long long>(bounds.min, key_info[source * 4 + 0]) : key_info[source * 4 + 0];
    bounds.max = bounds.has_values ? std::max<long long>(bounds.max, key_info[source * 4 + 1]) : key_info[source * 4 + 1];
    bounds.has_values = true;
  }
  if (!bounds.has_values) return bounds;
  uint32_t shift = 0;
  while ((1u << shift) < world) ++shift;
  const long long mask = static_cast<long long>(world) - 1;
  const long long aligned = bounds.min + ((static_cast<long long>(rank) - (bounds.min & mask)) & mask);
  bounds.min = aligned;
  bounds.max = std::max(bounds.max, aligned);
  bounds.constant_low_bits = shift;
  return bounds;
}

}  // namespace hyb

extern "C" {

int hyb_join_hash_distributed(hyb_context* context, hyb_peer_group_t group_handle, const hyb_join_side* build_side,
                              const hyb_join_side* probe_side, uint32_t build_chunk_base, uint32_t probe_chunk_base,
                              int32_t radix_bits, hyb_join_result_t* out_result) {
  HYB_CHECK(context && build_side && probe_side && out_result, HYB_ERR_INVALID, "NULL argument");
  *out_result = 0;
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  PeerGroup* group = find_peer_group(context, group_handle);
  HYB_CHECK(group, HYB_ERR_NOT_FOUND, "unknown peer group handle");
  HYB_CHECK(group->connected || group->world == 1, HYB_ERR_INVALID, "peer group is not connected");
  const uint32_t world = group->world, rank = group->rank;
  HYB_CHECK(radix_bits < 0 || (1u << radix_bits) >= world, HYB_ERR_INVALID,
            "radix_bits must give every rank a partition (2^radix_bits >= world)");
  cudaStream_t stream = context->stream;
  SideInfo sides[2];
  HYB_TRY(prepare_side(context, build_side, &sides[0]));
  HYB_TRY(prepare_side(context, probe_side, &sides[1]));
  HYB_CHECK(sides[0].positions < 0xFFFFFFF0ull && sides[1].positions < 0xFFFFFFF0ull, HYB_ERR_UNSUPPORTED,
            "more than 2^32 - 16 rows per join side");
  const unsigned long long epoch = peer_next_epoch(group);
  DeviceScratch scratch(context);
  group->stats = hyb_distributed_stats{};
  HYB_CUDA(cudaEventRecord(group->events[0], stream));
  PeerControl** controls = nullptr;
  HYB_TRY(scratch.alloc_array(kPeerMax, &controls));
  PeerControl* host_controls[kPeerMax] = {};
  for (uint32_t peer = 0; peer < world; ++peer) host_controls[peer] = group->control(peer);
  HYB_CUDA(cudaMemcpyAsync(controls, host_controls, sizeof(host_controls), cudaMemcpyHostToDevice, stream));

  // ---- 0. co-located shards? ------------------------------------------------------------------------------------------------
  // Every rank publishes the [min, max] of its build and probe keys (column statistics, cached with the table like the
  // reference's per-segment MinMaxFilter, statistics/statistics_objects/min_max_filter.hpp). If no rank's probe range touches
  // another rank's build range, every match is local: each rank joins its own shards and emits global RowIDs; partition p of
  // the global result is the concatenation of the ranks' partition-p slices in rank order (a rank's chunks precede those of
  // the next rank). Nothing crosses NVLink but these 64 bytes per pair of ranks. All ranks decide on the same matrix.
  bool colocated = false;
  Table::KeyBounds side_bounds[2]{};
  if (context->options.join_colocated && !sides[0].filter && !sides[1].filter) {
    uint32_t bounds_launches = 0;
    HYB_TRY(column_key_bounds(context, sides[0], &side_bounds[0], &bounds_launches));
    HYB_TRY(column_key_bounds(context, sides[1], &side_bounds[1], &bounds_launches));
    peer_publish_bounds_kernel<<<1, 32, 0, stream>>>(
        controls, rank, world, epoch, side_bounds[0].min, side_bounds[0].max, side_bounds[0].has_values ? 1 : 0,
        static_cast<long long>(sides[0].positions), side_bounds[1].min, side_bounds[1].max, side_bounds[1].has_values ? 1 : 0,
        static_cast<long long>(sides[1].positions));
    HYB_CUDA(cudaGetLastError());
    HYB_TRY(peer_wait(context, group->control(rank)->bounds_flag, world, epoch));
    long long* h_bounds = reinterpret_cast<long long*>(group->h_counts);
    HYB_CUDA(cudaMemcpyAsync(h_bounds, group->control(rank)->side_bounds, sizeof(PeerControl::side_bounds), cudaMemcpyDeviceToHost, stream));
    HYB_CUDA(cudaStreamSynchronize(stream));
    colocated = shards_colocated(h_bounds, world);
    if (colocated) {
      if (radix_bits < 0) {
        uint64_t global_build_rows = 0;
        for (uint32_t r = 0; r < world; ++r) global_build_rows += static_cast<uint64_t>(h_bounds[r * 8 + 3]);
        radix_bits = distributed_radix_bits(global_build_rows, world);
      }
      for (int e = 1; e <= 4; ++e) HYB_CUDA(cudaEventRecord(group->events[e], stream));  // split_count_ms = the bounds exchange
      hyb_join_result_t local_result = 0;
      HYB_TRY(join_hash_locked(context, build_side, probe_side, HYB_JOIN_INNER, radix_bits, &local_result, build_chunk_base,
                               probe_chunk_base));
      HYB_CUDA(cudaEventRecord(group->events[5], stream));
      HYB_CUDA(cudaEventRecord(group->events[6], stream));
      group->stats.colocated = 1;
      *out_result = local_result;
      return HYB_OK;
    }
  }

  // ---- 1. per-destination counts of both sides; publish them (and the build-key bounds) to every rank -------------------
  ProbeParams params[2];
  unsigned long long* offsets[2] = {nullptr, nullptr};
  HYB_TRY(peer_count_side(context, scratch, sides[0], world, build_chunk_base, &params[0], &offsets[0]));
  HYB_TRY(peer_count_side(context, scratch, sides[1], world, probe_chunk_base, &params[1], &offsets[1]));
  Table::KeyBounds local_bounds{};
  uint32_t bounds_launches = 0;
  HYB_TRY(column_key_bounds(context, sides[0], &local_bounds, &bounds_launches));
  peer_publish_counts_kernel<<<1, 32 * kPeerMax, 0, stream>>>(controls, rank, world, epoch, offsets[0], offsets[1], local_bounds.min,
                                                              local_bounds.max, local_bounds.has_values ? 1 : 0);
  HYB_CUDA(cudaGetLastError());
  HYB_CUDA(cudaEventRecord(group->events[1], stream));

  // ---- 2. wait (on the device) for every rank's counts; the one host round trip of the operator -------------------------
  HYB_TRY(peer_wait(context, group->control(rank)->count_flag, world, epoch));
  HYB_CUDA(cudaMemcpyAsync(group->h_counts, group->control(rank)->counts, sizeof(PeerControl::counts) + sizeof(PeerControl::key_info),
                           cudaMemcpyDeviceToHost, stream));
  HYB_CUDA(cudaEventRecord(group->events[2], stream));
  HYB_CUDA(cudaStreamSynchronize(stream));
  const auto count_at = [&](int side, uint32_t source, uint32_t destination) {
    return group->h_counts[(size_t(side) * kPeerMax + source) * kPeerMax + destination];
  };
  const long long* key_info = reinterpret_cast<const long long*>(group->h_counts + 2 * kPeerMax * kPeerMax);
  uint64_t received[2] = {0, 0}, sent_elsewhere = 0;
  for (int side = 0; side < 2; ++side) {
    for (uint32_t destination = 0; destination < world; ++destination) {
      uint64_t before = 0, total = 0;
      for (uint32_t source = 0; source < world; ++source) {
        if (source < rank) before += count_at(side, source, destination);
        total += count_at(side, source, destination);
      }
      HYB_CHECK(total <= group->capacity, HYB_ERR_OOM,
                "receive region of rank " + std::to_string(destination) + " too small: " + std::to_string(total) + " tuples > " +
                    std::to_string(group->capacity));
      params[side].peer_keys[destination] = reinterpret_cast<long long*>(group->region(destination, side == 0 ? 0 : 2)) + before;
      params[side].peer_rows[destination] = reinterpret_cast<long long*>(group->region(destination, side == 0 ? 1 : 3)) + before;
      if (destination == rank) received[side] = total;
      if (destination != rank) sent_elsewhere += count_at(side, rank, destination);
    }
  }
  group->stats.tuples_sent = sent_elsewhere;
  group->stats.tuples_received = received[0] + received[1];
  group->stats.nvlink_bytes = sent_elsewhere * 16;

  // ---- 3. fused split + NVLink stores of both sides; the last CTA raises this rank's done flag everywhere ------------------
  int write_blocks = 1;
  HYB_CUDA(cudaFuncSetAttribute(join_partition_write_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(kPartitionStageBytes)));
  HYB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&write_blocks, join_partition_write_kernel, kJoinThreads, kPartitionStageBytes));
  uint32_t grids[2];
  uint32_t expected = 0;
  for (int side = 0; side < 2; ++side) {
    const uint32_t tiles = sides[side].source.tile_count;
    grids[side] = tiles ? tile_grid(context, tiles, write_blocks) : 0;
    expected += grids[side];
  }
  HYB_CUDA(cudaMemsetAsync(group->d_arrivals, 0, sizeof(unsigned int), stream));
  for (int side = 0; side < 2; ++side) {
    params[side].signal_arrivals = group->d_arrivals;
    params[side].signal_expected = std::max<uint32_t>(expected, 1);
    params[side].signal_world = world;
    params[side].signal_epoch = epoch;
    for (uint32_t peer = 0; peer < world; ++peer) params[side].signal_flags[peer] = &group->control(peer)->done_flag[rank];
    if (grids[side]) {
      join_partition_write_kernel<<<grids[side], kJoinThreads, kPartitionStageBytes, stream>>>(params[side]);
      HYB_CUDA(cudaGetLastError());
    }
  }
  if (expected == 0) {
    peer_signal_kernel<<<1, 32, 0, stream>>>(params[0]);  // nothing to send: still tell the peers this rank is done
    HYB_CUDA(cudaGetLastError());
  }
  HYB_CUDA(cudaEventRecord(group->events[3], stream));

  // ---- 4. wait for every rank's stores, then join what arrived ------------------------------------------------------------
  HYB_TRY(peer_wait(context, group->control(rank)->done_flag, world, epoch));
  HYB_CUDA(cudaEventRecord(group->events[4], stream));
  if (radix_bits < 0) {
    uint64_t global_build = 0;
    for (uint32_t source = 0; source < world; ++source) {
      for (uint32_t destination = 0; destination < world; ++destination) global_build += count_at(0, source, destination);
    }
    radix_bits = distributed_radix_bits(global_build, world);
  }
  hyb_table_t tables[2];
  HYB_TRY(received_table(context, group, 0, received[0], &tables[0]));
  HYB_TRY(received_table(context, group, 1, received[1], &tables[1]));
  const Table::KeyBounds bounds = received_key_bounds(key_info, world, rank);
  if (bounds.has_values && received[0] > 0) find_table(context, tables[0])->key_bounds.emplace(0u, bounds);
  hyb_join_side local_build{tables[0], 0, 0}, local_probe{tables[1], 0, 0};
  hyb_join_result_t result_handle = 0;
  HYB_TRY(join_hash_locked(context, &local_build, &local_probe, HYB_JOIN_INNER, radix_bits, &result_handle));
  HYB_CUDA(cudaEventRecord(group->events[5], stream));

  // ---- 5. nothing to translate: the received tables carry the global RowIDs as their payload and the join emitted them ----
  HYB_CUDA(cudaEventRecord(group->events[6], stream));
  *out_result = result_handle;
  return HYB_OK;
}

}  // extern "C"

extern "C" {

// ---- peer-visible receive arenas (CUDA IPC) ----------------------------------------------------------------------------
int hyb_exchange_arena_create(hyb_context* context, uint64_t bytes, void** out_device_ptr, void* out_ipc_handle) {
  HYB_CHECK(context && out_device_ptr && out_ipc_handle && bytes, HYB_ERR_INVALID, "NULL argument");
  DeviceGuard guard(context->device);
  void* base = nullptr;
  HYB_CUDA(device_malloc_retry(context, &base, bytes));
  cudaIpcMemHandle_t handle;
  const cudaError_t error = cudaIpcGetMemHandle(&handle, base);
  if (error != cudaSuccess) {
    cudaFree(base);
    HYB_CUDA(error);
  }
  static_assert(sizeof(cudaIpcMemHandle_t) == HYB_IPC_HANDLE_BYTES, "IPC handle size");
  std::memcpy(out_ipc_handle, &handle, sizeof(handle));
  *out_device_ptr = base;
  return HYB_OK;
}

int hyb_exchange_arena_open(hyb_context* context, const void* ipc_handle, void** out_peer_ptr) {
  HYB_CHECK(context && ipc_handle && out_peer_ptr, HYB_ERR_INVALID, "NULL argument");
  DeviceGuard guard(context->device);
  cudaIpcMemHandle_t handle;
  std::memcpy(&handle, ipc_handle, sizeof(handle));
  HYB_CUDA(cudaIpcOpenMemHandle(out_peer_ptr, handle, cudaIpcMemLazyEnablePeerAccess));
  return HYB_OK;
}

int hyb_exchange_arena_close(hyb_context* context, void* peer_ptr) {
  HYB_CHECK(context, HYB_ERR_INVALID, "NULL argument");
  DeviceGuard guard(context->device);
  if (peer_ptr) HYB_CUDA(cudaIpcCloseMemHandle(peer_ptr));
  return HYB_OK;
}

int hyb_exchange_arena_destroy(hyb_context* context, void* device_ptr) {
  HYB_CHECK(context, HYB_ERR_INVALID, "NULL argument");
  DeviceGuard guard(context->device);
  if (device_ptr) HYB_CUDA(cudaFree(device_ptr));
  return HYB_OK;
}

static JoinResult* find_join_result(hyb_context* context, hyb_join_result_t handle) {
  auto it = context->join_results.find(handle);
  return it == context->join_results.end() ? nullptr : it->second.get();
}

static int ensure_join_host(hyb_context* context, JoinResult* result) {
  if (result->host_valid) return HYB_OK;
  result->h_partition_offsets.assign(size_t{result->partition_count} + 1, 0);
  HYB_CUDA(cudaMemcpyAsync(result->h_partition_offsets.data(), result->d_partition_offsets,
                           sizeof(uint64_t) * result->h_partition_offsets.size(), cudaMemcpyDeviceToHost, context->stream));
  HYB_CUDA(cudaStreamSynchronize(context->stream));
  result->host_valid = true;
  return HYB_OK;
}

int hyb_join_result_info(hyb_context* context, hyb_join_result_t handle, uint64_t* out_pair_count,
                         uint32_t* out_partition_count, int32_t* out_radix_bits) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* result = find_join_result(context, handle);
  HYB_CHECK(result, HYB_ERR_NOT_FOUND, "unknown join result handle");
  HYB_TRY(ensure_join_host(context, result));
  if (out_pair_count) *out_pair_count = result->h_partition_offsets.back();
  if (out_partition_count) *out_partition_count = result->partition_count;
  if (out_radix_bits) *out_radix_bits = result->radix_bits;
  return HYB_OK;
}

int hyb_join_result_partition_offsets(hyb_context* context, hyb_join_result_t handle, uint64_t* out_offsets) {
  HYB_CHECK(context && out_offsets, HYB_ERR_INVALID, "NULL argument");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* result = find_join_result(context, handle);
  HYB_CHECK(result, HYB_ERR_NOT_FOUND, "unknown join result handle");
  HYB_TRY(ensure_join_host(context, result));
  std::copy(result->h_partition_offsets.begin(), result->h_partition_offsets.end(), out_offsets);
  return HYB_OK;
}

int hyb_join_result_copy(hyb_context* context, hyb_join_result_t handle, uint64_t begin, uint64_t count,
                         hyb_row_id* out_build_row_ids, hyb_row_id* out_probe_row_ids) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* result = find_join_result(context, handle);
  HYB_CHECK(result, HYB_ERR_NOT_FOUND, "unknown join result handle");
  HYB_TRY(ensure_join_host(context, result));
  HYB_CHECK(begin + count <= result->h_partition_offsets.back(), HYB_ERR_INVALID, "range exceeds the join result");
  if (count == 0) return HYB_OK;
  if (out_build_row_ids) {
    HYB_CHECK(result->d_build, HYB_ERR_INVALID, "Semi/Anti joins have no build-side PosList");
    HYB_CUDA(cudaMemcpyAsync(out_build_row_ids, result->d_build + begin, sizeof(hyb_row_id) * count, cudaMemcpyDeviceToHost,
                             context->stream));
  }
  if (out_probe_row_ids) {
    HYB_CUDA(cudaMemcpyAsync(out_probe_row_ids, result->d_probe + begin, sizeof(hyb_row_id) * count, cudaMemcpyDeviceToHost,
                             context->stream));
  }
  HYB_CUDA(cudaStreamSynchronize(context->stream));
  return HYB_OK;
}

int hyb_join_result_pos_list(hyb_context* context, hyb_join_result_t handle, int32_t side, hyb_pos_list_t* out_pos_list) {
  HYB_CHECK(context && out_pos_list && (side == 0 || side == 1), HYB_ERR_INVALID, "bad argument");
  *out_pos_list = 0;
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* result = find_join_result(context, handle);
  HYB_CHECK(result, HYB_ERR_NOT_FOUND, "unknown join result handle");
  HYB_TRY(ensure_join_host(context, result));
  const hyb_row_id* source = side == 0 ? result->d_build : result->d_probe;
  HYB_CHECK(source, HYB_ERR_INVALID, "Semi/Anti joins have no build-side PosList");
  const hyb_table_t table = side == 0 ? result->build_table : result->probe_table;
  HYB_CHECK(table && find_table(context, table), HYB_ERR_INVALID, "the join's input table has been dropped");
  const uint64_t total = result->h_partition_offsets.back();
  auto list = std::make_unique<PosList>();
  list->table = table;
  list->chunk_count = 1;  // one list in result order (the rows of many chunks interleave)
  list->capacity = total;
  list->ascending = false;
  list->may_hold_null_rows = result->mode == HYB_JOIN_LEFT || result->mode == HYB_JOIN_RIGHT;
  list->stream = context->stream;
  list->owner = context;
  void* rows = nullptr;
  void* ends = nullptr;
  HYB_TRY(device_alloc(context, sizeof(hyb_row_id) * std::max<uint64_t>(total, 1), &rows));
  list->d_row_ids = static_cast<hyb_row_id*>(rows);
  HYB_TRY(device_alloc(context, sizeof(uint64_t) * 2, &ends));
  list->d_chunk_end = static_cast<uint64_t*>(ends);
  if (total) HYB_CUDA(cudaMemcpyAsync(rows, source, sizeof(hyb_row_id) * total, cudaMemcpyDeviceToDevice, context->stream));
  const uint64_t host_ends[2] = {total, total};
  HYB_CUDA(cudaMemcpyAsync(ends, host_ends, sizeof(host_ends), cudaMemcpyHostToDevice, context->stream));
  HYB_CUDA(cudaStreamSynchronize(context->stream));
  const auto id = context->next_handle++;
  context->pos_lists.emplace(id, std::move(list));
  *out_pos_list = id;
  return HYB_OK;
}

int hyb_join_result_output_chunks(hyb_context* context, hyb_join_result_t handle, uint64_t* out_offsets, uint32_t* inout_count) {
  HYB_CHECK(context && inout_count, HYB_ERR_INVALID, "NULL argument");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* result = find_join_result(context, handle);
  HYB_CHECK(result, HYB_ERR_NOT_FOUND, "unknown join result handle");
  // probe() cuts its slices every PROBE_SIZE_PER_CHUNK probe elements, which secondary predicates decouple from the rows
  HYB_CHECK(!result->secondary, HYB_ERR_UNSUPPORTED, "output chunks of a join with secondary predicates");
  HYB_TRY(ensure_join_host(context, result));
  // probe(): one PosList per non-empty partition and PROBE_SIZE_PER_CHUNK slice of it (join_hash_steps.hpp:47, :644-655)
  constexpr uint64_t kProbeSizePerChunk = uint64_t{HYB_DEFAULT_CHUNK_SIZE} * 2;
  std::vector<uint64_t> list_sizes;
  for (uint32_t partition = 0; partition < result->partition_count; ++partition) {
    const uint64_t rows = result->h_partition_offsets[partition + 1] - result->h_partition_offsets[partition];
    for (uint64_t begin = 0; begin < rows; begin += kProbeSizePerChunk) list_sizes.push_back(std::min(kProbeSizePerChunk, rows - begin));
  }
  // write_output_chunks (join_output_writing.cpp:247-296): merge small lists
  constexpr uint64_t kMinSize = 1000, kMaxSize = kMinSize * 4;
  std::vector<uint64_t> offsets;
  uint64_t position = 0;
  for (size_t list = 0; list < list_sizes.size();) {
    uint64_t size = list_sizes[list];
    offsets.push_back(position);
    while (list + 1 < list_sizes.size() && size < kMinSize && size + list_sizes[list + 1] < kMaxSize) size += list_sizes[++list];
    position += size;
    ++list;
  }
  offsets.push_back(position);
  const uint32_t chunk_count = static_cast<uint32_t>(offsets.size() - 1);
  if (out_offsets) {
    HYB_CHECK(*inout_count >= chunk_count, HYB_ERR_INVALID, "out_offsets holds fewer than the " + std::to_string(chunk_count) + " chunks");
    std::copy(offsets.begin(), offsets.end(), out_offsets);
  }
  *inout_count = chunk_count;
  return HYB_OK;
}

int hyb_join_result_device_ptrs(hyb_context* context, hyb_join_result_t handle, void** out_build_row_ids,
                                void** out_probe_row_ids) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* result = find_join_result(context, handle);
  HYB_CHECK(result, HYB_ERR_NOT_FOUND, "unknown join result handle");
  if (out_build_row_ids) *out_build_row_ids = result->d_build;
  if (out_probe_row_ids) *out_probe_row_ids = result->d_probe;
  return HYB_OK;
}

int hyb_join_result_free(hyb_context* context, hyb_join_result_t handle) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto it = context->join_results.find(handle);
  HYB_CHECK(it != context->join_results.end(), HYB_ERR_NOT_FOUND, "unknown join result handle");
  context->join_results.erase(it);
  return HYB_OK;
}

}  // extern "C"
