// Sort (operators/sort.cpp:287-516) on the device: a stable LSD radix sort per sort column, from the last definition to
// the first, as the reference's successive std::stable_sort calls. Only the permutation (u32 positions into the input)
// moves from one column to the next; no composite key is carried.
//
// Per sort column:
//   1. gather:    every position's value, decoded through the random-access decoders and mapped to an order-preserving
//                 unsigned word (int: sign bit flipped; float / double: the IEEE flip with -0.0 folded to +0.0 and every
//                 NaN one word above +inf; string: its rank; DESC: the complement), plus its null flag;
//   2. histogram: one read of the words builds every 8-bit digit's histogram and counts the NULL rows;
//   3. partition: a stable scatter on the null flag puts the NULL rows in front, in their current order (sort.cpp:435-443);
//   4. scatter:   one stable counting pass per digit of the non-NULL rows, skipped where every row falls into one bucket.
// A scatter pass is a per-tile bucket count, an exclusive scan of the (bucket, tile) counts by decoupled look-back, and a
// stable scatter that ranks each tile's entries by warp match in input order.
#include <algorithm>
#include <cstring>
#include <vector>

#include "device_utils.cuh"
#include "internal.hpp"

namespace hyb {
namespace {

constexpr uint32_t kSortThreads = 256;
constexpr uint32_t kSortWarps = kSortThreads / 32;
constexpr uint32_t kSortRounds = 8;                                // 32-entry rounds per warp in a scatter tile
constexpr uint32_t kSortTile = kSortThreads * kSortRounds;         // 2048 entries per count / scatter tile
constexpr uint32_t kRadixBuckets = 256;
constexpr uint32_t kNoBucket = kRadixBuckets;                      // past the input: counted nowhere
constexpr uint32_t kSortScanItems = 16;
constexpr uint32_t kSortScanTile = kSortThreads * kSortScanItems;  // counts per look-back scan tile

// Position p of the input -> its RowID: the PosList entry, or (table order) the row of the chunk that holds p.
struct SortInput {
  const hyb_row_id* row_ids;     // nullptr: table order
  const uint32_t* chunk_starts;  // table order: first position of every chunk
  uint32_t chunk_count;
};

// Where one sort column's words come from: a column of the table (decoded per row) or words the host computed per position
// (aggregate values).
struct SortKeySource {
  const DevSegment* segments;  // chunk_count descriptors of the column, or nullptr
  const void* words;           // order words per position (segments == nullptr)
  const uint8_t* nulls;        // 1 = NULL, per position (segments == nullptr)
  uint32_t descending;
};

__device__ __forceinline__ hyb_row_id sort_input_row(const SortInput& input, uint32_t position) {
  if (input.row_ids) return input.row_ids[position];
  const uint32_t chunk = find_owner(input.chunk_starts, input.chunk_count, position);
  return hyb_row_id{chunk, position - __ldg(input.chunk_starts + chunk)};
}

// Order-preserving words (host and device: aggregate values are mapped on the host).
__host__ __device__ __forceinline__ uint32_t sort_word_i32(int32_t value) {
  return static_cast<uint32_t>(value) ^ 0x80000000u;
}
__host__ __device__ __forceinline__ unsigned long long sort_word_i64(long long value) {
  return static_cast<unsigned long long>(value) ^ 0x8000000000000000ull;
}
__host__ __device__ __forceinline__ uint32_t sort_word_f32(float value) {
  if (value != value) return 0xFFFFFFFFu;  // every NaN: one word above +inf (0xFF800000)
  if (value == 0.0f) value = 0.0f;         // -0.0 ties with +0.0
  uint32_t bits;
  memcpy(&bits, &value, sizeof(bits));
  return (bits >> 31) ? ~bits : (bits | 0x80000000u);
}
__host__ __device__ __forceinline__ unsigned long long sort_word_f64(double value) {
  if (value != value) return 0xFFFFFFFFFFFFFFFFull;
  if (value == 0.0) value = 0.0;
  unsigned long long bits;
  memcpy(&bits, &value, sizeof(bits));
  return (bits >> 63) ? ~bits : (bits | 0x8000000000000000ull);
}

// The word of one row of a segment; K = uint32_t for int32 / float / string-rank columns, unsigned long long for int64 /
// double columns. String columns arrive as the INT32 dictionary view whose dictionaries are the rank words.
template <typename K>
__device__ __forceinline__ K segment_word(const DevSegment& segment, uint32_t row, bool& is_null) {
  uint32_t index = row;
  if (segment.encoding == HYB_ENC_DICTIONARY) {
    index = load_code1(segment.av, segment.vector_type, segment.bit_width, row);
    is_null = index >= segment.dict_size;
    if (is_null) return 0;
  } else {
    is_null = segment.nulls && segment.nulls[row];
    if (is_null) return 0;
    if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) {
      const uint32_t code = load_code1(segment.av, segment.vector_type, segment.bit_width, row);
      const int32_t minimum = __ldg(static_cast<const int32_t*>(segment.values) + row / HYB_FOR_BLOCK_SIZE);
      return static_cast<K>(sort_word_i32(static_cast<int32_t>(static_cast<uint32_t>(minimum) + code)));
    }
  }
  if constexpr (sizeof(K) == 4) {
    if (segment.data_type == HYB_TYPE_FLOAT32) return sort_word_f32(__ldg(static_cast<const float*>(segment.values) + index));
    return sort_word_i32(__ldg(static_cast<const int32_t*>(segment.values) + index));
  } else {
    if (segment.data_type == HYB_TYPE_FLOAT64) return sort_word_f64(__ldg(static_cast<const double*>(segment.values) + index));
    return sort_word_i64(__ldg(static_cast<const long long*>(segment.values) + index));
  }
}

// 1. words[i], positions[i] and flags[i] (1 = not NULL; flags may be nullptr) of position perm[i] (perm == nullptr: i).
// Writes at index i only after reading perm[i], so positions may be perm itself.
template <typename K>
__global__ void __launch_bounds__(kSortThreads) sort_gather_kernel(SortInput input, SortKeySource source,
                                                                   const uint32_t* perm, uint32_t count, K* __restrict__ words,
                                                                   uint32_t* positions, uint8_t* __restrict__ flags) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
    const uint32_t position = perm ? perm[i] : i;
    bool is_null = false;
    K word = 0;
    if (source.segments) {
      const hyb_row_id row = sort_input_row(input, position);
      if (row.chunk_id == HYB_INVALID_CHUNK_ID) {
        is_null = true;
      } else {
        word = segment_word<K>(source.segments[row.chunk_id], row.chunk_offset, is_null);
      }
    } else {
      is_null = source.nulls[position] != 0;
      word = static_cast<const K*>(source.words)[position];
    }
    if (source.descending) word = ~word;
    words[i] = word;
    positions[i] = position;
    if (flags) flags[i] = is_null ? 0 : 1;
  }
}

// Warp-aggregated shared-memory increment: lanes with the same bucket add once (many rows share the high digits).
__device__ __forceinline__ void count_bucket(uint32_t* counts, uint32_t bucket, uint32_t lane) {
  const uint32_t peers = __match_any_sync(kFullMask, bucket);
  if (bucket != kNoBucket && lane == static_cast<uint32_t>(__ffs(peers) - 1)) atomicAdd(counts + bucket, __popc(peers));
}

// 2. histogram[d * 256 + b]: non-NULL rows whose digit d is b; histogram[sizeof(K) * 256]: NULL rows.
template <typename K>
__global__ void __launch_bounds__(kSortThreads) sort_histogram_kernel(const K* __restrict__ words,
                                                                      const uint8_t* __restrict__ flags, uint32_t count,
                                                                      uint32_t* __restrict__ histogram) {
  constexpr uint32_t kDigits = sizeof(K);
  __shared__ uint32_t s_counts[kDigits * kRadixBuckets + 1];
  for (uint32_t i = threadIdx.x; i < kDigits * kRadixBuckets + 1; i += blockDim.x) s_counts[i] = 0;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t stride = gridDim.x * blockDim.x;
  uint32_t nulls = 0;
  for (uint32_t base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < count; base += stride) {
    const uint32_t i = base + lane;
    const bool present = i < count;
    const bool valid = present && (!flags || flags[i]);
    nulls += present && !valid;
    const K word = valid ? words[i] : K{0};
#pragma unroll
    for (uint32_t d = 0; d < kDigits; ++d) {
      count_bucket(s_counts + d * kRadixBuckets, valid ? static_cast<uint32_t>(word >> (8 * d)) & 0xFFu : kNoBucket, lane);
    }
  }
  if (nulls) atomicAdd(s_counts + kDigits * kRadixBuckets, nulls);
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < kDigits * kRadixBuckets + 1; i += blockDim.x) {
    if (s_counts[i]) atomicAdd(histogram + i, s_counts[i]);
  }
}

template <typename K, bool kFlag>
__device__ __forceinline__ uint32_t entry_bucket(const K* words, const uint8_t* flags, uint32_t i, uint32_t shift) {
  if constexpr (kFlag) {
    return flags[i];  // 0 = NULL: in front
  } else {
    return static_cast<uint32_t>(words[i] >> shift) & 0xFFu;
  }
}

// 4a. counts[b * tile_count + t]: entries of tile t in bucket b (bucket-major, so one exclusive scan gives every
// (bucket, tile) its first output index).
template <typename K, bool kFlag>
__global__ void __launch_bounds__(kSortThreads) sort_count_kernel(const K* __restrict__ words, const uint8_t* __restrict__ flags,
                                                                  uint32_t count, uint32_t shift, uint32_t tile_count,
                                                                  uint32_t* __restrict__ counts) {
  __shared__ uint32_t s_counts[kRadixBuckets];
  const uint32_t lane = threadIdx.x & 31;
  s_counts[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t tile = blockIdx.x;
  const uint32_t first = tile * kSortTile;
#pragma unroll 4
  for (uint32_t r = 0; r < kSortRounds; ++r) {
    const uint32_t i = first + r * kSortThreads + threadIdx.x;
    count_bucket(s_counts, i < count ? entry_bucket<K, kFlag>(words, flags, i, shift) : kNoBucket, lane);
  }
  __syncthreads();
  counts[static_cast<size_t>(threadIdx.x) * tile_count + tile] = s_counts[threadIdx.x];
}

// 4b. In-place exclusive scan of `count` u32 values (the total stays below 2^32) by decoupled look-back.
__global__ void __launch_bounds__(kSortThreads) sort_scan_kernel(uint32_t* values, uint32_t count,
                                                                 unsigned long long* status, uint32_t* ticket) {
  __shared__ uint32_t s_warp[kSortWarps];
  __shared__ uint32_t s_base;
  __shared__ uint32_t s_tile;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
  __syncthreads();
  const uint32_t tile = s_tile;
  const size_t first = static_cast<size_t>(tile) * kSortScanTile + threadIdx.x * kSortScanItems;
  uint32_t items[kSortScanItems];
  uint32_t sum = 0;
#pragma unroll
  for (uint32_t j = 0; j < kSortScanItems; ++j) {
    items[j] = first + j < count ? values[first + j] : 0u;
    sum += items[j];
  }
  const uint32_t inclusive = warp_inclusive_scan(sum, lane);
  if (lane == 31) s_warp[warp] = inclusive;
  __syncthreads();
  uint32_t warp_base = 0, tile_total = 0;
#pragma unroll
  for (uint32_t w = 0; w < kSortWarps; ++w) {
    if (w < warp) warp_base += s_warp[w];
    tile_total += s_warp[w];
  }
  if (warp == 0) {
    const unsigned long long base = lookback_exclusive_prefix(status, tile, tile_total, lane);
    if (lane == 0) s_base = static_cast<uint32_t>(base);
  }
  __syncthreads();
  uint32_t running = s_base + warp_base + inclusive - sum;
#pragma unroll
  for (uint32_t j = 0; j < kSortScanItems; ++j) {
    if (first + j < count) values[first + j] = running;
    running += items[j];
  }
}

// 4c. Stable scatter of one tile. Warp w owns entries [w * 256, (w + 1) * 256) of the tile and ranks them in eight rounds
// of 32 by warp match: an entry's index inside the tile's bucket = entries of its bucket in earlier warps + in earlier
// rounds of its warp + in lower lanes of its round, i.e. its input order. words_out == nullptr: the words are not needed
// any more (the last pass of a sort column), only the positions move.
template <typename K, bool kFlag>
__global__ void __launch_bounds__(kSortThreads) sort_scatter_kernel(const K* __restrict__ words_in,
                                                                    const uint32_t* __restrict__ positions_in,
                                                                    const uint8_t* __restrict__ flags, uint32_t count,
                                                                    uint32_t shift, const uint32_t* __restrict__ offsets,
                                                                    uint32_t tile_count, K* __restrict__ words_out,
                                                                    uint32_t* __restrict__ positions_out) {
  __shared__ uint32_t s_counts[kSortWarps][kRadixBuckets];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lower_lanes = (1u << lane) - 1u;
#pragma unroll
  for (uint32_t w = 0; w < kSortWarps; ++w) s_counts[w][threadIdx.x] = 0;
  __syncthreads();
  const uint32_t first = blockIdx.x * kSortTile + warp * (kSortRounds * 32);
  uint32_t bucket[kSortRounds], rank[kSortRounds], position[kSortRounds];
  K word[kSortRounds];
#pragma unroll
  for (uint32_t r = 0; r < kSortRounds; ++r) {
    const uint32_t i = first + r * 32 + lane;
    const bool valid = i < count;
    word[r] = valid ? words_in[i] : K{0};
    position[r] = valid ? positions_in[i] : 0u;
    bucket[r] = !valid ? kNoBucket : kFlag ? static_cast<uint32_t>(flags[i]) : static_cast<uint32_t>(word[r] >> shift) & 0xFFu;
  }
#pragma unroll
  for (uint32_t r = 0; r < kSortRounds; ++r) {
    const uint32_t peers = __match_any_sync(kFullMask, bucket[r]);
    const uint32_t before = bucket[r] != kNoBucket ? s_counts[warp][bucket[r]] : 0u;
    rank[r] = before + __popc(peers & lower_lanes);
    __syncwarp();
    if (bucket[r] != kNoBucket && (peers & lower_lanes) == 0) s_counts[warp][bucket[r]] = before + __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  {  // thread b: the first output index of bucket b for every warp of the tile
    uint32_t running = offsets[static_cast<size_t>(threadIdx.x) * tile_count + blockIdx.x];
#pragma unroll
    for (uint32_t w = 0; w < kSortWarps; ++w) {
      const uint32_t entries = s_counts[w][threadIdx.x];
      s_counts[w][threadIdx.x] = running;
      running += entries;
    }
  }
  __syncthreads();
#pragma unroll
  for (uint32_t r = 0; r < kSortRounds; ++r) {
    if (bucket[r] == kNoBucket) continue;
    const uint32_t target = s_counts[warp][bucket[r]] + rank[r];
    if (words_out) words_out[target] = word[r];
    positions_out[target] = position[r];
  }
}

// 5. out[i] = the input RowID at perm[i].
__global__ void __launch_bounds__(kSortThreads) sort_output_kernel(SortInput input, const uint32_t* __restrict__ perm,
                                                                   uint32_t count, hyb_row_id* __restrict__ out) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) out[i] = sort_input_row(input, perm[i]);
}

// One sort column as the driver sees it.
struct SortKeyPlan {
  SortKeySource source;
  uint32_t word_bytes;      // 4 or 8
  bool may_hold_nulls;      // else the flags and the partition are skipped
  uint64_t gather_bytes;    // what the gather reads besides the permutation (codes, values, words)
};

// Scratch of one sort, allocated once for the largest word.
struct SortBuffers {
  void* words[2];
  uint32_t* positions[2];
  uint8_t* flags;
  uint32_t* counts;        // kRadixBuckets * tile_count
  unsigned long long* scan_status;  // scan tiles + ticket
  uint32_t* histogram;     // 8 * 256 + 1
  uint32_t tile_count;
  uint32_t scan_tile_count;
};

uint32_t sort_grid(const hyb_context* context, uint64_t count) {
  return static_cast<uint32_t>(std::max<uint64_t>(1, std::min<uint64_t>((count + kSortThreads - 1) / kSortThreads,
                                                                        static_cast<uint64_t>(context->sm_count) * 8)));
}

struct SortProgress {
  uint32_t launches = 0;
  uint32_t scatter_passes = 0;
  uint64_t bytes = 0;
};

// One counting pass over [begin, begin + count) of buffer `from` into buffer 1 - from: count, scan, scatter.
template <typename K, bool kFlag>
int sort_scatter_pass(hyb_context* context, SortBuffers& buffers, uint32_t from, uint32_t begin, uint32_t count,
                      uint32_t shift, bool keep_words, SortProgress& progress) {
  cudaStream_t stream = context->stream;
  const uint32_t tiles = static_cast<uint32_t>((uint64_t{count} + kSortTile - 1) / kSortTile);
  const uint32_t scanned = tiles * kRadixBuckets;
  const uint32_t scan_tiles = (scanned + kSortScanTile - 1) / kSortScanTile;
  const K* words_in = static_cast<const K*>(buffers.words[from]) + begin;
  const uint8_t* flags = buffers.flags ? buffers.flags + begin : nullptr;
  sort_count_kernel<K, kFlag><<<tiles, kSortThreads, 0, stream>>>(words_in, flags, count, shift, tiles, buffers.counts);
  HYB_CUDA(cudaGetLastError());
  HYB_CUDA(cudaMemsetAsync(buffers.scan_status, 0, sizeof(unsigned long long) * (size_t{scan_tiles} + 1), stream));
  sort_scan_kernel<<<scan_tiles, kSortThreads, 0, stream>>>(buffers.counts, scanned, buffers.scan_status,
                                                            reinterpret_cast<uint32_t*>(buffers.scan_status + scan_tiles));
  HYB_CUDA(cudaGetLastError());
  sort_scatter_kernel<K, kFlag><<<tiles, kSortThreads, 0, stream>>>(
      words_in, buffers.positions[from] + begin, flags, count, shift, buffers.counts, tiles,
      keep_words ? static_cast<K*>(buffers.words[1 - from]) + begin : nullptr, buffers.positions[1 - from] + begin);
  HYB_CUDA(cudaGetLastError());
  progress.launches += 3;
  progress.scatter_passes += 1;
  const uint64_t digit_bytes = kFlag ? 1 : sizeof(K);  // what selects the bucket: the null flag or the word
  progress.bytes += uint64_t{count} * digit_bytes                                          // count pass
                    + uint64_t{count} * (sizeof(K) + sizeof(uint32_t) + (kFlag ? 1 : 0))   // scatter reads
                    + uint64_t{count} * ((keep_words ? sizeof(K) : 0) + sizeof(uint32_t))  // scatter writes
                    + uint64_t{scanned} * sizeof(uint32_t) * 3;                            // counts written, scanned, read
  return HYB_OK;
}

// One sort column: gather, histogram, partition, digit passes. `current` names the buffer holding the permutation.
template <typename K>
int sort_one_column(hyb_context* context, const SortInput& input, const SortKeyPlan& key, bool first_step, uint32_t count,
                    SortBuffers& buffers, uint32_t& current, SortProgress& progress) {
  constexpr uint32_t kDigits = sizeof(K);
  cudaStream_t stream = context->stream;
  uint8_t* flags = key.may_hold_nulls ? buffers.flags : nullptr;
  sort_gather_kernel<K><<<sort_grid(context, count), kSortThreads, 0, stream>>>(
      input, key.source, first_step ? nullptr : buffers.positions[current], count, static_cast<K*>(buffers.words[current]),
      buffers.positions[current], flags);
  HYB_CUDA(cudaGetLastError());
  HYB_CUDA(cudaMemsetAsync(buffers.histogram, 0, sizeof(uint32_t) * (kDigits * kRadixBuckets + 1), stream));
  sort_histogram_kernel<K><<<sort_grid(context, count), kSortThreads, 0, stream>>>(
      static_cast<const K*>(buffers.words[current]), flags, count, buffers.histogram);
  HYB_CUDA(cudaGetLastError());
  progress.launches += 2;
  progress.bytes += key.gather_bytes + (first_step ? 0 : uint64_t{count} * sizeof(uint32_t)) +
                    uint64_t{count} * (sizeof(K) + sizeof(uint32_t) + (flags ? 1 : 0))  // gather writes
                    + uint64_t{count} * (sizeof(K) + (flags ? 1 : 0));                  // histogram reads
  uint32_t histogram[kDigits * kRadixBuckets + 1];
  HYB_CUDA(cudaMemcpyAsync(histogram, buffers.histogram, sizeof(histogram), cudaMemcpyDeviceToHost, stream));
  HYB_CUDA(cudaStreamSynchronize(stream));
  const uint32_t nulls = histogram[kDigits * kRadixBuckets];
  const uint32_t values = count - nulls;
  std::vector<uint32_t> digits;  // the digits whose rows do not all share one bucket
  for (uint32_t d = 0; d < kDigits && values > 1; ++d) {
    const uint32_t* bins = histogram + d * kRadixBuckets;
    if (*std::max_element(bins, bins + kRadixBuckets) != values) digits.push_back(d);
  }
  if (nulls && values) {  // 3. NULL rows in front, in their current order
    HYB_TRY((sort_scatter_pass<K, true>(context, buffers, current, 0, count, 0, !digits.empty(), progress)));
    current = 1 - current;
  }
  const uint32_t prefix_buffer = current;
  for (size_t index = 0; index < digits.size(); ++index) {
    HYB_TRY((sort_scatter_pass<K, false>(context, buffers, current, nulls, values, 8 * digits[index],
                                         index + 1 < digits.size(), progress)));
    current = 1 - current;
  }
  if (nulls && current != prefix_buffer) {  // the NULL prefix stayed where the partition wrote it
    HYB_CUDA(cudaMemcpyAsync(buffers.positions[current], buffers.positions[prefix_buffer], sizeof(uint32_t) * nulls,
                             cudaMemcpyDeviceToDevice, stream));
    progress.bytes += uint64_t{nulls} * sizeof(uint32_t) * 2;
  }
  return HYB_OK;
}

// The whole sort: the permutation of [0, count) that orders the input by `keys` (most significant first), left in
// *out_perm (a buffer of `scratch`).
int run_sort(hyb_context* context, DeviceScratch& scratch, const SortInput& input, uint32_t count,
             const std::vector<SortKeyPlan>& keys, uint32_t** out_perm, SortProgress& progress) {
  SortBuffers buffers{};
  uint32_t word_bytes = 4;
  bool any_nulls = false;
  for (const auto& key : keys) {
    word_bytes = std::max(word_bytes, key.word_bytes);
    any_nulls = any_nulls || key.may_hold_nulls;
  }
  buffers.tile_count = static_cast<uint32_t>((uint64_t{count} + kSortTile - 1) / kSortTile);
  const uint64_t scanned = uint64_t{buffers.tile_count} * kRadixBuckets;
  buffers.scan_tile_count = static_cast<uint32_t>((scanned + kSortScanTile - 1) / kSortScanTile);
  for (int b = 0; b < 2; ++b) {
    HYB_TRY(scratch.alloc(size_t{word_bytes} * count + 16, &buffers.words[b]));
    HYB_TRY(scratch.alloc_array(size_t{count}, &buffers.positions[b]));
  }
  if (any_nulls) HYB_TRY(scratch.alloc_array(size_t{count}, &buffers.flags));
  HYB_TRY(scratch.alloc_array(scanned, &buffers.counts));
  HYB_TRY(scratch.alloc_array(size_t{buffers.scan_tile_count} + 1, &buffers.scan_status));
  HYB_TRY(scratch.alloc_array(size_t{8} * kRadixBuckets + 1, &buffers.histogram));
  uint32_t current = 0;
  for (size_t step = keys.size(); step-- > 0;) {
    const bool first_step = step + 1 == keys.size();
    SortBuffers view = buffers;
    if (!keys[step].may_hold_nulls) view.flags = nullptr;
    if (keys[step].word_bytes == 8) {
      HYB_TRY(sort_one_column<unsigned long long>(context, input, keys[step], first_step, count, view, current, progress));
    } else {
      HYB_TRY(sort_one_column<uint32_t>(context, input, keys[step], first_step, count, view, current, progress));
    }
  }
  *out_perm = buffers.positions[current];
  return HYB_OK;
}

// The plan of one sort column of `table`: its descriptors (a string column's rank view), word size and null flag.
int column_key_plan(Table* table, uint32_t column, bool descending, uint64_t rows, SortKeyPlan* out) {
  HYB_CHECK(column < table->column_count, HYB_ERR_INVALID, "sort column " + std::to_string(column) + " out of range");
  const uint32_t chunk_count = table->chunk_count();
  const int32_t type = table->column_types[column];
  SortKeyPlan plan{};
  plan.source.descending = descending ? 1u : 0u;
  plan.word_bytes = (type == HYB_TYPE_INT64 || type == HYB_TYPE_FLOAT64) ? 8 : 4;
  if (type == HYB_TYPE_STRING) {
    auto it = table->string_views.find(column);
    HYB_CHECK(it != table->string_views.end() && it->second->ordered, HYB_ERR_UNSUPPORTED,
              "sorting by string column " + std::to_string(column) + " needs hyb_table_set_string_order");
    plan.source.segments = it->second->d_segments;
  } else {
    plan.source.segments = table->d_segments + size_t{column} * chunk_count;
  }
  uint64_t stored = 0;
  for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
    const DevSegment& segment = table->segments[size_t{chunk} * table->column_count + column];
    plan.may_hold_nulls = plan.may_hold_nulls || (segment.pad & kSegmentMayContainNulls);
    stored += segment.encoding == HYB_ENC_UNENCODED
                  ? size_t{segment.row_count} * data_type_size(segment.data_type)
                  : vector_bytes(segment.vector_type, segment.bit_width, segment.row_count);
    if (segment.nulls) stored += segment.row_count;
  }
  // a filtered input reads its share of the column's codes (RowIDs are counted by the caller)
  const uint64_t table_rows = table->row_count();
  plan.gather_bytes = table_rows ? static_cast<uint64_t>(static_cast<double>(stored) * rows / table_rows) : 0;
  *out = plan;
  return HYB_OK;
}

// Host words of an aggregate column (hyb_aggregate_result_values' values), 4 or 8 bytes per group.
void aggregate_words(const AggregateColumn& column, uint64_t groups, std::vector<uint8_t>& words, uint32_t* word_bytes) {
  const bool wide = column.value_type == HYB_TYPE_INT64 || column.value_type == HYB_TYPE_FLOAT64;
  *word_bytes = wide ? 8 : 4;
  words.assign(groups * *word_bytes, 0);
  for (uint64_t g = 0; g < groups; ++g) {
    if (column.nulls[g]) continue;
    const uint8_t* value = column.values.data() + g * *word_bytes;
    switch (column.value_type) {
      case HYB_TYPE_INT32: {
        int32_t v;
        std::memcpy(&v, value, 4);
        const uint32_t w = sort_word_i32(v);
        std::memcpy(words.data() + g * 4, &w, 4);
        break;
      }
      case HYB_TYPE_FLOAT32: {
        float v;
        std::memcpy(&v, value, 4);
        const uint32_t w = sort_word_f32(v);
        std::memcpy(words.data() + g * 4, &w, 4);
        break;
      }
      case HYB_TYPE_INT64: {
        long long v;
        std::memcpy(&v, value, 8);
        const unsigned long long w = sort_word_i64(v);
        std::memcpy(words.data() + g * 8, &w, 8);
        break;
      }
      default: {
        double v;
        std::memcpy(&v, value, 8);
        const unsigned long long w = sort_word_f64(v);
        std::memcpy(words.data() + g * 8, &w, 8);
        break;
      }
    }
  }
}

// Chunk starts of a table as u32 positions (the table holds fewer than 2^32 rows).
int upload_chunk_starts(hyb_context* context, DeviceScratch& scratch, const Table* table, const uint32_t** out) {
  std::vector<uint32_t> starts(std::max<uint32_t>(table->chunk_count(), 1), 0);
  for (uint32_t chunk = 0; chunk < table->chunk_count(); ++chunk) starts[chunk] = static_cast<uint32_t>(table->chunk_row_start[chunk]);
  uint32_t* device = nullptr;
  HYB_TRY(scratch.alloc_array(starts.size(), &device));
  HYB_CUDA(cudaMemcpyAsync(device, starts.data(), sizeof(uint32_t) * starts.size(), cudaMemcpyHostToDevice, context->stream));
  *out = device;
  return HYB_OK;
}

AggregateResult* find_sort_aggregate_result(hyb_context* context, hyb_aggregate_result_t handle) {
  auto it = context->aggregate_results.find(handle);
  return it == context->aggregate_results.end() ? nullptr : it->second.get();
}

}  // namespace
}  // namespace hyb

using namespace hyb;

extern "C" {

int hyb_sort(hyb_context* context, hyb_table_t table_handle, hyb_pos_list_t input_filter, const hyb_sort_column* columns,
             uint32_t column_count, hyb_pos_list_t* out_pos_list) {
  HYB_CHECK(context && out_pos_list && (columns || column_count == 0), HYB_ERR_INVALID, "NULL argument");
  *out_pos_list = 0;
  HYB_CHECK(column_count >= 1, HYB_ERR_INVALID, "a sort needs at least one column");
  HYB_CHECK(column_count <= HYB_MAX_SORT_COLUMNS, HYB_ERR_UNSUPPORTED,
            "more than " + std::to_string(HYB_MAX_SORT_COLUMNS) + " sort columns run on the CPU operator");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* table = find_table(context, table_handle);
  HYB_CHECK(table, HYB_ERR_INVALID, "unknown table handle");
  PosList* filter = nullptr;
  if (input_filter) {
    filter = find_pos_list(context, input_filter);
    HYB_CHECK(filter, HYB_ERR_INVALID, "unknown input_filter handle");
    HYB_CHECK(filter->table == table_handle, HYB_ERR_INVALID, "input_filter belongs to a different table");
  }
  uint64_t rows = table->row_count();
  if (filter) HYB_TRY(pos_list_total(context, filter, &rows));
  HYB_CHECK(rows < 0xFFFFFFFFull, HYB_ERR_UNSUPPORTED, "sorting 2^32 or more rows runs on the CPU operator");
  HYB_TRY(sync_table_descriptors(context, table));
  const uint32_t count = static_cast<uint32_t>(rows);
  std::vector<SortKeyPlan> keys(column_count);
  for (uint32_t c = 0; c < column_count; ++c) {
    HYB_TRY(column_key_plan(table, columns[c].column_id, columns[c].descending != 0, rows, &keys[c]));
    keys[c].may_hold_nulls = keys[c].may_hold_nulls || (filter && filter->may_hold_null_rows);
  }

  timing_begin(context);
  auto result = std::make_unique<PosList>();
  result->table = table_handle;
  result->chunk_count = 1;  // one list in result order
  result->capacity = rows;
  result->ascending = false;
  result->may_hold_null_rows = filter && filter->may_hold_null_rows;
  result->stream = context->stream;
  result->owner = context;
  void* out_rows = nullptr;
  void* ends = nullptr;
  HYB_TRY(device_alloc(context, sizeof(hyb_row_id) * std::max<uint64_t>(rows, 1), &out_rows));
  result->d_row_ids = static_cast<hyb_row_id*>(out_rows);
  HYB_TRY(device_alloc(context, sizeof(uint64_t) * 2, &ends));
  result->d_chunk_end = static_cast<uint64_t*>(ends);
  const uint64_t host_ends[2] = {rows, rows};
  HYB_CUDA(cudaMemcpyAsync(ends, host_ends, sizeof(host_ends), cudaMemcpyHostToDevice, context->stream));

  SortProgress progress;
  timing_kernel_begin(context);
  if (count) {
    DeviceScratch scratch(context);
    SortInput input{};
    if (filter) {
      input.row_ids = filter->d_row_ids;
    } else {
      HYB_TRY(upload_chunk_starts(context, scratch, table, &input.chunk_starts));
      input.chunk_count = table->chunk_count();
    }
    uint32_t* perm = nullptr;
    HYB_TRY(run_sort(context, scratch, input, count, keys, &perm, progress));
    sort_output_kernel<<<sort_grid(context, count), kSortThreads, 0, context->stream>>>(input, perm, count,
                                                                                       result->d_row_ids);
    HYB_CUDA(cudaGetLastError());
    progress.launches += 1;
    const uint64_t input_row_bytes = filter ? uint64_t{count} * sizeof(hyb_row_id) * column_count : 0;  // RowID reads
    progress.bytes += input_row_bytes + uint64_t{count} * (sizeof(uint32_t) + sizeof(hyb_row_id));
  }
  timing_kernel_end(context);
  timing_end(context, progress.launches, progress.bytes, rows, rows);
  context->timing.stats.path = progress.scatter_passes;

  const auto handle = context->next_handle++;
  context->pos_lists.emplace(handle, std::move(result));
  *out_pos_list = handle;
  return HYB_OK;
}

int hyb_aggregate_result_sort(hyb_context* context, hyb_aggregate_result_t handle, const hyb_aggregate_sort_key* keys,
                              uint32_t key_count, uint32_t* out_group_indexes) {
  HYB_CHECK(context && (keys || key_count == 0), HYB_ERR_INVALID, "NULL argument");
  HYB_CHECK(key_count >= 1, HYB_ERR_INVALID, "a sort needs at least one key");
  HYB_CHECK(key_count <= HYB_MAX_SORT_COLUMNS, HYB_ERR_UNSUPPORTED,
            "more than " + std::to_string(HYB_MAX_SORT_COLUMNS) + " sort keys run on the CPU operator");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* result = find_sort_aggregate_result(context, handle);
  HYB_CHECK(result, HYB_ERR_INVALID, "unknown aggregate result handle");
  const uint64_t groups = result->group_count;
  HYB_CHECK(groups < 0xFFFFFFFFull, HYB_ERR_UNSUPPORTED, "sorting 2^32 or more groups runs on the CPU operator");
  Table* table = nullptr;
  bool column_keys = false;
  for (uint32_t k = 0; k < key_count; ++k) {
    const auto& key = keys[k];
    if (key.kind == HYB_SORT_KEY_AGGREGATE) {
      HYB_CHECK(key.index < result->columns.size(), HYB_ERR_INVALID, "aggregate sort key out of range");
      const auto& column = result->columns[key.index];
      HYB_CHECK(!column.is_any, HYB_ERR_UNSUPPORTED, "ANY has no values to sort by: sort by its column instead");
      HYB_CHECK(column.value_type != HYB_TYPE_STRING, HYB_ERR_UNSUPPORTED,
                "sorting by a string aggregate runs on the CPU operator");
    } else {
      HYB_CHECK(key.kind == HYB_SORT_KEY_COLUMN, HYB_ERR_INVALID, "unknown sort key kind");
      column_keys = true;
    }
  }
  if (column_keys) {
    table = find_table(context, result->table);
    HYB_CHECK(table, HYB_ERR_INVALID, "the aggregated table has been dropped");
    HYB_TRY(sync_table_descriptors(context, table));
  }
  std::vector<SortKeyPlan> plans(key_count);
  for (uint32_t k = 0; k < key_count; ++k) {
    if (keys[k].kind == HYB_SORT_KEY_COLUMN) {
      HYB_TRY(column_key_plan(table, keys[k].index, keys[k].descending != 0, groups, &plans[k]));
      plans[k].may_hold_nulls = true;  // representative RowIDs are few: no need to prove the column NULL-free
    }
  }
  if (column_keys) {  // representative RowIDs must point into the table (a distributed result's may not)
    for (const hyb_row_id& row : result->row_ids) {
      if (row.chunk_id == HYB_INVALID_CHUNK_ID) continue;
      HYB_CHECK(row.chunk_id < table->chunk_count() && row.chunk_offset < table->chunk_rows[row.chunk_id], HYB_ERR_INVALID,
                "a representative RowID lies outside the aggregated table: sort by the aggregate's columns on the host");
    }
  }
  if (groups == 0) return HYB_OK;
  HYB_CHECK(out_group_indexes, HYB_ERR_INVALID, "NULL argument");
  const uint32_t count = static_cast<uint32_t>(groups);

  timing_begin(context);
  timing_kernel_begin(context);
  DeviceScratch scratch(context);
  cudaStream_t stream = context->stream;
  SortInput input{};
  uint64_t upload_bytes = 0;
  if (column_keys) {
    hyb_row_id* row_ids = nullptr;
    HYB_TRY(scratch.alloc_array(groups, &row_ids));
    HYB_CUDA(cudaMemcpyAsync(row_ids, result->row_ids.data(), sizeof(hyb_row_id) * groups, cudaMemcpyHostToDevice, stream));
    input.row_ids = row_ids;
    upload_bytes += sizeof(hyb_row_id) * groups;
  }
  std::vector<std::vector<uint8_t>> host_words(key_count);
  for (uint32_t k = 0; k < key_count; ++k) {
    if (keys[k].kind != HYB_SORT_KEY_AGGREGATE) continue;
    const auto& column = result->columns[keys[k].index];
    SortKeyPlan& plan = plans[k];
    aggregate_words(column, groups, host_words[k], &plan.word_bytes);
    void* words = nullptr;
    uint8_t* nulls = nullptr;
    HYB_TRY(scratch.alloc(host_words[k].size(), &words));
    HYB_TRY(scratch.alloc_array(groups, &nulls));
    HYB_CUDA(cudaMemcpyAsync(words, host_words[k].data(), host_words[k].size(), cudaMemcpyHostToDevice, stream));
    HYB_CUDA(cudaMemcpyAsync(nulls, column.nulls.data(), groups, cudaMemcpyHostToDevice, stream));
    plan.source.words = words;
    plan.source.nulls = nulls;
    plan.source.descending = keys[k].descending ? 1u : 0u;
    plan.may_hold_nulls = std::find(column.nulls.begin(), column.nulls.end(), uint8_t{1}) != column.nulls.end();
    plan.gather_bytes = host_words[k].size() + groups;
    upload_bytes += host_words[k].size() + groups;
  }
  SortProgress progress;
  uint32_t* perm = nullptr;
  HYB_TRY(run_sort(context, scratch, input, count, plans, &perm, progress));
  HYB_CUDA(cudaMemcpyAsync(out_group_indexes, perm, sizeof(uint32_t) * groups, cudaMemcpyDeviceToHost, stream));
  HYB_CUDA(cudaStreamSynchronize(stream));
  timing_kernel_end(context);
  timing_end(context, progress.launches, progress.bytes + upload_bytes + sizeof(uint32_t) * groups, groups, groups);
  context->timing.stats.path = progress.scatter_passes;
  return HYB_OK;
}

}  // extern "C"
