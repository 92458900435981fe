// TableScan on the device: predicate evaluation on encoded segments + order-preserving compaction into a RowIDPosList.
//
// Replaces the hot loop AbstractTableScanImpl::_scan_with_iterators / _simd_scan_with_iterators
// (src/lib/operators/table_scan/abstract_table_scan_impl.hpp:56-242) and the per-chunk dispatch of
// ColumnVsValueTableScanImpl (column_vs_value_table_scan_impl.cpp:43-272), ColumnBetweenTableScanImpl
// (column_between_table_scan_impl.cpp:42-226) and ColumnIsNullTableScanImpl for Value / Dictionary / FrameOfReference
// segments. One launch scans every chunk of the column:
//
//   scan_prepare_kernel   one thread per chunk: turns the predicate into a per-chunk test. Dictionary segments get the
//                         value-ID range the reference derives from lower_bound/upper_bound (binary search on the
//                         device-resident dictionary); "no row can match" chunks are marked so the scan skips their
//                         bytes (the reference's early-outs, column_vs_value_table_scan_impl.cpp:228-272).
//   scan_kernel           persistent CTAs claim 4096-row tiles through an atomic ticket. Per tile: 128-bit streaming
//                         loads of value-IDs / values, in-register decode, 8 predicates per thread -> bit mask, warp
//                         prefix sums, one decoupled look-back per tile for the global output offset, matches staged in
//                         shared memory and written as coalesced 8-byte RowIDs. Output order == reference order
//                         (chunk by chunk, ascending ChunkOffset), in a single pass over the input.
//
// HBM traffic per launch = N * (bytes per row of the scanned column) + M * 8 (RowIDs) — the compulsory bytes.
//
// Column-vs-column predicates (hyb_table_scan_columns, ColumnVsColumnTableScanImpl) run through the same two-pass and
// position-filtered kernels: scan_mask_kernel and filtered_scan_kernel are templates on the row evaluator (ColumnRows:
// one column against its ChunkTest; PairRows: two columns against a PairTest, column_pair.cuh). `<column> [NOT] IN (...)`
// (hyb_table_scan_in, the ExpressionEvaluator's _evaluate_in_expression on a literal list) uses them too, with InRows:
// dictionary chunks scan a value-ID range or set built by in_prepare_kernel (numeric) or from the caller's dictionary
// bitmaps (strings), Value / FrameOfReference chunks search the list's intervals (in_list.cuh).
//
// Host side: each of the five entry points (hyb_table_scan, _columns, _in, _expression, _expression_tests) checks and
// prepares its predicate into a ScanPlan and the row evaluator's Extra, then ends in run_scan<Rows>: the result PosList,
// the unfiltered launch (launch_unfiltered; only ColumnRows has the single-pass and bulk kernels) or the position-filtered
// one, the operator stats and the handle. Every scratch block of a call belongs to a DeviceScratch.
#include <algorithm>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <limits>

#include "bulk_copy.cuh"
#include "column_pair.cuh"
#include "device_utils.cuh"
#include "expression_scan.cuh"
#include "in_list.cuh"
#include "internal.hpp"
#include "predicate.cuh"

namespace hyb {

constexpr int kScanThreads = 512;  // 16 warps x 1024 rows: 16384-row tiles (see the look-back note at scan_kernel)
constexpr int kScanWarps = kScanThreads / 32;
constexpr int kScanIterations = 4;                       // 8 rows per thread per iteration
constexpr int kScanWarpRows = 32 * 8 * kScanIterations;  // rows owned by one warp in a tile (contiguous)
constexpr int kScanTileRows = kScanWarps * kScanWarpRows;  // 8192
constexpr int kFilteredTileRows = 4096;                  // position-filtered scan: inputs per tile

struct ScanPredicateDevice {
  int32_t condition;
  int32_t data_type;
  hyb_value lower;
  hyb_value upper;
  const uint32_t* value_id_bounds;  // device copy or nullptr
};

// ---------------------------------------------------------------------------------------------------------------------
// Per-chunk predicate preparation
// ---------------------------------------------------------------------------------------------------------------------
template <typename T>
__device__ uint32_t device_lower_bound(const T* dictionary, uint32_t size, T value) {
  uint32_t lo = 0, hi = size;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (dictionary[mid] < value) {
      lo = mid + 1;
    } else {
      hi = mid;
    }
  }
  return lo;
}

template <typename T>
__device__ uint32_t device_upper_bound(const T* dictionary, uint32_t size, T value) {
  uint32_t lo = 0, hi = size;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (!(value < dictionary[mid])) {
      lo = mid + 1;
    } else {
      hi = mid;
    }
  }
  return lo;
}

__device__ void dictionary_bounds(const DevSegment& segment, hyb_value value, uint32_t& lower, uint32_t& upper) {
  const uint32_t size = segment.dict_size;
  switch (segment.data_type) {
    case HYB_TYPE_INT32:
      lower = device_lower_bound(static_cast<const int32_t*>(segment.values), size, value.i32);
      upper = device_upper_bound(static_cast<const int32_t*>(segment.values), size, value.i32);
      break;
    case HYB_TYPE_INT64:
      lower = device_lower_bound(static_cast<const long long*>(segment.values), size, static_cast<long long>(value.i64));
      upper = device_upper_bound(static_cast<const long long*>(segment.values), size, static_cast<long long>(value.i64));
      break;
    case HYB_TYPE_FLOAT32:
      lower = device_lower_bound(static_cast<const float*>(segment.values), size, value.f32);
      upper = device_upper_bound(static_cast<const float*>(segment.values), size, value.f32);
      break;
    default:
      lower = device_lower_bound(static_cast<const double*>(segment.values), size, value.f64);
      upper = device_upper_bound(static_cast<const double*>(segment.values), size, value.f64);
      break;
  }
}

__device__ __forceinline__ bool is_between(int32_t condition) {
  return condition >= HYB_PRED_BETWEEN_INCLUSIVE && condition <= HYB_PRED_BETWEEN_EXCLUSIVE;
}
__device__ __forceinline__ bool lower_inclusive(int32_t condition) {
  return condition == HYB_PRED_BETWEEN_INCLUSIVE || condition == HYB_PRED_BETWEEN_UPPER_EXCLUSIVE;
}
__device__ __forceinline__ bool upper_inclusive(int32_t condition) {
  return condition == HYB_PRED_BETWEEN_INCLUSIVE || condition == HYB_PRED_BETWEEN_LOWER_EXCLUSIVE;
}

__device__ long long value_as_int(hyb_value value, int32_t data_type) {
  return data_type == HYB_TYPE_INT32 ? static_cast<long long>(value.i32) : static_cast<long long>(value.i64);
}
__device__ double value_as_float(hyb_value value, int32_t data_type) {
  return data_type == HYB_TYPE_FLOAT32 ? static_cast<double>(value.f32) : value.f64;
}

__global__ void scan_prepare_kernel(const DevSegment* __restrict__ segments, uint32_t chunk_count,
                                    ScanPredicateDevice predicate, ChunkTest* __restrict__ tests) {
  const uint32_t chunk = blockIdx.x * blockDim.x + threadIdx.x;
  if (chunk >= chunk_count) return;
  const DevSegment segment = segments[chunk];
  ChunkTest test{};
  test.mode = kTestNone;
  const int32_t condition = predicate.condition;

  if (segment.row_count == 0) {
    tests[chunk] = test;
    return;
  }

  if (segment.encoding == HYB_ENC_DICTIONARY) {
    // Value-ID range [lo, hi) following column_vs_value_table_scan_impl.cpp:96-110 and
    // column_between_table_scan_impl.cpp:112-125. INVALID_VALUE_ID ("past the end") is represented as dict_size.
    const uint32_t size = segment.dict_size;
    uint32_t lo = 0, hi = 0;
    bool negate = false;
    if (condition == HYB_PRED_IS_NULL) {
      lo = size;
      hi = size + 1;
    } else if (condition == HYB_PRED_IS_NOT_NULL) {
      lo = 0;
      hi = size;
    } else if (is_between(condition)) {
      uint32_t lower_lb, lower_ub, upper_lb, upper_ub;
      if (predicate.value_id_bounds) {
        lower_lb = min(predicate.value_id_bounds[4 * chunk + 0], size);
        lower_ub = min(predicate.value_id_bounds[4 * chunk + 1], size);
        upper_lb = min(predicate.value_id_bounds[4 * chunk + 2], size);
        upper_ub = min(predicate.value_id_bounds[4 * chunk + 3], size);
      } else {
        dictionary_bounds(segment, predicate.lower, lower_lb, lower_ub);
        dictionary_bounds(segment, predicate.upper, upper_lb, upper_ub);
      }
      lo = lower_inclusive(condition) ? lower_lb : lower_ub;
      hi = upper_inclusive(condition) ? upper_ub : upper_lb;
    } else {
      uint32_t lb, ub;
      if (predicate.value_id_bounds) {
        lb = min(predicate.value_id_bounds[2 * chunk + 0], size);
        ub = min(predicate.value_id_bounds[2 * chunk + 1], size);
      } else {
        dictionary_bounds(segment, predicate.lower, lb, ub);
      }
      switch (condition) {
        case HYB_PRED_EQUALS:
          lo = lb;
          hi = ub;
          break;
        case HYB_PRED_NOT_EQUALS:
          lo = lb;
          hi = ub;
          negate = true;
          break;
        case HYB_PRED_LESS_THAN:
          lo = 0;
          hi = lb;
          break;
        case HYB_PRED_LESS_THAN_EQUALS:
          lo = 0;
          hi = ub;
          break;
        case HYB_PRED_GREATER_THAN:
          lo = ub;
          hi = size;
          break;
        default:  // HYB_PRED_GREATER_THAN_EQUALS
          lo = lb;
          hi = size;
          break;
      }
    }
    if (negate && lo >= hi) {
      // value not in the dictionary: every non-NULL row matches
      negate = false;
      lo = 0;
      hi = size;
    }
    if (!negate && lo >= hi) {
      test.mode = kTestNone;
    } else {
      test.mode = kTestIdRange;
      test.negate = negate;
      test.id_lo = lo;
      test.id_span = hi - lo;
    }
    tests[chunk] = test;
    return;
  }

  // ValueSegment / FrameOfReferenceSegment: typed comparison (type_comparison.hpp:87-180).
  if (condition == HYB_PRED_IS_NULL || condition == HYB_PRED_IS_NOT_NULL) {
    if (!segment.nulls) {
      if (condition == HYB_PRED_IS_NULL) {
        test.mode = kTestNone;
      } else {
        test.mode = kTestNull;  // no null vector: every row matches
        test.want_null = 0;
      }
    } else {
      test.mode = kTestNull;
      test.want_null = condition == HYB_PRED_IS_NULL;
    }
    tests[chunk] = test;
    return;
  }

  const bool integral = segment.data_type == HYB_TYPE_INT32 || segment.data_type == HYB_TYPE_INT64;
  if (integral) {
    const long long type_min = segment.data_type == HYB_TYPE_INT32 ? INT_MIN : LLONG_MIN;
    const long long type_max = segment.data_type == HYB_TYPE_INT32 ? INT_MAX : LLONG_MAX;
    long long lo = type_min, hi = type_max;
    bool empty = false, negate = false;
    const long long a = value_as_int(predicate.lower, segment.data_type);
    const long long b = value_as_int(predicate.upper, segment.data_type);
    switch (condition) {
      case HYB_PRED_EQUALS:
        lo = hi = a;
        break;
      case HYB_PRED_NOT_EQUALS:
        lo = hi = a;
        negate = true;
        break;
      case HYB_PRED_LESS_THAN:
        if (a == type_min) empty = true;
        hi = a - 1;
        break;
      case HYB_PRED_LESS_THAN_EQUALS:
        hi = a;
        break;
      case HYB_PRED_GREATER_THAN:
        if (a == type_max) empty = true;
        lo = a + 1;
        break;
      case HYB_PRED_GREATER_THAN_EQUALS:
        lo = a;
        break;
      default: {  // BETWEEN (column_between_table_scan_impl.cpp:88-97: empty integer ranges produce no output)
        lo = a;
        hi = b;
        if (!lower_inclusive(condition)) {
          if (a == type_max) empty = true;
          lo = a + 1;
        }
        if (!upper_inclusive(condition)) {
          if (b == type_min) empty = true;
          hi = b - 1;
        }
        break;
      }
    }
    if (empty || lo > hi) {
      test.mode = kTestNone;
    } else {
      test.mode = kTestInt;
      test.negate = negate;
      test.int_lo = lo;
      test.int_hi = hi;
    }
  } else {
    const double a = value_as_float(predicate.lower, segment.data_type);
    const double b = value_as_float(predicate.upper, segment.data_type);
    test.mode = kTestFloat;
    test.float_lo = -INFINITY;
    test.float_hi = INFINITY;
    test.float_lo_inclusive = 1;
    test.float_hi_inclusive = 1;
    switch (condition) {
      case HYB_PRED_EQUALS:
        test.float_lo = test.float_hi = a;
        break;
      case HYB_PRED_NOT_EQUALS:
        test.float_lo = test.float_hi = a;
        test.negate = 1;
        break;
      case HYB_PRED_LESS_THAN:
        test.float_hi = a;
        test.float_hi_inclusive = 0;
        break;
      case HYB_PRED_LESS_THAN_EQUALS:
        test.float_hi = a;
        break;
      case HYB_PRED_GREATER_THAN:
        test.float_lo = a;
        test.float_lo_inclusive = 0;
        break;
      case HYB_PRED_GREATER_THAN_EQUALS:
        test.float_lo = a;
        break;
      default:
        test.float_lo = a;
        test.float_hi = b;
        test.float_lo_inclusive = lower_inclusive(condition);
        test.float_hi_inclusive = upper_inclusive(condition);
        break;
    }
  }
  tests[chunk] = test;
}

struct ScanParams {
  const DevSegment* segments;     // descriptors of the scanned column, one per chunk
  const ChunkTest* tests;         // per chunk
  const uint2* tile_map;          // per tile: {chunk, first row | last-tile-of-chunk << 31}
  uint32_t chunk_count;
  uint32_t tile_count;
  unsigned long long* tile_status;  // tile_count, zero-initialised
  uint32_t* ticket;               // zero-initialised
  hyb_row_id* out;                // capacity = table rows
  unsigned long long* chunk_end;  // [chunk] = inclusive prefix after the chunk's last tile; [chunk_count] = total
  uint32_t prefetch;              // 1: hint the next tile's codes into L2 during the write-out
};

// Per-tile schedule, all of it latency: (1) ticket + tile map entry — prefetched one tile ahead by thread 0;
// (2) column loads, 4 x 128 bit in flight per thread; (3) barrier A: warp totals; (4) warp 0: look-back for the global
// offset, other warps: stage matches in shared memory; (5) barrier B; (6) coalesced RowID stores. Two barriers per
// 8192-row tile; shared-memory reuse across iterations is ordered by those same two barriers (see comments inline).
__global__ void __launch_bounds__(kScanThreads) scan_kernel(const ScanParams params) {
  __shared__ uint16_t s_offsets[kScanTileRows];  // tile-relative offsets of the matches, in row order
  __shared__ uint32_t s_warp_totals[kScanWarps];
  __shared__ uint32_t s_next[2][3];              // double-buffered {tile, chunk, row0|last}
  __shared__ unsigned long long s_base;

  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = threadIdx.x >> 5;

  if (threadIdx.x == 0) {
    const uint32_t tile = atomicAdd(params.ticket, 1u);
    const uint2 info = tile < params.tile_count ? __ldg(params.tile_map + tile) : make_uint2(0, 0);
    s_next[0][0] = tile;
    s_next[0][1] = info.x;
    s_next[0][2] = info.y;
  }
  __syncthreads();

  for (uint32_t iteration = 0;; ++iteration) {
    const uint32_t slot = iteration & 1;
    const uint32_t tile = s_next[slot][0];
    if (tile >= params.tile_count) return;
    const uint32_t chunk = s_next[slot][1];
    const uint32_t tile_row0 = s_next[slot][2] & 0x7FFFFFFFu;
    const bool last_tile_of_chunk = (s_next[slot][2] >> 31) != 0;

    // Claim the next tile now; the answer is only needed after barrier B.
    uint32_t next_tile = 0;
    uint2 next_info = make_uint2(0, 0);
    if (threadIdx.x == 0) {
      next_tile = atomicAdd(params.ticket, 1u);
      if (next_tile < params.tile_count) next_info = __ldg(params.tile_map + next_tile);
    }

    const DevSegment segment = params.segments[chunk];
    const ChunkTest test = params.tests[chunk];

    // 1. predicate masks for this thread's kScanIterations x 8 rows (the warp owns kScanWarpRows contiguous rows)
    uint32_t masks[kScanIterations];
    unsigned long long packed_counts = 0;  // iteration i's count in bits [16i, 16i+16)
#pragma unroll
    for (int it = 0; it < kScanIterations; ++it) {
      const uint32_t row0 = tile_row0 + warp * kScanWarpRows + it * 256 + lane * 8;
      masks[it] = (test.mode != kTestNone && row0 < segment.row_count) ? evaluate8(segment, test, row0) : 0u;
      packed_counts |= static_cast<unsigned long long>(__popc(masks[it])) << (16 * it);
    }

    // 2. warp scan of all iterations at once (each field <= 256 fits 16 bits)
    unsigned long long inclusive = packed_counts;
#pragma unroll
    for (int delta = 1; delta < 32; delta <<= 1) {
      const unsigned long long other = __shfl_up_sync(kFullMask, inclusive, delta);
      if (lane >= static_cast<uint32_t>(delta)) inclusive += other;
    }
    const unsigned long long warp_sums = __shfl_sync(kFullMask, inclusive, 31);
    const unsigned long long exclusive = inclusive - packed_counts;
    uint32_t warp_total = 0;
#pragma unroll
    for (int it = 0; it < kScanIterations; ++it) warp_total += static_cast<uint32_t>((warp_sums >> (16 * it)) & 0xFFFFu);
    if (lane == 31) s_warp_totals[warp] = warp_total;
    __syncthreads();  // barrier A. (s_warp_totals of the previous tile was last read before its barrier B.)

    uint32_t warp_base = 0, tile_total = 0;
#pragma unroll
    for (int w = 0; w < kScanWarps; ++w) {
      const uint32_t total = s_warp_totals[w];
      if (w < static_cast<int>(warp)) warp_base += total;
      tile_total += total;
    }

    // 3. warp 0 resolves the global offset while the other warps stage their matches. s_offsets / s_base of the
    //    previous tile are free: every warp finished its write-out before arriving at barrier A.
    if (warp == 0) {
      const unsigned long long base = lookback_exclusive_prefix(params.tile_status, tile, tile_total, lane);
      if (lane == 0) {
        s_base = base;
        if (last_tile_of_chunk) params.chunk_end[chunk] = base + tile_total;
        if (tile + 1 == params.tile_count) params.chunk_end[params.chunk_count] = base + tile_total;
        s_next[slot ^ 1][0] = next_tile;
        s_next[slot ^ 1][1] = next_info.x;
        s_next[slot ^ 1][2] = next_info.y;
      }
    }
    {
      uint32_t position = warp_base;
#pragma unroll
      for (int it = 0; it < kScanIterations; ++it) {
        // rows of iteration `it` come after all rows of earlier iterations of this warp
        uint32_t at = position + static_cast<uint32_t>((exclusive >> (16 * it)) & 0xFFFFu);
        const uint32_t relative = warp * kScanWarpRows + it * 256 + lane * 8;
        const uint32_t mask = masks[it];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (mask & (1u << j)) s_offsets[at++] = static_cast<uint16_t>(relative + j);
        }
        position += static_cast<uint32_t>((warp_sums >> (16 * it)) & 0xFFFFu);
      }
    }
    __syncthreads();  // barrier B: staging, s_base and s_next[slot ^ 1] are visible

    // 4. coalesced RowID write-out, with the next tile's codes on their way into L2 meanwhile
    if (params.prefetch) {
      const uint32_t following = s_next[slot ^ 1][0];
      if (following < params.tile_count) {
        const DevSegment& next_segment = params.segments[s_next[slot ^ 1][1]];
        const uint32_t next_row = (s_next[slot ^ 1][2] & 0x7FFFFFFFu) + threadIdx.x * (kScanTileRows / kScanThreads);
        if (next_row < next_segment.row_count) prefetch_codes(next_segment, next_row);
      }
    }
    hyb_row_id* out = params.out + s_base;
    for (uint32_t i = threadIdx.x; i < tile_total; i += kScanThreads) {
      st_stream_v2(out + i, chunk, tile_row0 + s_offsets[i]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Two-pass scan (options.scan_two_pass): no CTA ever waits for another one.
//   scan_mask_kernel    reads the column once, evaluates the predicate and keeps one match BIT per row (1/16 of a 2-byte
//                       vector) plus the match count of every tile;
//   scan_bases_kernel   exclusive prefix of the tile counts (one CTA; the counts are a few thousand words);
//   scan_expand_kernel  turns the bits into RowIDs at the tile's known output offset: warp scan, staging in shared memory,
//                       coalesced stores — scan_kernel without its loads, its predicate and its look-back chain.
// Traffic: column + 2 x rows / 8 + RowIDs, i.e. ~5 % more than the single pass; the kernels are plain streaming kernels.
//
// Row evaluators: scan_mask_kernel and filtered_scan_kernel take the chunk's test through `Rows`. `Extra` is what the
// evaluator needs beyond ScanParams / FilteredScanParams; it is the kernels' LAST parameter, so the one-column kernels
// (empty Extra) keep their parameter layout and code.
// ---------------------------------------------------------------------------------------------------------------------
struct ColumnRows {  // <column> <predicate>: the chunk's ChunkTest
  struct Extra {};
  struct Chunk {
    DevSegment segment;
    ChunkTest test;
  };
  static __device__ __forceinline__ Chunk chunk(const ScanParams& params, const Extra&, uint32_t chunk) {
    return Chunk{params.segments[chunk], params.tests[chunk]};
  }
  static __device__ __forceinline__ uint32_t mask8(const Chunk& state, uint32_t row0) {
    return (state.test.mode != kTestNone && row0 < state.segment.row_count) ? evaluate8(state.segment, state.test, row0)
                                                                            : 0u;
  }
  static __device__ __forceinline__ bool test1(const DevSegment* segments, const ChunkTest* tests, const Extra&,
                                               uint32_t chunk, uint32_t row) {
    const DevSegment& segment = segments[chunk];
    const ChunkTest& test = tests[chunk];
    return evaluate1(segment, test, row);
  }
};

struct PairRows {  // <left column> <condition> <right column>: the params' segments are the left column's
  struct Extra {
    const DevSegment* right_segments;  // descriptors of the right column, one per chunk
    const PairTest* tests;             // per chunk
  };
  struct Chunk {
    DevSegment left, right;
    PairTest test;
  };
  static __device__ __forceinline__ Chunk chunk(const ScanParams& params, const Extra& extra, uint32_t chunk) {
    return Chunk{params.segments[chunk], extra.right_segments[chunk], extra.tests[chunk]};
  }
  static __device__ __forceinline__ uint32_t mask8(const Chunk& state, uint32_t row0) {
    return (state.test.mode != kPairNone && row0 < state.left.row_count)
               ? evaluate8_pair(state.left, state.right, state.test, row0)
               : 0u;
  }
  static __device__ __forceinline__ bool test1(const DevSegment* segments, const ChunkTest*, const Extra& extra,
                                               uint32_t chunk, uint32_t row) {
    const PairTest& test = extra.tests[chunk];
    if (test.mode == kPairNone) return false;
    return evaluate1_pair(segments[chunk], extra.right_segments[chunk], test, row);
  }
};

struct InRows {  // <column> [NOT] IN (<literal>, ...): the chunk's ChunkTest, and the list's intervals for Value / FoR chunks
  using Extra = InList;
  struct Chunk {
    DevSegment segment;
    ChunkTest test;
    InList list;
  };
  static __device__ __forceinline__ Chunk chunk(const ScanParams& params, const Extra& extra, uint32_t chunk) {
    return Chunk{params.segments[chunk], params.tests[chunk], extra};
  }
  static __device__ __forceinline__ uint32_t mask8(const Chunk& state, uint32_t row0) {
    if (row0 >= state.segment.row_count) return 0u;
    switch (state.test.mode) {
      case kTestIdRange:
      case kTestIdSet:
        return evaluate8(state.segment, state.test, row0);
      case kTestInList:
        return evaluate8_in(state.segment, state.test, state.list, row0);
      case kTestAll: {
        const uint32_t rows = state.segment.row_count - row0;
        return rows >= 8 ? 0xFFu : ((1u << rows) - 1u);
      }
      default:
        return 0u;
    }
  }
  static __device__ __forceinline__ bool test1(const DevSegment* segments, const ChunkTest* tests, const Extra& extra,
                                               uint32_t chunk, uint32_t row) {
    const ChunkTest& test = tests[chunk];
    switch (test.mode) {
      case kTestIdRange:
      case kTestIdSet:
        return evaluate1(segments[chunk], test, row);
      case kTestInList:
        return evaluate1_in(segments[chunk], test, extra, row);
      case kTestAll:
        return true;
      default:
        return false;
    }
  }
};

struct ExprRows {  // an expression predicate (expression_scan.cuh): the params' segments only give the chunks' row counts
  using Extra = const ExprProgram*;
  struct Chunk {
    const ExprProgram* program;
    uint32_t chunk;
    uint32_t rows;
  };
  static __device__ __forceinline__ Chunk chunk(const ScanParams& params, const Extra& extra, uint32_t chunk) {
    return Chunk{extra, chunk, params.segments[chunk].row_count};
  }
  static __device__ __forceinline__ uint32_t mask8(const Chunk& state, uint32_t row0) {
    return row0 < state.rows ? evaluate8_expression(*state.program, state.chunk, row0, state.rows) : 0u;
  }
  static __device__ __forceinline__ bool test1(const DevSegment*, const ChunkTest*, const Extra& extra, uint32_t chunk,
                                               uint32_t row) {
    return evaluate1_expression(*extra, chunk, row);
  }
};

template <bool kOperands>
struct TestRows {  // an expression predicate with column-test leaves (expression_scan.cuh); kOperands: and operand leaves
  using Extra = const TestProgram*;
  struct Chunk {
    const TestProgram* program;
    uint32_t chunk;
    uint32_t rows;
  };
  static __device__ __forceinline__ Chunk chunk(const ScanParams& params, const Extra& extra, uint32_t chunk) {
    return Chunk{extra, chunk, params.segments[chunk].row_count};
  }
  static __device__ __forceinline__ uint32_t mask8(const Chunk& state, uint32_t row0) {
    return row0 < state.rows ? evaluate8_tests<kOperands>(*state.program, state.chunk, row0, state.rows) : 0u;
  }
  static __device__ __forceinline__ bool test1(const DevSegment*, const ChunkTest*, const Extra& extra, uint32_t chunk,
                                               uint32_t row) {
    return evaluate1_tests<kOperands>(*extra, chunk, row);
  }
};

template <typename Rows>
__global__ void __launch_bounds__(kScanThreads) scan_mask_kernel(const ScanParams params, uint32_t* __restrict__ masks_out,
                                                                 uint32_t* __restrict__ tile_counts,
                                                                 const typename Rows::Extra extra) {
  __shared__ uint32_t s_warp_totals[kScanWarps];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // Two tiles per iteration: their 2 x 4 vector loads per thread are independent and all in flight before the first
  // predicate is evaluated; the two match counts (<= 16 384 each) share one reduction as the halves of a 32-bit word.
  for (uint32_t tile = blockIdx.x; tile < params.tile_count; tile += 2 * gridDim.x) {
    uint32_t packed[2] = {0u, 0u}, counts = 0;
    const uint32_t tiles[2] = {tile, tile + gridDim.x};
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      if (tiles[t] >= params.tile_count) continue;  // uniform
      const uint2 info = __ldg(params.tile_map + tiles[t]);
      const uint32_t chunk = info.x, tile_row0 = info.y & 0x7FFFFFFFu;
      const typename Rows::Chunk state = Rows::chunk(params, extra, chunk);
#pragma unroll
      for (int it = 0; it < kScanIterations; ++it) {
        const uint32_t row0 = tile_row0 + warp * kScanWarpRows + it * 256 + lane * 8;
        const uint32_t mask = Rows::mask8(state, row0);
        packed[t] |= mask << (8 * it);
        counts += static_cast<uint32_t>(__popc(mask)) << (16 * t);
      }
    }
    masks_out[static_cast<size_t>(tiles[0]) * kScanThreads + threadIdx.x] = packed[0];
    if (tiles[1] < params.tile_count) masks_out[static_cast<size_t>(tiles[1]) * kScanThreads + threadIdx.x] = packed[1];
    counts = __reduce_add_sync(kFullMask, counts);  // no carry between the halves: a warp holds <= 1024 rows per tile
    if (lane == 0) s_warp_totals[warp] = counts;
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t total = 0;
#pragma unroll
      for (int w = 0; w < kScanWarps; ++w) total += s_warp_totals[w];
      tile_counts[tiles[0]] = total & 0xFFFFu;
      if (tiles[1] < params.tile_count) tile_counts[tiles[1]] = total >> 16;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(1024) scan_bases_kernel(const uint32_t* __restrict__ tile_counts, uint32_t tile_count,
                                                          unsigned long long* __restrict__ tile_bases) {
  __shared__ unsigned long long s_partial[1024];
  const uint32_t per_thread = (tile_count + 1023) / 1024;
  const uint32_t begin = min(tile_count, threadIdx.x * per_thread), end = min(tile_count, begin + per_thread);
  unsigned long long sum = 0;
  for (uint32_t tile = begin; tile < end; ++tile) sum += tile_counts[tile];
  s_partial[threadIdx.x] = sum;
  __syncthreads();
  for (uint32_t stride = 1; stride < 1024; stride <<= 1) {  // Hillis-Steele inclusive scan of the thread sums
    const unsigned long long other = threadIdx.x >= stride ? s_partial[threadIdx.x - stride] : 0ull;
    __syncthreads();
    s_partial[threadIdx.x] += other;
    __syncthreads();
  }
  unsigned long long running = s_partial[threadIdx.x] - sum;
  for (uint32_t tile = begin; tile < end; ++tile) {
    tile_bases[tile] = running;
    running += tile_counts[tile];
  }
  if (threadIdx.x == 1023) tile_bases[tile_count] = s_partial[1023];
}

__global__ void __launch_bounds__(kScanThreads) scan_expand_kernel(const ScanParams params, const uint32_t* __restrict__ masks_in,
                                                                   const unsigned long long* __restrict__ tile_bases) {
  __shared__ uint16_t s_offsets[kScanTileRows];
  __shared__ uint32_t s_warp_totals[kScanWarps];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t tile = blockIdx.x; tile < params.tile_count; tile += gridDim.x) {
    const uint2 info = __ldg(params.tile_map + tile);
    const uint32_t chunk = info.x, tile_row0 = info.y & 0x7FFFFFFFu;
    const unsigned long long base = __ldg(tile_bases + tile);
    const uint32_t packed = ld_stream_u32(masks_in + static_cast<size_t>(tile) * kScanThreads + threadIdx.x);
    unsigned long long packed_counts = 0;
#pragma unroll
    for (int it = 0; it < kScanIterations; ++it) {
      packed_counts |= static_cast<unsigned long long>(__popc((packed >> (8 * it)) & 0xFFu)) << (16 * it);
    }
    unsigned long long inclusive = packed_counts;
#pragma unroll
    for (int delta = 1; delta < 32; delta <<= 1) {
      const unsigned long long other = __shfl_up_sync(kFullMask, inclusive, delta);
      if (lane >= static_cast<uint32_t>(delta)) inclusive += other;
    }
    const unsigned long long warp_sums = __shfl_sync(kFullMask, inclusive, 31);
    const unsigned long long exclusive = inclusive - packed_counts;
    uint32_t warp_total = 0;
#pragma unroll
    for (int it = 0; it < kScanIterations; ++it) warp_total += static_cast<uint32_t>((warp_sums >> (16 * it)) & 0xFFFFu);
    if (lane == 31) s_warp_totals[warp] = warp_total;
    __syncthreads();  // also: every warp has finished the previous tile's write-out
    uint32_t warp_base = 0, tile_total = 0;
#pragma unroll
    for (int w = 0; w < kScanWarps; ++w) {
      const uint32_t total = s_warp_totals[w];
      if (w < static_cast<int>(warp)) warp_base += total;
      tile_total += total;
    }
    if (threadIdx.x == 0) {
      if (info.y >> 31) params.chunk_end[chunk] = base + tile_total;
      if (tile + 1 == params.tile_count) params.chunk_end[params.chunk_count] = base + tile_total;
    }
    uint32_t position = warp_base;
#pragma unroll
    for (int it = 0; it < kScanIterations; ++it) {
      uint32_t at = position + static_cast<uint32_t>((exclusive >> (16 * it)) & 0xFFFFu);
      const uint32_t relative = warp * kScanWarpRows + it * 256 + lane * 8;
      const uint32_t mask = (packed >> (8 * it)) & 0xFFu;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (mask & (1u << j)) s_offsets[at++] = static_cast<uint16_t>(relative + j);
      }
      position += static_cast<uint32_t>((warp_sums >> (16 * it)) & 0xFFFFu);
    }
    __syncthreads();
    hyb_row_id* out = params.out + base;
    for (uint32_t i = threadIdx.x; i < tile_total; i += kScanThreads) {
      st_stream_v2(out + i, chunk, tile_row0 + s_offsets[i]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// scan_bulk_kernel: the same single-pass ordered compaction, restructured around the Hopper asynchronous machinery
// (TMA bulk copies and mbarriers, sm_90).
//
//   producer warp   one lane claims tiles through the atomic ticket (so every predecessor of a claimed tile is owned by a
//                   running CTA: the look-back cannot deadlock), reads the tile-map entry and the segment descriptor and
//                   issues ONE cp.async.bulk per tile (the TMA unit moves the tile's 8192 codes, <= 32 KB, global ->
//                   shared) that completes on the stage's `full` mbarrier; it runs kBulkStages - 1 tiles ahead of the
//                   consumers and is throttled by the `empty` mbarriers. No load latency is left on the consumers' path.
//   8 consumer warps  wait on `full`, evaluate their 1024 rows from shared memory (conflict-free 128-bit LDS), release
//                   the stage, scan their match counts and publish the warp total. There is no CTA-wide barrier: the
//                   warp that arrives LAST (shared-memory counter) owns the tile's decoupled look-back and publishes the
//                   global offset through the `ready` mbarrier, while the other warps compact their matches into
//                   warp-private staging; each warp then writes its own run of RowIDs (contiguous, 256 bytes per store).
//
// Eligible columns (checked on the host per call): every chunk streams a fixed-width vector of 1, 2 or 4 bytes per row
// (dictionary value-IDs, FrameOfReference offsets, int32 / float values) and has no NULL vector; anything else takes
// scan_kernel.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kBulkStages = 2;
constexpr int kBulkConsumerWarps = kScanWarps;                   // 8 x 1024 rows = one 8192-row tile
constexpr int kBulkThreads = (kBulkConsumerWarps + 1) * 32;      // + the producer warp
constexpr uint32_t kBulkEndOfTiles = 0xFFFFFFFFu;

__device__ __forceinline__ uint32_t evaluate8_staged(const DevSegment& segment, const ChunkTest& test, uint32_t row0,
                                                     const unsigned char* staged, uint32_t width) {
  const uint32_t rows = segment.row_count;
  const uint32_t valid = rows - row0 >= 8 ? 0xFFu : ((1u << (rows - row0)) - 1u);
  uint32_t codes[8];
  if (width == 2) {
    const uint4 v = *reinterpret_cast<const uint4*>(staged);
    codes[0] = v.x & 0xFFFFu;
    codes[1] = v.x >> 16;
    codes[2] = v.y & 0xFFFFu;
    codes[3] = v.y >> 16;
    codes[4] = v.z & 0xFFFFu;
    codes[5] = v.z >> 16;
    codes[6] = v.w & 0xFFFFu;
    codes[7] = v.w >> 16;
  } else if (width == 1) {
    const uint2 v = *reinterpret_cast<const uint2*>(staged);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      codes[j] = (v.x >> (8 * j)) & 0xFFu;
      codes[4 + j] = (v.y >> (8 * j)) & 0xFFu;
    }
  } else {
    const uint4 a = *reinterpret_cast<const uint4*>(staged);
    const uint4 b = *reinterpret_cast<const uint4*>(staged + 16);
    codes[0] = a.x;
    codes[1] = a.y;
    codes[2] = a.z;
    codes[3] = a.w;
    codes[4] = b.x;
    codes[5] = b.y;
    codes[6] = b.z;
    codes[7] = b.w;
  }
  uint32_t mask = 0;
  switch (test.mode) {
    case kTestIdRange:
      if (!test.negate) {
#pragma unroll
        for (int j = 0; j < 8; ++j) mask |= ((codes[j] - test.id_lo) < test.id_span) ? (1u << j) : 0u;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const bool inside = (codes[j] - test.id_lo) < test.id_span;
          mask |= (!inside && codes[j] < segment.dict_size) ? (1u << j) : 0u;
        }
      }
      break;
    case kTestIdSet:
#pragma unroll
      for (int j = 0; j < 8; ++j) mask |= id_set_contains(test.id_bits, segment.dict_size, codes[j]) ? (1u << j) : 0u;
      break;
    case kTestInt: {
      uint32_t minimum = 0;
      if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) {
        minimum = static_cast<uint32_t>(__ldg(static_cast<const int32_t*>(segment.values) + row0 / HYB_FOR_BLOCK_SIZE));
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const long long value = static_cast<int32_t>(minimum + codes[j]);
        const bool inside = value >= test.int_lo && value <= test.int_hi;
        mask |= (inside != static_cast<bool>(test.negate)) ? (1u << j) : 0u;
      }
      break;
    }
    case kTestFloat:
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const double value = __uint_as_float(codes[j]);
        const bool above = test.float_lo_inclusive ? value >= test.float_lo : value > test.float_lo;
        const bool below = test.float_hi_inclusive ? value <= test.float_hi : value < test.float_hi;
        mask |= ((above && below) != static_cast<bool>(test.negate)) ? (1u << j) : 0u;
      }
      break;
    case kTestNull:  // no NULL vector on this path: IS NOT NULL matches every row
      mask = test.want_null ? 0u : 0xFFu;
      break;
    default:
      break;
  }
  return mask & valid;
}

__global__ void __launch_bounds__(kBulkThreads, 2) scan_bulk_kernel(const ScanParams params, const uint32_t stage_bytes) {
  extern __shared__ __align__(128) unsigned char s_dynamic[];  // kBulkStages input stages, then the match staging
  __shared__ __align__(8) unsigned long long s_full[kBulkStages], s_empty[kBulkStages], s_ready[2];
  __shared__ uint4 s_info[kBulkStages];  // {tile, chunk, row0 | last-tile-of-chunk << 31, bytes per row}
  __shared__ __align__(16) DevSegment s_segment[kBulkStages];  // the tile's chunk: descriptor and predicate test
  __shared__ __align__(16) ChunkTest s_test[kBulkStages];
  __shared__ uint32_t s_totals[2][kBulkConsumerWarps];
  __shared__ uint32_t s_arrived[2];
  __shared__ unsigned long long s_base[2];

  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (int stage = 0; stage < kBulkStages; ++stage) {
      mbarrier_init(&s_full[stage], 1);                    // the producer's arrive (+ the copy's bytes)
      mbarrier_init(&s_empty[stage], kBulkConsumerWarps);  // one arrival per consumer warp
    }
    mbarrier_init(&s_ready[0], 1);
    mbarrier_init(&s_ready[1], 1);
    s_arrived[0] = 0;
    s_arrived[1] = 0;
    mbarrier_init_fence();
  }
  __syncthreads();  // the only CTA-wide barrier of the kernel

  if (warp == kBulkConsumerWarps) {
    // ---- producer warp: lane 0 claims tiles and issues the copies; lanes 0-2 / 3-6 fetch the chunk's segment descriptor /
    //      predicate test (16 bytes each, in parallel) and hand them to the consumers through the stage header ------------
    for (uint32_t fill = 0;; ++fill) {
      const uint32_t stage = fill % kBulkStages;
      uint32_t tile = 0;
      if (lane == 0) {
        mbarrier_wait(&s_empty[stage], ((fill / kBulkStages) & 1u) ^ 1u);  // passes at once for the first kBulkStages fills
        tile = atomicAdd(params.ticket, 1u);
      }
      tile = __shfl_sync(kFullMask, tile, 0);
      if (tile >= params.tile_count) {
        if (lane == 0) {
          s_info[stage] = make_uint4(kBulkEndOfTiles, 0u, 0u, 0u);
          mbarrier_arrive(&s_full[stage]);
        }
        return;
      }
      const uint2 info = __ldg(params.tile_map + tile);
      static_assert(sizeof(DevSegment) == 48 && sizeof(ChunkTest) == 64, "copied as 3 + 4 uint4");
      if (lane < 3) {
        reinterpret_cast<uint4*>(&s_segment[stage])[lane] = __ldg(reinterpret_cast<const uint4*>(params.segments + info.x) + lane);
      } else if (lane < 7) {
        reinterpret_cast<uint4*>(&s_test[stage])[lane - 3] = __ldg(reinterpret_cast<const uint4*>(params.tests + info.x) + (lane - 3));
      }
      __syncwarp();
      if (lane == 0) {
        const DevSegment& segment = s_segment[stage];
        const uint32_t row0 = info.y & 0x7FFFFFFFu;
        const char* base;
        const uint32_t width = segment_stream(segment, base);
        s_info[stage] = make_uint4(tile, info.x, info.y, width);
        if (s_test[stage].mode != kTestNone) {
          const uint32_t rows = min(static_cast<uint32_t>(kScanTileRows), segment.row_count - row0);
          const uint32_t bytes = (rows * width + 15u) & ~15u;  // the readable tail pad covers the round-up
          mbarrier_arrive_expect_tx(&s_full[stage], bytes);
          bulk_copy_to_shared(s_dynamic + size_t{stage} * stage_bytes, base + size_t{row0} * width, bytes, &s_full[stage]);
        } else {
          mbarrier_arrive(&s_full[stage]);  // "no row can match": the chunk's bytes are never read
        }
      }
    }
  }

  // ---- consumers ----------------------------------------------------------------------------------------------------
  uint16_t* staging = reinterpret_cast<uint16_t*>(s_dynamic + size_t{kBulkStages} * stage_bytes) + warp * kScanWarpRows;
  for (uint32_t iteration = 0;; ++iteration) {
    const uint32_t stage = iteration % kBulkStages;
    const uint32_t slot = iteration & 1u;
    mbarrier_wait(&s_full[stage], (iteration / kBulkStages) & 1u);
    const uint4 info = s_info[stage];
    if (info.x == kBulkEndOfTiles) return;
    const uint32_t tile = info.x, chunk = info.y, width = info.w;
    const uint32_t tile_row0 = info.z & 0x7FFFFFFFu;
    const bool last_tile_of_chunk = (info.z >> 31) != 0;
    const DevSegment& segment = s_segment[stage];  // shared memory: no global access on the consumers' path
    const ChunkTest& test = s_test[stage];
    const unsigned char* staged = s_dynamic + size_t{stage} * stage_bytes;

    // 1. predicate masks of this thread's kScanIterations x 8 rows, read from the staged tile
    uint32_t masks[kScanIterations];
    unsigned long long packed_counts = 0;  // iteration i's count in bits [16i, 16i+16)
#pragma unroll
    for (int it = 0; it < kScanIterations; ++it) {
      const uint32_t relative = warp * kScanWarpRows + it * 256 + lane * 8;
      const uint32_t row0 = tile_row0 + relative;
      masks[it] = (test.mode != kTestNone && row0 < segment.row_count)
                      ? evaluate8_staged(segment, test, row0, staged + size_t{relative} * width, width)
                      : 0u;
      packed_counts |= static_cast<unsigned long long>(__popc(masks[it])) << (16 * it);
    }
    __syncwarp();
    if (lane == 0) mbarrier_arrive(&s_empty[stage]);  // the producer may refill the stage

    // 2. warp scan of all iterations at once
    unsigned long long inclusive = packed_counts;
#pragma unroll
    for (int delta = 1; delta < 32; delta <<= 1) {
      const unsigned long long other = __shfl_up_sync(kFullMask, inclusive, delta);
      if (lane >= static_cast<uint32_t>(delta)) inclusive += other;
    }
    const unsigned long long warp_sums = __shfl_sync(kFullMask, inclusive, 31);
    const unsigned long long exclusive = inclusive - packed_counts;
    uint32_t warp_total = 0;
#pragma unroll
    for (int it = 0; it < kScanIterations; ++it) warp_total += static_cast<uint32_t>((warp_sums >> (16 * it)) & 0xFFFFu);

    // 3. publish the warp total; the last warp to arrive resolves the tile's global offset (decoupled look-back)
    uint32_t arrived = 0;
    if (lane == 0) {
      s_totals[slot][warp] = warp_total;
      __threadfence_block();
      arrived = atomicAdd(&s_arrived[slot], 1u);
    }
    arrived = __shfl_sync(kFullMask, arrived, 0);
    if (arrived == kBulkConsumerWarps - 1) {
      __threadfence_block();
      uint32_t tile_total = lane < kBulkConsumerWarps ? *reinterpret_cast<volatile uint32_t*>(&s_totals[slot][lane]) : 0u;
#pragma unroll
      for (int delta = 16; delta > 0; delta >>= 1) tile_total += __shfl_xor_sync(kFullMask, tile_total, delta);
      const unsigned long long base = lookback_exclusive_prefix(params.tile_status, tile, tile_total, lane);
      if (lane == 0) {
        s_base[slot] = base;
        if (last_tile_of_chunk) params.chunk_end[chunk] = base + tile_total;
        if (tile + 1 == params.tile_count) params.chunk_end[params.chunk_count] = base + tile_total;
        s_arrived[slot] = 0;  // next use: iteration + 2, after every warp has passed this tile's `ready`
        mbarrier_arrive(&s_ready[slot]);
      }
    }

    // 4. compact this warp's matches (tile-relative offsets, row order) into its private staging
    {
      uint32_t position = 0;
#pragma unroll
      for (int it = 0; it < kScanIterations; ++it) {
        uint32_t at = position + static_cast<uint32_t>((exclusive >> (16 * it)) & 0xFFFFu);
        const uint32_t relative = warp * kScanWarpRows + it * 256 + lane * 8;
        const uint32_t mask = masks[it];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (mask & (1u << j)) staging[at++] = static_cast<uint16_t>(relative + j);
        }
        position += static_cast<uint32_t>((warp_sums >> (16 * it)) & 0xFFFFu);
      }
    }
    __syncwarp();

    // 5. this warp's run of RowIDs: contiguous in the output, 256 bytes per warp store
    mbarrier_wait(&s_ready[slot], (iteration >> 1) & 1u);
    unsigned long long at = s_base[slot];
#pragma unroll
    for (int w = 0; w < kBulkConsumerWarps; ++w) at += w < static_cast<int>(warp) ? s_totals[slot][w] : 0u;
    hyb_row_id* out = params.out + at;
    for (uint32_t i = lane; i < warp_total; i += 32) st_stream_v2(out + i, chunk, tile_row0 + staging[i]);
    __syncwarp();  // staging is rewritten by the next tile
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Position-filtered scan (reference-table input whose pos lists reference a single chunk each — what a previous
// TableScan on the same table produced; abstract_dereferenced_column_table_scan_impl.cpp:38-46 +
// table_scan.cpp:150-197): gather the referenced rows, test, and emit the referenced RowIDs in input order.
// ---------------------------------------------------------------------------------------------------------------------
struct FilteredScanParams {
  const DevSegment* segments;
  const ChunkTest* tests;
  const hyb_row_id* input;            // flat input pos list
  unsigned long long input_count;
  const unsigned long long* input_chunk_end;  // inclusive prefix per chunk of the input list (chunk_count entries)
  uint32_t chunk_count;
  uint32_t tile_count;                // ceil(input_count / kFilteredTileRows)
  unsigned long long* tile_status;
  uint32_t* ticket;
  hyb_row_id* out;
  unsigned long long* out_total;      // [0] = total matches
  uint32_t null_row_matches;          // 1: the predicate is IS NULL — a NULL_ROW_ID (outer join) is a NULL value and matches
};

template <typename Rows>
__global__ void __launch_bounds__(kScanThreads) filtered_scan_kernel(const FilteredScanParams params,
                                                                     const typename Rows::Extra extra) {
  __shared__ hyb_row_id s_rows[kFilteredTileRows];
  __shared__ uint32_t s_warp_totals[kScanWarps];
  __shared__ uint32_t s_tile;
  __shared__ unsigned long long s_base;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = threadIdx.x >> 5;
  constexpr int kPerThread = kFilteredTileRows / kScanThreads;  // 16 consecutive inputs per thread

  while (true) {
    if (threadIdx.x == 0) s_tile = atomicAdd(params.ticket, 1u);
    __syncthreads();
    const uint32_t tile = s_tile;
    if (tile >= params.tile_count) return;
    const unsigned long long first = static_cast<unsigned long long>(tile) * kFilteredTileRows +
                                     static_cast<unsigned long long>(threadIdx.x) * kPerThread;
    uint32_t mask = 0;
    hyb_row_id rows[kPerThread];
#pragma unroll
    for (int j = 0; j < kPerThread; ++j) {
      const unsigned long long index = first + j;
      if (index < params.input_count) {
        rows[j] = params.input[index];
        if (rows[j].chunk_id != HYB_INVALID_CHUNK_ID) {
          if (Rows::test1(params.segments, params.tests, extra, rows[j].chunk_id, rows[j].chunk_offset)) mask |= 1u << j;
        } else if (params.null_row_matches) {  // NULL_ROW_ID (outer join): the value is NULL; only IS NULL holds
          mask |= 1u << j;
        }
      }
    }
    const uint32_t count = __popc(mask);
    const uint32_t inclusive = warp_inclusive_scan(count, lane);
    if (lane == 31) s_warp_totals[warp] = inclusive;
    __syncthreads();
    uint32_t warp_base = 0, tile_total = 0;
#pragma unroll
    for (int w = 0; w < kScanWarps; ++w) {
      const uint32_t total = s_warp_totals[w];
      if (w < static_cast<int>(warp)) warp_base += total;
      tile_total += total;
    }
    if (warp == 0) {
      const unsigned long long base = lookback_exclusive_prefix(params.tile_status, tile, tile_total, lane);
      if (lane == 0) {
        s_base = base;
        if (tile + 1 == params.tile_count) params.out_total[0] = base + tile_total;
      }
    }
    uint32_t position = warp_base + inclusive - count;
#pragma unroll
    for (int j = 0; j < kPerThread; ++j) {
      if (mask & (1u << j)) s_rows[position++] = rows[j];
    }
    __syncthreads();
    hyb_row_id* out = params.out + s_base;
    for (uint32_t i = threadIdx.x; i < tile_total; i += kScanThreads) {
      st_stream_v2(out + i, s_rows[i].chunk_id, s_rows[i].chunk_offset);
    }
  }
}

// Per-chunk boundaries of a filtered scan's output: the output is ordered by chunk (it is a subsequence of an input that
// is), so chunk c ends at upper_bound(out, c).
__global__ void pos_list_chunk_ends_kernel(const hyb_row_id* __restrict__ rows, const unsigned long long* total_ptr,
                                           uint32_t chunk_count, unsigned long long* __restrict__ chunk_end) {
  const uint32_t chunk = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long total = *total_ptr;
  if (chunk > chunk_count) return;
  if (chunk == chunk_count) {
    chunk_end[chunk] = total;
    return;
  }
  unsigned long long lo = 0, hi = total;
  while (lo < hi) {
    const unsigned long long mid = (lo + hi) >> 1;
    if (rows[mid].chunk_id <= chunk) {
      lo = mid + 1;
    } else {
      hi = mid;
    }
  }
  chunk_end[chunk] = lo;
}

static bool supported_condition(int32_t condition) {
  return (condition >= HYB_PRED_EQUALS && condition <= HYB_PRED_BETWEEN_EXCLUSIVE) || is_like_condition(condition) ||
         condition == HYB_PRED_IS_NULL || condition == HYB_PRED_IS_NOT_NULL;
}

// Dictionary match bitmaps of a string column (LIKE: ColumnLikeTableScanImpl::_find_matches_in_dictionary,
// column_like_table_scan_impl.cpp:75-140; IN: hyb_in_dictionary_matches) become per-chunk tests on the host, which reads
// the bitmaps anyway. No bit set: kTestNone (the chunk's bytes are skipped); one contiguous run of set bits (every entry,
// or a prefix pattern on a sorted dictionary): kTestIdRange, as fast as a range scan; anything else: kTestIdSet, and only
// those chunks' words are uploaded (*out_uploaded_words, optional, counts them).
static int prepare_bitmap_tests(hyb_context* context, Table* table, uint32_t column_id, const uint32_t* bitmaps, void* tests,
                                void** out_bitmap_scratch, uint64_t* out_uploaded_words = nullptr) {
  const uint32_t chunk_count = table->chunk_count();
  std::vector<ChunkTest> host(chunk_count);
  std::vector<uint32_t> set_words;
  size_t word = 0;
  for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
    const DevSegment& segment = table->segments[size_t{chunk} * table->column_count + column_id];
    const uint32_t size = segment.dict_size;
    const uint32_t* bits = bitmaps + word;
    word += (size_t{size} + 31) / 32;
    ChunkTest& test = host[chunk];
    test = ChunkTest{};
    test.mode = kTestNone;
    if (segment.row_count == 0) continue;
    HYB_CHECK(segment.encoding == HYB_ENC_DICTIONARY, HYB_ERR_INVALID,
              "dictionary bitmaps need dictionary-encoded string segments");
    uint32_t count = 0, first = 0, last = 0;
    for (uint32_t w = 0; w < (size + 31) / 32; ++w) {
      uint32_t bits_w = bits[w];
      if (w == size / 32) bits_w &= (1u << (size & 31)) - 1u;  // padding bits of the last word are ignored
      if (!bits_w) continue;
      if (count == 0) first = 32 * w + static_cast<uint32_t>(__builtin_ctz(bits_w));
      last = 32 * w + 31 - static_cast<uint32_t>(__builtin_clz(bits_w));
      count += static_cast<uint32_t>(__builtin_popcount(bits_w));
    }
    if (count == 0) continue;
    if (last - first + 1 == count) {
      test.mode = kTestIdRange;
      test.id_lo = first;
      test.id_span = count;
    } else {
      test.mode = kTestIdSet;
      test.int_hi = static_cast<long long>(set_words.size());  // word offset until the scratch address is known
      set_words.insert(set_words.end(), bits, bits + (size + 31) / 32);
    }
  }
  if (out_uploaded_words) *out_uploaded_words = set_words.size();
  if (!set_words.empty()) {
    HYB_TRY(device_alloc(context, sizeof(uint32_t) * set_words.size(), out_bitmap_scratch));
    const auto* base = static_cast<const uint32_t*>(*out_bitmap_scratch);
    for (auto& test : host) {
      if (test.mode != kTestIdSet) continue;
      test.id_bits = base + test.int_hi;
      test.int_hi = 0;
    }
    // pageable sources: both copies are staged before cudaMemcpyAsync returns
    HYB_CUDA(cudaMemcpyAsync(*out_bitmap_scratch, set_words.data(), sizeof(uint32_t) * set_words.size(),
                             cudaMemcpyHostToDevice, context->stream));
  }
  if (chunk_count) {
    HYB_CUDA(cudaMemcpyAsync(tests, host.data(), sizeof(ChunkTest) * chunk_count, cudaMemcpyHostToDevice, context->stream));
  }
  return HYB_OK;
}

// Shared by hyb_table_scan and the fused predicates of hyb_aggregate_hash: builds the per-chunk tests on the device. The
// caller owns both blocks on success; on failure neither is left allocated.
int prepare_chunk_tests(hyb_context* context, Table* table, const hyb_scan_predicate* predicate, ChunkTest** out_tests,
                        void** out_bounds_scratch, uint64_t* out_uploaded_bytes) {
  *out_tests = nullptr;
  *out_bounds_scratch = nullptr;
  if (out_uploaded_bytes) *out_uploaded_bytes = 0;
  HYB_CHECK(predicate->column_id < table->column_count, HYB_ERR_INVALID, "predicate column out of range");
  HYB_CHECK(supported_condition(predicate->condition), HYB_ERR_UNSUPPORTED,
            "predicate condition " + std::to_string(predicate->condition) + " is not on the GPU path");
  const uint32_t chunk_count = table->chunk_count();
  const int32_t data_type = table->column_types[predicate->column_id];
  const bool needs_value =
      predicate->condition != HYB_PRED_IS_NULL && predicate->condition != HYB_PRED_IS_NOT_NULL;
  if (is_like_condition(predicate->condition)) {
    // table_scan.cpp creates a ColumnLikeTableScanImpl only for string columns (ScanLikeNonStringColumn)
    HYB_CHECK(data_type == HYB_TYPE_STRING, HYB_ERR_INVALID, "LIKE needs a string column");
    HYB_CHECK(predicate->value_id_bounds, HYB_ERR_INVALID,
              "LIKE scans need host-computed dictionary match bitmaps in value_id_bounds (hyb_like_dictionary_matches)");
    DeviceScratch scratch(context);  // released to the caller on success
    ChunkTest* tests = nullptr;
    HYB_TRY(scratch.alloc_array(chunk_count, &tests));
    void* bitmaps = nullptr;
    uint64_t words = 0;
    const int status = prepare_bitmap_tests(context, table, predicate->column_id, predicate->value_id_bounds, tests,
                                            &bitmaps, &words);
    scratch.adopt(bitmaps);
    if (out_uploaded_bytes) *out_uploaded_bytes = sizeof(uint32_t) * words;
    HYB_TRY(status);
    *out_bounds_scratch = scratch.release(bitmaps);
    *out_tests = static_cast<ChunkTest*>(scratch.release(tests));
    return HYB_OK;
  }
  if (data_type == HYB_TYPE_STRING && needs_value) {
    HYB_CHECK(predicate->value_id_bounds, HYB_ERR_INVALID,
              "string dictionary scans need host-computed value_id_bounds (dictionary_segment.cpp:94-119)");
  }
  ScanPredicateDevice device_predicate{};
  device_predicate.condition = predicate->condition;
  device_predicate.data_type = data_type;
  device_predicate.lower = predicate->lower;
  device_predicate.upper = predicate->upper;
  DeviceScratch scratch(context);  // released to the caller on success
  uint32_t* bounds = nullptr;
  if (predicate->value_id_bounds && needs_value && chunk_count) {
    const bool between = predicate->condition >= HYB_PRED_BETWEEN_INCLUSIVE &&
                         predicate->condition <= HYB_PRED_BETWEEN_EXCLUSIVE;
    const size_t words = size_t{chunk_count} * (between ? 4 : 2);
    HYB_TRY(scratch.alloc_array(words, &bounds));
    HYB_CUDA(cudaMemcpyAsync(bounds, predicate->value_id_bounds, sizeof(uint32_t) * words, cudaMemcpyHostToDevice,
                             context->stream));
    // value_id_bounds is borrowed pageable memory: the copy is staged before cudaMemcpyAsync returns.
    device_predicate.value_id_bounds = bounds;
    if (out_uploaded_bytes) *out_uploaded_bytes = sizeof(uint32_t) * words;
  }
  ChunkTest* tests = nullptr;
  HYB_TRY(scratch.alloc_array(chunk_count, &tests));
  if (chunk_count) {
    const DevSegment* column_segments = table->d_segments + size_t{predicate->column_id} * chunk_count;
    scan_prepare_kernel<<<(chunk_count + 127) / 128, 128, 0, context->stream>>>(column_segments, chunk_count,
                                                                                device_predicate, tests);
    HYB_CUDA(cudaGetLastError());
  }
  *out_bounds_scratch = scratch.release(bounds);
  *out_tests = static_cast<ChunkTest*>(scratch.release(tests));
  return HYB_OK;
}

static uint64_t column_bytes_per_launch(const Table* table, uint32_t column_id) {
  uint64_t bytes = 0;
  for (uint32_t chunk = 0; chunk < table->chunk_count(); ++chunk) {
    const auto& segment = table->segments[size_t{chunk} * table->column_count + column_id];
    if (segment.encoding == HYB_ENC_UNENCODED) {
      bytes += data_type_size(segment.data_type) * segment.row_count;
    } else {
      bytes += vector_bytes(segment.vector_type, segment.bit_width, segment.row_count);
      if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) {
        bytes += sizeof(int32_t) * ((segment.row_count + HYB_FOR_BLOCK_SIZE - 1) / HYB_FOR_BLOCK_SIZE);
      }
    }
    if (segment.nulls) bytes += segment.row_count;
  }
  return bytes;
}

// The two-pass pipeline over params.tile_count (> 0) tiles: match bits and tile counts, their prefix, the expansion.
template <typename Rows>
static int launch_two_pass(hyb_context* context, const ScanParams& params, const typename Rows::Extra& extra) {
  const uint32_t tile_count = params.tile_count;
  DeviceScratch scratch(context);
  uint32_t* masks = nullptr;
  uint32_t* tile_counts = nullptr;
  unsigned long long* tile_bases = nullptr;
  HYB_TRY(scratch.alloc_array(size_t{tile_count} * kScanThreads, &masks));
  HYB_TRY(scratch.alloc_array(tile_count, &tile_counts));
  HYB_TRY(scratch.alloc_array(size_t{tile_count} + 1, &tile_bases));
  int mask_blocks = 1, expand_blocks = 1;
  HYB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&mask_blocks, scan_mask_kernel<Rows>, kScanThreads, 0));
  HYB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&expand_blocks, scan_expand_kernel, kScanThreads, 0));
  scan_mask_kernel<Rows><<<std::min<uint32_t>(tile_count, context->sm_count * std::max(mask_blocks, 1)), kScanThreads, 0,
                           context->stream>>>(params, masks, tile_counts, extra);
  scan_bases_kernel<<<1, 1024, 0, context->stream>>>(tile_counts, tile_count, tile_bases);
  scan_expand_kernel<<<std::min<uint32_t>(tile_count, context->sm_count * std::max(expand_blocks, 1)), kScanThreads, 0,
                       context->stream>>>(params, masks, tile_bases);
  return HYB_OK;
}

// Input = a previous operator's PosList on the same table: gather, test and emit the referenced RowIDs in input order.
// null_row_matches: a NULL_ROW_ID (outer join) satisfies the predicate (IS NULL only).
template <typename Rows>
static int launch_filtered(hyb_context* context, const PosList* filter, const DevSegment* column_segments,
                           const ChunkTest* tests, const typename Rows::Extra& extra, bool null_row_matches,
                           PosList* result, uint64_t* out_input_rows) {
  const uint32_t chunk_count = result->chunk_count;
  uint64_t input_count = 0;
  HYB_TRY(pos_list_total(context, filter, &input_count));
  *out_input_rows = input_count;
  result->capacity = input_count;
  void* out = nullptr;
  HYB_TRY(device_alloc(context, sizeof(hyb_row_id) * std::max<uint64_t>(input_count, 1), &out));
  result->d_row_ids = static_cast<hyb_row_id*>(out);
  const uint32_t tile_count = static_cast<uint32_t>((input_count + kFilteredTileRows - 1) / kFilteredTileRows);
  DeviceScratch scratch(context);
  unsigned long long* status = nullptr;
  HYB_TRY(scratch.alloc_array(size_t{tile_count} + 2, &status));
  HYB_CUDA(cudaMemsetAsync(status, 0, sizeof(uint64_t) * (size_t{tile_count} + 2), context->stream));
  unsigned long long* total = status + tile_count + 1;
  timing_kernel_begin(context);
  if (tile_count > 0) {
    FilteredScanParams params{};
    params.segments = column_segments;
    params.tests = tests;
    params.input = filter->d_row_ids;
    params.input_count = input_count;
    params.chunk_count = chunk_count;
    params.tile_count = tile_count;
    params.tile_status = status;
    params.ticket = reinterpret_cast<uint32_t*>(status + tile_count);
    params.out = result->d_row_ids;
    params.out_total = total;
    params.null_row_matches = null_row_matches;
    int blocks_per_sm = 0;
    HYB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, filtered_scan_kernel<Rows>, kScanThreads, 0));
    const uint32_t grid = std::min<uint32_t>(tile_count, context->sm_count * std::max(blocks_per_sm, 1));
    filtered_scan_kernel<Rows><<<grid, kScanThreads, 0, context->stream>>>(params, extra);
    HYB_CUDA(cudaGetLastError());
  }
  timing_kernel_end(context);
  if (filter->ascending) {
    pos_list_chunk_ends_kernel<<<(chunk_count + 1 + 127) / 128, 128, 0, context->stream>>>(
        result->d_row_ids, total, chunk_count, reinterpret_cast<unsigned long long*>(result->d_chunk_end));
  } else {
    // input in another order than the table's (a join's output, abstract_dereferenced_column_table_scan_impl.cpp:49-86):
    // the matches keep the input order and form ONE list
    result->chunk_count = 1;
    result->ascending = false;
    result->may_hold_null_rows = filter->may_hold_null_rows && null_row_matches;
    pos_list_chunk_ends_kernel<<<1, 128, 0, context->stream>>>(result->d_row_ids, total, 0u,
                                                               reinterpret_cast<unsigned long long*>(result->d_chunk_end));
    HYB_CUDA(cudaMemcpyAsync(result->d_chunk_end + 1, result->d_chunk_end, sizeof(uint64_t), cudaMemcpyDeviceToDevice, context->stream));
  }
  HYB_CUDA(cudaGetLastError());
  return HYB_OK;
}

// What an entry point prepared for run_scan.
struct ScanPlan {
  uint32_t row_column;        // the chunks' row counts come from this column's segments (ColumnRows: the scanned column)
  const ChunkTest* tests;     // ColumnRows / InRows; nullptr otherwise
  uint32_t prepare_launches;  // kernels counted before the scan's own
  uint64_t prepared_bytes;    // uploaded lists / programs / translation words
  uint64_t column_bytes;      // what one unfiltered pass reads (column_bytes_per_launch of every column read)
  bool null_row_matches;      // filtered input: a NULL_ROW_ID satisfies the predicate
};

// The unfiltered scan over params.tile_count tiles; *launches grows by the kernels it starts. Only the one-column
// predicate (ColumnRows, below) has the single-pass and bulk kernels: every other row evaluator takes the two-pass pipeline
// whatever scan_two_pass / scan_bulk say.
template <typename Rows>
static int launch_unfiltered(hyb_context* context, const Table*, const ScanPlan&, const ScanParams& params,
                             const typename Rows::Extra& extra, uint32_t* launches) {
  if (context->options.trace && (!context->options.scan_two_pass || context->options.scan_bulk)) {
    std::fprintf(stderr, "[hyb] table scan: two-pass pipeline (only one-column predicates have the single-pass and bulk "
                         "kernels)\n");
  }
  timing_kernel_begin(context);
  if (params.tile_count > 0) {
    HYB_TRY(launch_two_pass<Rows>(context, params, extra));
    *launches += 3;
  }
  timing_kernel_end(context);
  return HYB_OK;
}

// One column against its ChunkTest: scan_two_pass selects the two-pass pipeline; otherwise scan_bulk selects the
// TMA-staged kernel where every chunk streams a fixed-width vector of <= 4 bytes per row without a NULL vector, and
// scan_kernel runs everywhere else.
template <>
int launch_unfiltered<ColumnRows>(hyb_context* context, const Table* table, const ScanPlan& plan, const ScanParams& column,
                                  const ColumnRows::Extra& extra, uint32_t* launches) {
  const uint32_t tile_count = column.tile_count;
  if (tile_count == 0) {
    timing_kernel_begin(context);
    timing_kernel_end(context);
    return HYB_OK;
  }
  DeviceScratch scratch(context);
  unsigned long long* status = nullptr;  // look-back status per tile, then the ticket
  HYB_TRY(scratch.alloc_array(size_t{tile_count} + 1, &status));
  HYB_CUDA(cudaMemsetAsync(status, 0, sizeof(uint64_t) * (size_t{tile_count} + 1), context->stream));
  ScanParams params = column;
  params.tile_status = status;
  params.ticket = reinterpret_cast<uint32_t*>(status + tile_count);
  params.prefetch = 1;  // measured -8 % kernel time at SF 10
  uint32_t stream_width = 0;
  bool bulk = context->options.scan_bulk;
  for (uint32_t chunk = 0; chunk < params.chunk_count && bulk; ++chunk) {
    const DevSegment& segment = table->segments[size_t{chunk} * table->column_count + plan.row_column];
    uint32_t width = 0;
    if (segment.encoding == HYB_ENC_UNENCODED) {
      width = static_cast<uint32_t>(data_type_size(segment.data_type));
    } else {
      width = segment.vector_type == HYB_VEC_FIXED_1B ? 1u : segment.vector_type == HYB_VEC_FIXED_2B ? 2u
              : segment.vector_type == HYB_VEC_FIXED_4B ? 4u : 0u;
    }
    if (width == 0 || width > 4 || segment.nulls) bulk = false;
    stream_width = std::max(stream_width, width);
  }
  timing_kernel_begin(context);
  if (context->options.scan_two_pass) {
    HYB_TRY(launch_two_pass<ColumnRows>(context, params, extra));
    *launches += 3;
  } else if (bulk) {
    const uint32_t stage_bytes = kScanTileRows * stream_width;
    const size_t dynamic_bytes = size_t{kBulkStages} * stage_bytes + sizeof(uint16_t) * kScanTileRows;
    HYB_CUDA(cudaFuncSetAttribute(scan_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(dynamic_bytes)));
    int blocks_per_sm = 0;
    HYB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, scan_bulk_kernel, kBulkThreads, dynamic_bytes));
    const uint32_t grid = std::min<uint32_t>(tile_count, context->sm_count * std::max(blocks_per_sm, 1));
    scan_bulk_kernel<<<grid, kBulkThreads, dynamic_bytes, context->stream>>>(params, stage_bytes);
    *launches += 1;
  } else {
    int blocks_per_sm = 0;
    HYB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, scan_kernel, kScanThreads, 0));
    const uint32_t grid = std::min<uint32_t>(tile_count, context->sm_count * std::max(blocks_per_sm, 1));
    scan_kernel<<<grid, kScanThreads, 0, context->stream>>>(params);
    *launches += 1;
  }
  timing_kernel_end(context);
  return HYB_OK;
}

// Everything every scan entry point ends in: the result PosList, the unfiltered or the filtered launch, the operator
// stats and the handle.
template <typename Rows>
static int run_scan(hyb_context* context, hyb_table_t table_handle, Table* table, const PosList* filter, const ScanPlan& plan,
                    const typename Rows::Extra& extra, hyb_pos_list_t* out_pos_list) {
  const uint32_t chunk_count = table->chunk_count();
  const DevSegment* row_segments = table->d_segments + size_t{plan.row_column} * chunk_count;
  auto result = std::make_unique<PosList>();
  result->table = table_handle;
  result->chunk_count = chunk_count;
  result->stream = context->stream;
  result->owner = context;
  void* chunk_end = nullptr;
  HYB_TRY(device_alloc(context, sizeof(uint64_t) * (size_t{chunk_count} + 1), &chunk_end));
  result->d_chunk_end = static_cast<uint64_t*>(chunk_end);
  uint32_t launches = plan.prepare_launches;
  uint64_t input_rows = 0, input_bytes = plan.prepared_bytes;

  if (!filter) {
    const uint2* tile_map = nullptr;
    uint32_t tile_count = 0;
    HYB_TRY(get_tile_map(context, table, kScanTileRows, &tile_map, &tile_count));
    input_rows = table->row_count();
    input_bytes += plan.column_bytes;
    result->capacity = table->row_count();
    void* out = nullptr;
    HYB_TRY(device_alloc(context, sizeof(hyb_row_id) * result->capacity, &out));
    result->d_row_ids = static_cast<hyb_row_id*>(out);
    // chunk_end is pre-filled with "unset" so chunks without rows can be patched on the host.
    HYB_CUDA(cudaMemsetAsync(chunk_end, 0xFF, sizeof(uint64_t) * (size_t{chunk_count} + 1), context->stream));
    ScanParams params{};
    params.segments = row_segments;
    params.tests = plan.tests;
    params.tile_map = tile_map;
    params.chunk_count = chunk_count;
    params.tile_count = tile_count;
    params.out = result->d_row_ids;
    params.chunk_end = reinterpret_cast<unsigned long long*>(result->d_chunk_end);
    HYB_TRY(launch_unfiltered<Rows>(context, table, plan, params, extra, &launches));
    HYB_CUDA(cudaGetLastError());
  } else {
    HYB_TRY(launch_filtered<Rows>(context, filter, row_segments, plan.tests, extra, plan.null_row_matches, result.get(),
                                  &input_rows));
    input_bytes += input_rows * sizeof(hyb_row_id);
    launches += 2;  // filtered_scan_kernel, pos_list_chunk_ends_kernel
  }
  timing_end(context, launches, input_bytes, input_rows, 0);
  // result->chunk_count: a filter in another order than the table's leaves one chunk
  timing_output_count(context, result->d_chunk_end + result->chunk_count, sizeof(hyb_row_id));

  const auto handle = context->next_handle++;
  context->pos_lists.emplace(handle, std::move(result));
  *out_pos_list = handle;
  return HYB_OK;
}

// Per-chunk PairTests of a column-vs-column predicate, built on the host from the segment descriptors (ColumnVsColumn-
// TableScanImpl::scan_chunk, column_vs_column_table_scan_impl.cpp). String pairs: the caller's right_in_left words are
// uploaded once and every chunk points at its slice.
static int prepare_pair_tests(hyb_context* context, const Table* table, const hyb_column_scan_predicate* predicate,
                              PairCompare compare, DeviceScratch& scratch, PairTest** out_tests, uint64_t* out_words) {
  const uint32_t chunk_count = table->chunk_count();
  const bool strings = table->column_types[predicate->left_column_id] == HYB_TYPE_STRING;
  std::vector<PairTest> host(chunk_count);
  std::vector<uint64_t> first_word(chunk_count, 0);
  uint64_t words = 0;
  for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
    const DevSegment& left = table->segments[size_t{chunk} * table->column_count + predicate->left_column_id];
    const DevSegment& right = table->segments[size_t{chunk} * table->column_count + predicate->right_column_id];
    PairTest& test = host[chunk];
    test = PairTest{};
    test.mode = kPairNone;
    test.condition = predicate->condition;
    test.compare = compare;
    if (strings) {
      HYB_CHECK(left.encoding == HYB_ENC_DICTIONARY && right.encoding == HYB_ENC_DICTIONARY, HYB_ERR_INVALID,
                "string column-vs-column scans need dictionary segments");
      HYB_CHECK(left.dict_size < (1u << 31) && right.dict_size < (1u << 31), HYB_ERR_UNSUPPORTED,
                "column-vs-column scans need dictionaries of fewer than 2^31 entries");
      first_word[chunk] = words;
      words += right.dict_size;
    }
    const bool all_null = (left.encoding == HYB_ENC_DICTIONARY && left.dict_size == 0) ||
                          (right.encoding == HYB_ENC_DICTIONARY && right.dict_size == 0);
    if (left.row_count == 0 || all_null) continue;
    test.mode = strings ? kPairStringIds : kPairDecoded;
  }
  *out_words = words;
  uint32_t* d_words = nullptr;
  if (strings && words > 0) {
    HYB_TRY(scratch.alloc_array(words, &d_words));
    // pageable source: the copy is staged before cudaMemcpyAsync returns
    HYB_CUDA(cudaMemcpyAsync(d_words, predicate->right_in_left, sizeof(uint32_t) * words, cudaMemcpyHostToDevice,
                             context->stream));
  }
  for (uint32_t chunk = 0; chunk < chunk_count && d_words; ++chunk) host[chunk].right_in_left = d_words + first_word[chunk];
  HYB_TRY(scratch.alloc_array(chunk_count, out_tests));
  if (chunk_count) {
    HYB_CUDA(cudaMemcpyAsync(*out_tests, host.data(), sizeof(PairTest) * chunk_count, cudaMemcpyHostToDevice,
                             context->stream));
  }
  return HYB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// [NOT] IN on a numeric column: per-chunk tests from the list's intervals. A dictionary chunk maps every interval [lo, hi]
// to the value-IDs [lower_bound(lo), upper_bound(hi)) of its device-resident dictionary; the ranges are sorted and
// disjoint like the intervals, and ranges that touch form one run. No run: kTestNone (IN) or every non-NULL row (NOT IN);
// one run: kTestIdRange, negated for NOT IN; more: a kTestIdSet bitmap written here (inverted for NOT IN; the NULL id is
// never set). Value / FrameOfReference chunks search the intervals per row (kTestInList).
// ---------------------------------------------------------------------------------------------------------------------
template <typename Conv>
__device__ void dictionary_id_range(const DevSegment& segment, const InList& list, uint32_t interval, uint32_t& lower,
                                    uint32_t& upper) {
  using T = typename Conv::T;
  const T lo = static_cast<const T*>(list.bounds)[2 * interval];
  const T hi = static_cast<const T*>(list.bounds)[2 * interval + 1];
  uint32_t a = 0, b = segment.dict_size;
  while (a < b) {  // first entry >= lo
    const uint32_t mid = (a + b) >> 1;
    if (gather_entry<Conv>(segment, mid) < lo) {
      a = mid + 1;
    } else {
      b = mid;
    }
  }
  lower = a;
  b = segment.dict_size;
  while (a < b) {  // first entry > hi; a NaN entry (sorted last) counts as greater
    const uint32_t mid = (a + b) >> 1;
    if (gather_entry<Conv>(segment, mid) <= hi) {
      a = mid + 1;
    } else {
      b = mid;
    }
  }
  upper = a;
}

template <typename Conv>
__device__ void in_dictionary_test(const DevSegment& segment, const InList& list, bool negate, uint32_t* bits,
                                   ChunkTest& test) {
  const uint32_t size = segment.dict_size;
  uint32_t runs = 0, first_lo = 0, first_hi = 0, last_hi = 0;
  for (uint32_t i = 0; i < list.interval_count; ++i) {
    uint32_t a, b;
    dictionary_id_range<Conv>(segment, list, i, a, b);
    if (a >= b) continue;
    if (runs > 0 && a == last_hi) {  // touches the previous run
      last_hi = b;
      if (runs == 1) first_hi = b;
      continue;
    }
    if (runs == 0) {
      first_lo = a;
      first_hi = b;
    }
    ++runs;
    last_hi = b;
  }
  if (runs == 0) {
    if (negate && size > 0) {  // no entry is in the list: every non-NULL row matches NOT IN
      test.mode = kTestIdRange;
      test.id_lo = 0;
      test.id_span = size;
    }
    return;
  }
  if (runs == 1) {
    test.mode = kTestIdRange;
    test.negate = negate;
    test.id_lo = first_lo;
    test.id_span = first_hi - first_lo;
    return;
  }
  const uint32_t words = (size + 31) / 32;
  for (uint32_t w = 0; w < words; ++w) bits[w] = 0u;
  for (uint32_t i = 0; i < list.interval_count; ++i) {
    uint32_t a, b;
    dictionary_id_range<Conv>(segment, list, i, a, b);
    for (uint32_t id = a; id < b;) {  // whole words where the range covers them
      const uint32_t bit = id & 31u, take = min(32u - bit, b - id);
      bits[id >> 5] |= (take == 32u ? 0xFFFFFFFFu : ((1u << take) - 1u)) << bit;
      id += take;
    }
  }
  if (negate) {
    for (uint32_t w = 0; w < words; ++w) bits[w] = ~bits[w];
    if (size & 31u) bits[words - 1] &= (1u << (size & 31u)) - 1u;
  }
  test.mode = kTestIdSet;
  test.id_bits = bits;
}

__global__ void in_prepare_kernel(const DevSegment* __restrict__ segments, uint32_t chunk_count, InList list,
                                  uint32_t negate, const unsigned long long* __restrict__ word_offsets,
                                  uint32_t* __restrict__ bits, ChunkTest* __restrict__ tests) {
  const uint32_t chunk = blockIdx.x * blockDim.x + threadIdx.x;
  if (chunk >= chunk_count) return;
  const DevSegment segment = segments[chunk];
  ChunkTest test{};
  test.mode = kTestNone;
  if (segment.row_count > 0) {
    if (segment.encoding != HYB_ENC_DICTIONARY) {
      test.mode = kTestInList;
      test.negate = negate;
    } else {
      uint32_t* chunk_bits = bits ? bits + word_offsets[chunk] : nullptr;
      if (list.compare == kInInt32) {
        in_dictionary_test<AsInt32>(segment, list, negate, chunk_bits, test);
      } else if (list.compare == kInInt64) {
        in_dictionary_test<AsInt64>(segment, list, negate, chunk_bits, test);
      } else if (list.compare == kInFloat) {
        in_dictionary_test<AsFloat>(segment, list, negate, chunk_bits, test);
      } else {
        in_dictionary_test<AsDouble>(segment, list, negate, chunk_bits, test);
      }
    }
  }
  tests[chunk] = test;
}

// The device copy of a numeric list's intervals in its compare type; a list that matches no value of the column becomes
// one empty interval (lo > hi), so a search always has an interval to land on.
template <typename T, typename Member>
static int upload_intervals(hyb_context* context, const std::vector<hyb_value>& bounds, Member hyb_value::*member_of,
                            DeviceScratch& scratch, InList& list, uint64_t* out_bytes) {
  std::vector<T> typed;
  for (const hyb_value& bound : bounds) typed.push_back(static_cast<T>(bound.*member_of));
  if (typed.empty()) typed = {T(1), T(0)};
  T* device = nullptr;
  HYB_TRY(scratch.alloc_array(typed.size(), &device));
  // pageable source: the copy is staged before cudaMemcpyAsync returns
  HYB_CUDA(cudaMemcpyAsync(device, typed.data(), sizeof(T) * typed.size(), cudaMemcpyHostToDevice, context->stream));
  list.bounds = device;
  list.interval_count = static_cast<uint32_t>(typed.size() / 2);
  *out_bytes = sizeof(T) * typed.size();
  return HYB_OK;
}


// Rules 1-3 of hyb_table_scan_in: which elements count, and whether the list reduces to "no row" or "every row". Host
// checks only; `bounds` receives a numeric list's intervals.
static int check_in_predicate(const Table* table, const hyb_in_predicate* predicate, InForm* out_form,
                              std::vector<hyb_value>& bounds) {
  const int32_t condition = predicate->condition;
  HYB_CHECK(condition == HYB_PRED_IN || condition == HYB_PRED_NOT_IN, HYB_ERR_INVALID,
            "hyb_table_scan_in takes IN or NOT IN (condition " + std::to_string(condition) + ")");
  HYB_CHECK(predicate->column_id < table->column_count, HYB_ERR_INVALID, "IN scan column out of range");
  const int32_t data_type = table->column_types[predicate->column_id];
  const bool strings = data_type == HYB_TYPE_STRING;
  const bool negate = condition == HYB_PRED_NOT_IN;
  HYB_CHECK(strings || !predicate->dictionary_matches, HYB_ERR_INVALID,
            "dictionary_matches is for string columns; a numeric column takes its elements");
  bool compatible;
  if (strings) {
    compatible = predicate->dictionary_matches != nullptr;
  } else {
    HYB_TRY(normalize_in_list(data_type, predicate->elements, predicate->element_count, bounds));
    compatible = predicate->element_count > 0 || predicate->has_null_element;
  }
  *out_form = kInList;
  if (!compatible) {
    *out_form = negate ? kInEveryRow : kInNoRow;  // `x IN ()` is false, `x NOT IN ()` is true, NULL rows included
  } else if (!strings && negate && predicate->has_null_element) {
    *out_form = kInNoRow;  // `x != NULL` is NULL: no row satisfies the conjunction
  }
  return HYB_OK;
}

// The per-chunk tests of a checked IN predicate (shared by hyb_table_scan_in and the IN leaves of
// hyb_table_scan_expression_tests): kTestAll / kTestNone for a reduced list, the dictionary bitmaps of a string column,
// in_prepare_kernel over the uploaded intervals of a numeric one. Every buffer belongs to `scratch`; *out_list_bytes
// counts the uploaded bitmap words or intervals.
static int prepare_in_tests(hyb_context* context, Table* table, const hyb_in_predicate* predicate, InForm form,
                            const std::vector<hyb_value>& bounds, DeviceScratch& scratch, ChunkTest** out_tests,
                            InList* out_list, uint64_t* out_list_bytes) {
  const uint32_t chunk_count = table->chunk_count();
  const DevSegment* column_segments = table->d_segments + size_t{predicate->column_id} * chunk_count;
  const int32_t data_type = table->column_types[predicate->column_id];
  const bool strings = data_type == HYB_TYPE_STRING;
  const bool negate = predicate->condition == HYB_PRED_NOT_IN;
  ChunkTest* tests = nullptr;
  HYB_TRY(scratch.alloc_array(chunk_count, &tests));
  *out_tests = tests;
  InList& list = *out_list;
  list = InList{};
  list.interval_count = 1;
  uint64_t& list_bytes = *out_list_bytes;
  list_bytes = 0;
  if (form != kInList) {

    std::vector<ChunkTest> host(chunk_count);
    for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
      host[chunk] = ChunkTest{};
      const bool rows = table->segments[size_t{chunk} * table->column_count + predicate->column_id].row_count > 0;
      host[chunk].mode = form == kInEveryRow && rows ? kTestAll : kTestNone;
    }
    if (chunk_count) {
      HYB_CUDA(cudaMemcpyAsync(tests, host.data(), sizeof(ChunkTest) * chunk_count, cudaMemcpyHostToDevice, context->stream));
    }
  } else if (strings) {
    void* bitmap_scratch = nullptr;
    uint64_t words = 0;
    const int status = prepare_bitmap_tests(context, table, predicate->column_id, predicate->dictionary_matches, tests,
                                            &bitmap_scratch, &words);
    scratch.adopt(bitmap_scratch);
    HYB_TRY(status);
    list_bytes = sizeof(uint32_t) * words;
  } else {
    if (data_type == HYB_TYPE_INT32) {
      list.compare = kInInt32;
      HYB_TRY(upload_intervals<int32_t>(context, bounds, &hyb_value::i32, scratch, list, &list_bytes));
    } else if (data_type == HYB_TYPE_INT64) {
      list.compare = kInInt64;
      HYB_TRY(upload_intervals<long long>(context, bounds, &hyb_value::i64, scratch, list, &list_bytes));
    } else if (data_type == HYB_TYPE_FLOAT32) {
      list.compare = kInFloat;
      HYB_TRY(upload_intervals<float>(context, bounds, &hyb_value::f32, scratch, list, &list_bytes));
    } else {
      list.compare = kInDouble;
      HYB_TRY(upload_intervals<double>(context, bounds, &hyb_value::f64, scratch, list, &list_bytes));
    }
    // bitmap words of the dictionary chunks, in case their value-IDs do not form one run
    std::vector<unsigned long long> word_offsets(std::max<uint32_t>(chunk_count, 1), 0);
    unsigned long long words = 0;
    for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
      const DevSegment& segment = table->segments[size_t{chunk} * table->column_count + predicate->column_id];
      word_offsets[chunk] = words;
      if (segment.encoding == HYB_ENC_DICTIONARY) words += (size_t{segment.dict_size} + 31) / 32;
    }
    uint32_t* bits = nullptr;
    unsigned long long* d_word_offsets = nullptr;
    if (words > 0) {
      HYB_TRY(scratch.alloc_array(words, &bits));
      HYB_TRY(scratch.alloc_array(word_offsets.size(), &d_word_offsets));
      HYB_CUDA(cudaMemcpyAsync(d_word_offsets, word_offsets.data(), sizeof(unsigned long long) * word_offsets.size(),
                               cudaMemcpyHostToDevice, context->stream));
    }
    if (chunk_count) {
      in_prepare_kernel<<<(chunk_count + 127) / 128, 128, 0, context->stream>>>(column_segments, chunk_count, list, negate,
                                                                                d_word_offsets, bits, tests);
      HYB_CUDA(cudaGetLastError());
    }
  }

  return HYB_OK;
}

// The predicate with every column NULL: what a NULL_ROW_ID of an outer join reads, and the value of a predicate that
// reads no column. One thread.
__global__ void expression_null_row_kernel(ExprProgram* program, uint32_t* out) {
  unsigned long long values[HYB_MAX_EXPRESSION_COLUMNS][8] = {};
  const uint32_t result = evaluate_predicate(*program, values, ~0ull, 1) & 1u;
  program->constant = result;
  *out = result;
}

// The predicate on a NULL_ROW_ID: every column NULL. One thread.
template <bool kOperands>
__global__ void expression_tests_null_row_kernel(const TestProgram* program, uint32_t* out) {
  unsigned long long low = 0, high = 0;
  for (uint32_t k = 0; k < program->test_count; ++k) set_test_mask(k, (program->null_row_tests >> k) & 1u, low, high);
  unsigned long long operands = 0;
  if constexpr (kOperands) {
    unsigned long long values[HYB_MAX_EXPRESSION_COLUMNS][8] = {};
    operands = operand_masks(*program->operands, program->operand_count, values, ~0ull, 1);
  }
  *out = combine_terms(*program, operands, low, high) & 1u;
}

// ---------------------------------------------------------------------------------------------------------------------
// Expression predicates (hyb_table_scan_expression): the host validates and types the term list and every operand
// program, numbers the distinct columns, and lays the predicate out as the device's ExprProgram (expression_scan.cuh).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int32_t kTypeNull = -1;  // a NULL literal: takes its sibling's type (expression_utils.cpp:172-205)

static int compile_operand(const Table* table, const hyb_expr_node* nodes, uint32_t count, ExprProgram& program,
                           uint32_t* column_ids, int32_t* out_type) {
  HYB_CHECK(count <= HYB_MAX_EXPR_NODES, HYB_ERR_UNSUPPORTED, "an operand holds more than HYB_MAX_EXPR_NODES nodes");
  HYB_CHECK(count >= 1, HYB_ERR_INVALID, "empty operand program");
  std::vector<int32_t> stack;
  for (uint32_t n = 0; n < count; ++n) {
    const hyb_expr_node& node = nodes[n];
    ExprNode& device = program.nodes[program.node_count++];
    device = ExprNode{};
    device.op = node.op;
    switch (node.op) {
      case HYB_EXPR_COLUMN: {
        HYB_CHECK(node.column_id < table->column_count, HYB_ERR_INVALID, "expression column out of range");
        const int32_t type = table->column_types[node.column_id];
        HYB_CHECK(type != HYB_TYPE_STRING, HYB_ERR_UNSUPPORTED, "string columns in expression predicates run on the CPU");
        uint32_t slot = 0;
        while (slot < program.column_count && column_ids[slot] != node.column_id) ++slot;
        if (slot == program.column_count) {
          HYB_CHECK(program.column_count < HYB_MAX_EXPRESSION_COLUMNS, HYB_ERR_UNSUPPORTED,
                    "an expression predicate reads more than HYB_MAX_EXPRESSION_COLUMNS columns");
          column_ids[slot] = node.column_id;
          program.column_types[slot] = type;
          ++program.column_count;
        }
        device.type = type;
        device.slot = slot;
        stack.push_back(type);
        break;
      }
      case HYB_EXPR_LITERAL:
        HYB_CHECK(node.literal_type != HYB_TYPE_STRING, HYB_ERR_UNSUPPORTED, "string literals run on the CPU");
        HYB_CHECK(node.literal_type >= HYB_TYPE_INT32 && node.literal_type <= HYB_TYPE_FLOAT64, HYB_ERR_INVALID,
                  "bad literal type");
        device.type = node.literal_type;
        device.literal = node.literal;
        stack.push_back(node.literal_type);
        break;
      case HYB_EXPR_NULL:
        device.type = HYB_TYPE_INT32;
        stack.push_back(kTypeNull);
        break;
      case HYB_EXPR_ADD:
      case HYB_EXPR_SUB:
      case HYB_EXPR_MUL:
      case HYB_EXPR_DIV:
      case HYB_EXPR_MOD: {
        HYB_CHECK(stack.size() >= 2, HYB_ERR_INVALID, "malformed expression: stack underflow");
        const int32_t b = stack.back();
        stack.pop_back();
        const int32_t a = stack.back();
        stack.pop_back();
        const int32_t type = a == kTypeNull ? b : b == kTypeNull ? a : expression_common_type(a, b);
        device.type = type == kTypeNull ? HYB_TYPE_INT32 : type;
        stack.push_back(type);
        break;
      }
      default:
        HYB_CHECK(false, HYB_ERR_INVALID, "bad expression op " + std::to_string(node.op));
    }
  }
  HYB_CHECK(stack.size() == 1, HYB_ERR_INVALID, "malformed expression: values left on the stack");
  *out_type = stack[0];
  return HYB_OK;
}

// Validates the postfix term list and compiles its operand leaves into `program`. tests == nullptr: the term list of
// hyb_table_scan_expression (operand leaves only) goes to program.terms; otherwise column-test leaves are accepted too
// and the list goes to *tests.
static int compile_expression(const Table* table, const hyb_expression_scan_predicate* predicate, ExprProgram& program,
                              uint32_t* column_ids, TestTerms* tests = nullptr) {
  HYB_CHECK(predicate->reserved == 0, HYB_ERR_INVALID, "hyb_expression_scan_predicate.reserved must be 0");
  HYB_CHECK(predicate->term_count > 0 && predicate->terms, HYB_ERR_INVALID, "an expression predicate needs terms");
  uint32_t leaves = 0, test_leaves = 0;
  for (uint32_t t = 0; t < predicate->term_count; ++t) {
    leaves += predicate->terms[t].kind == HYB_TERM_LEAF;
    test_leaves += predicate->terms[t].kind == HYB_TERM_SCAN || predicate->terms[t].kind == HYB_TERM_IN;
  }
  HYB_CHECK(leaves <= HYB_MAX_EXPRESSION_LEAVES, HYB_ERR_UNSUPPORTED,
            "an expression predicate holds more than HYB_MAX_EXPRESSION_LEAVES leaves");
  if (tests) {
    HYB_CHECK(test_leaves <= HYB_MAX_EXPRESSION_TESTS, HYB_ERR_UNSUPPORTED,
              "an expression predicate holds more than HYB_MAX_EXPRESSION_TESTS column-test leaves");
  }
  HYB_CHECK(predicate->term_count <= static_cast<uint32_t>(tests ? kTestMaxTerms : kExprMaxTerms), HYB_ERR_INVALID,
            "malformed term list: too many AND / OR nodes");
  int32_t* terms = tests ? tests->terms : program.terms;
  uint32_t depth = 0, leaf = 0, test = 0;
  for (uint32_t t = 0; t < predicate->term_count; ++t) {
    const hyb_expression_term& term = predicate->terms[t];
    HYB_CHECK(term.reserved == 0, HYB_ERR_INVALID, "hyb_expression_term.reserved must be 0");
    if (term.kind == HYB_TERM_AND || term.kind == HYB_TERM_OR) {
      HYB_CHECK(depth >= 2, HYB_ERR_INVALID, "malformed term list: AND / OR needs two selections");
      --depth;
      terms[t] = term.kind == HYB_TERM_AND ? kExprTermAnd : kExprTermOr;
      continue;
    }
    if (tests && (term.kind == HYB_TERM_SCAN || term.kind == HYB_TERM_IN)) {
      HYB_CHECK(term.condition == 0 && term.node_counts[0] == 0 && term.node_counts[1] == 0 && term.node_counts[2] == 0,
                HYB_ERR_INVALID, "a column-test leaf takes its predicate from hyb_expression_leaf_tests: condition and "
                                 "node_counts must be 0");
      tests->kinds[test] = term.kind;
      terms[t] = kExprTermTest + static_cast<int32_t>(test++);
      HYB_CHECK(++depth <= HYB_MAX_EXPRESSION_DEPTH, HYB_ERR_UNSUPPORTED,
                "more than HYB_MAX_EXPRESSION_DEPTH selections on the postfix stack");
      continue;
    }
    HYB_CHECK(term.kind == HYB_TERM_LEAF, HYB_ERR_INVALID, "bad term kind " + std::to_string(term.kind));
    const int32_t condition = term.condition;
    uint32_t operands = 0;
    if (condition >= HYB_PRED_EQUALS && condition <= HYB_PRED_GREATER_THAN_EQUALS) {
      operands = 2;
    } else if (condition >= HYB_PRED_BETWEEN_INCLUSIVE && condition <= HYB_PRED_BETWEEN_EXCLUSIVE) {
      operands = 3;
    } else if (condition == HYB_PRED_IS_NULL || condition == HYB_PRED_IS_NOT_NULL) {
      operands = 1;
    } else {
      HYB_CHECK(condition < HYB_PRED_IN || condition > HYB_PRED_NOT_LIKE_INSENSITIVE, HYB_ERR_UNSUPPORTED,
                "IN and LIKE leaves in expression predicates run on the CPU");
      HYB_CHECK(false, HYB_ERR_INVALID, "bad leaf condition " + std::to_string(condition));
    }
    ExprLeaf& device = program.leaves[leaf];
    device = ExprLeaf{};
    device.condition = condition;
    for (uint32_t o = 0; o < 3; ++o) {
      if (o >= operands) {
        HYB_CHECK(term.node_counts[o] == 0, HYB_ERR_INVALID, "unused operand programs must be empty");
        continue;
      }
      int32_t type = 0;
      device.begin[o] = static_cast<uint16_t>(program.node_count);
      HYB_TRY(compile_operand(table, term.operands[o], term.node_counts[o], program, column_ids, &type));
      device.count[o] = static_cast<uint16_t>(term.node_counts[o]);
    }
    terms[t] = static_cast<int32_t>(leaf++);
    ++depth;
    if (tests) {
      HYB_CHECK(depth <= HYB_MAX_EXPRESSION_DEPTH, HYB_ERR_UNSUPPORTED,
                "more than HYB_MAX_EXPRESSION_DEPTH selections on the postfix stack");
    }
  }
  HYB_CHECK(depth == 1, HYB_ERR_INVALID, "malformed term list: more than one selection left");
  if (tests) {
    tests->count = test;
    tests->operand_count = leaf;
  } else {
    program.term_count = predicate->term_count;
  }
  return HYB_OK;
}

// The number of HYB_TERM_SCAN / HYB_TERM_IN terms, checked against `leaf_tests`.
static int count_test_terms(const hyb_expression_scan_predicate* predicate, const hyb_expression_leaf_tests* leaf_tests,
                            uint32_t* out_scans, uint32_t* out_ins) {
  uint32_t scan_terms = 0, in_terms = 0;
  for (uint32_t t = 0; predicate->terms && t < predicate->term_count; ++t) {
    scan_terms += predicate->terms[t].kind == HYB_TERM_SCAN;
    in_terms += predicate->terms[t].kind == HYB_TERM_IN;
  }
  HYB_CHECK(scan_terms == leaf_tests->scan_count && in_terms == leaf_tests->in_count, HYB_ERR_INVALID,
            "hyb_expression_leaf_tests counts differ from the HYB_TERM_SCAN / HYB_TERM_IN terms");
  HYB_CHECK((scan_terms == 0 || leaf_tests->scans) && (in_terms == 0 || leaf_tests->ins), HYB_ERR_INVALID,
            "NULL hyb_expression_leaf_tests.scans / ins");
  *out_scans = scan_terms;
  *out_ins = in_terms;
  return HYB_OK;
}

int compile_expression_tree(const Table* table, const hyb_expression_scan_predicate* predicate,
                            const hyb_expression_leaf_tests* leaf_tests, ExpressionTree* tree) {
  uint32_t scan_terms = 0, in_terms = 0;
  if (leaf_tests) HYB_TRY(count_test_terms(predicate, leaf_tests, &scan_terms, &in_terms));
  tree->leaf_tests = leaf_tests;
  tree->term_count = predicate->term_count;
  if (scan_terms + in_terms == 0) {
    // operand leaves only: hyb_table_scan_expression's rules, laid out as a tree without test leaves
    HYB_TRY(compile_expression(table, predicate, tree->program, tree->column_ids));
    std::copy(tree->program.terms, tree->program.terms + predicate->term_count, tree->terms.terms);
    for (uint32_t t = 0; t < predicate->term_count; ++t) tree->terms.operand_count += predicate->terms[t].kind == HYB_TERM_LEAF;
    return HYB_OK;
  }
  HYB_TRY(compile_expression(table, predicate, tree->program, tree->column_ids, &tree->terms));
  for (uint32_t k = 0; k < scan_terms; ++k) {
    const hyb_scan_predicate& scan = leaf_tests->scans[k];
    HYB_CHECK(scan.column_id < table->column_count, HYB_ERR_INVALID, "predicate column out of range");
    HYB_CHECK(scan.condition != HYB_PRED_IN && scan.condition != HYB_PRED_NOT_IN, HYB_ERR_INVALID,
              "an IN / NOT IN leaf is a HYB_TERM_IN term");
  }
  tree->forms.assign(in_terms, kInList);
  tree->bounds.assign(in_terms, {});
  for (uint32_t k = 0; k < in_terms; ++k) {
    HYB_TRY(check_in_predicate(table, &leaf_tests->ins[k], &tree->forms[k], tree->bounds[k]));
  }
  return HYB_OK;
}

int upload_expression_tree(hyb_context* context, Table* table, ExpressionTree& tree, DeviceScratch& scratch) {
  const uint32_t chunk_count = table->chunk_count();
  TestProgram* host = &tree.host;
  *host = TestProgram{};
  host->test_count = tree.terms.count;
  host->operand_count = tree.terms.operand_count;
  host->term_count = tree.term_count;
  std::copy(tree.terms.terms, tree.terms.terms + tree.term_count, host->terms);
  uint32_t* test_columns = tree.test_columns;
  uint64_t& uploaded_bytes = tree.uploaded_bytes;
  uint32_t& launches = tree.launches;
  uploaded_bytes = 0;
  launches = 0;
  const hyb_expression_leaf_tests* leaf_tests = tree.leaf_tests;
  for (uint32_t k = 0, scan = 0, in = 0; k < tree.terms.count; ++k) {
    TestLeaf& leaf = host->leaves[k];
    ChunkTest* tests = nullptr;
    uint32_t column_id = 0;
    uint64_t bytes = 0;
    if (tree.terms.kinds[k] == HYB_TERM_SCAN) {
      const hyb_scan_predicate& predicate_k = leaf_tests->scans[scan++];
      void* bounds_scratch = nullptr;
      const int status = prepare_chunk_tests(context, table, &predicate_k, &tests, &bounds_scratch, &bytes);
      scratch.adopt(tests);
      scratch.adopt(bounds_scratch);
      HYB_TRY(status);
      column_id = predicate_k.column_id;
      if (predicate_k.condition == HYB_PRED_IS_NULL) host->null_row_tests |= 1u << k;
      launches += !is_like_condition(predicate_k.condition) && chunk_count > 0;  // scan_prepare_kernel
    } else {
      const hyb_in_predicate& predicate_k = leaf_tests->ins[in];
      HYB_TRY(prepare_in_tests(context, table, &predicate_k, tree.forms[in], tree.bounds[in], scratch, &tests, &leaf.list,
                               &bytes));
      column_id = predicate_k.column_id;
      if (tree.forms[in] == kInEveryRow) host->null_row_tests |= 1u << k;
      launches += tree.forms[in] == kInList && table->column_types[column_id] != HYB_TYPE_STRING && chunk_count > 0;  // in_prepare_kernel
      ++in;
    }
    leaf.tests = tests;
    uploaded_bytes += bytes + sizeof(ChunkTest) * chunk_count;
    uint32_t slot = 0;
    while (slot < host->column_count && test_columns[slot] != column_id) ++slot;
    if (slot == host->column_count) {
      test_columns[slot] = column_id;
      host->columns[slot] = table->d_segments + size_t{column_id} * chunk_count;
      ++host->column_count;
    }
    leaf.column = slot;
  }
  // evaluation order: the leaves of one column back to back, in postfix order within a column
  for (uint32_t c = 0, n = 0; c < host->column_count; ++c) {
    for (uint32_t k = 0; k < host->test_count; ++k) {
      if (host->leaves[k].column == c) host->order[n++] = static_cast<uint8_t>(k);
    }
    host->column_end[c] = static_cast<uint8_t>(n);
  }
  if (tree.operands()) {
    ExprProgram& program = tree.program;
    for (uint32_t c = 0; c < program.column_count; ++c) {
      program.columns[c] = table->d_segments + size_t{tree.column_ids[c]} * chunk_count;
    }
    const size_t program_bytes = offsetof(ExprProgram, nodes) + sizeof(ExprNode) * program.node_count;
    void* d_program = nullptr;
    HYB_TRY(scratch.alloc(program_bytes, &d_program));
    // pageable source: the copy is staged before cudaMemcpyAsync returns
    HYB_CUDA(cudaMemcpyAsync(d_program, &program, program_bytes, cudaMemcpyHostToDevice, context->stream));
    host->operands = static_cast<const ExprProgram*>(d_program);
    uploaded_bytes += program_bytes;
  }
  TestProgram* d_tests = nullptr;
  HYB_TRY(scratch.alloc_array(1, &d_tests));
  HYB_CUDA(cudaMemcpyAsync(d_tests, host, sizeof(TestProgram), cudaMemcpyHostToDevice, context->stream));
  tree.device = d_tests;
  uploaded_bytes += sizeof(TestProgram);
  return HYB_OK;
}

std::string expression_tree_signature(const ExpressionTree& tree) {
  std::string signature;
  const auto add = [&](const void* data, size_t bytes) { signature.append(static_cast<const char*>(data), bytes); };
  const ExprProgram& program = tree.program;
  add(&tree.term_count, sizeof(tree.term_count));
  add(tree.terms.terms, sizeof(int32_t) * tree.term_count);
  add(&program.node_count, sizeof(program.node_count));
  add(&program.column_count, sizeof(program.column_count));
  add(tree.column_ids, sizeof(uint32_t) * program.column_count);
  add(program.leaves, sizeof(ExprLeaf) * tree.terms.operand_count);
  add(program.nodes, sizeof(ExprNode) * program.node_count);
  for (uint32_t k = 0, scan = 0, in = 0; k < tree.terms.count; ++k) {
    const bool is_scan = tree.terms.kinds[k] == HYB_TERM_SCAN;
    const uint32_t column = is_scan ? tree.leaf_tests->scans[scan].column_id : tree.leaf_tests->ins[in].column_id;
    const int32_t condition = is_scan ? tree.leaf_tests->scans[scan++].condition : tree.leaf_tests->ins[in++].condition;
    add(&tree.terms.kinds[k], sizeof(int32_t));
    add(&column, sizeof(column));
    add(&condition, sizeof(condition));
  }
  return signature;
}

// The table and the optional input_filter of a scan call (context->mutex held).
static int find_scan_inputs(hyb_context* context, hyb_table_t table_handle, hyb_pos_list_t input_filter, Table** out_table,
                            PosList** out_filter) {
  *out_table = find_table(context, table_handle);
  HYB_CHECK(*out_table, HYB_ERR_NOT_FOUND, "unknown table handle");
  *out_filter = nullptr;
  if (input_filter) {
    *out_filter = find_pos_list(context, input_filter);
    HYB_CHECK(*out_filter, HYB_ERR_NOT_FOUND, "unknown input_filter handle");
    HYB_CHECK((*out_filter)->table == table_handle, HYB_ERR_INVALID, "input_filter belongs to a different table");
  }
  return HYB_OK;
}

// Launches the one-thread `kernel`: the predicate on a NULL_ROW_ID, every column NULL. With `read`, waits for its answer.
template <typename Program>
static int probe_null_row(hyb_context* context, DeviceScratch& scratch, void (*kernel)(Program, uint32_t*), Program program,
                          bool read, bool* out_matches) {
  uint32_t* d_matches = nullptr;
  HYB_TRY(scratch.alloc_array(1, &d_matches));
  kernel<<<1, 1, 0, context->stream>>>(program, d_matches);
  HYB_CUDA(cudaGetLastError());
  uint32_t matches = 0;
  if (read) {
    HYB_CUDA(cudaMemcpyAsync(&matches, d_matches, sizeof(uint32_t), cudaMemcpyDeviceToHost, context->stream));
    HYB_CUDA(cudaStreamSynchronize(context->stream));
  }
  *out_matches = matches != 0;
  return HYB_OK;
}

}  // namespace hyb

using namespace hyb;

extern "C" {

int hyb_table_scan(hyb_context* context, hyb_table_t table_handle, const hyb_scan_predicate* predicate,
                   hyb_pos_list_t input_filter, hyb_pos_list_t* out_pos_list) {
  HYB_CHECK(context && predicate && out_pos_list, HYB_ERR_INVALID, "NULL argument");
  *out_pos_list = 0;
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  Table* table = nullptr;
  PosList* filter = nullptr;
  HYB_TRY(find_scan_inputs(context, table_handle, input_filter, &table, &filter));
  HYB_TRY(sync_table_descriptors(context, table));

  timing_begin(context);
  DeviceScratch scratch(context);
  ChunkTest* tests = nullptr;
  void* bounds_scratch = nullptr;
  HYB_TRY(prepare_chunk_tests(context, table, predicate, &tests, &bounds_scratch));
  scratch.adopt(tests);
  scratch.adopt(bounds_scratch);
  ScanPlan plan{};
  plan.row_column = predicate->column_id;
  plan.tests = tests;
  plan.prepare_launches = 1;  // prepared_bytes stays 0: this call's stats have never counted the uploaded value_id_bounds
  plan.column_bytes = column_bytes_per_launch(table, predicate->column_id);
  plan.null_row_matches = predicate->condition == HYB_PRED_IS_NULL;
  return run_scan<ColumnRows>(context, table_handle, table, filter, plan, ColumnRows::Extra{}, out_pos_list);
}

int hyb_table_scan_columns(hyb_context* context, hyb_table_t table_handle, const hyb_column_scan_predicate* predicate,
                           hyb_pos_list_t input_filter, hyb_pos_list_t* out_pos_list) {
  HYB_CHECK(context && predicate && out_pos_list, HYB_ERR_INVALID, "NULL argument");
  *out_pos_list = 0;
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  Table* table = nullptr;
  PosList* filter = nullptr;
  HYB_TRY(find_scan_inputs(context, table_handle, input_filter, &table, &filter));
  const int32_t condition = predicate->condition;
  HYB_CHECK(!is_like_condition(condition), HYB_ERR_UNSUPPORTED, "column-vs-column LIKE is not on the GPU path");
  HYB_CHECK(condition >= HYB_PRED_EQUALS && condition <= HYB_PRED_GREATER_THAN_EQUALS, HYB_ERR_INVALID,
            "column-vs-column scans take =, !=, <, <=, >, >= (condition " + std::to_string(condition) + ")");
  HYB_CHECK(predicate->left_column_id < table->column_count && predicate->right_column_id < table->column_count,
            HYB_ERR_INVALID, "column-vs-column scan column out of range");
  HYB_CHECK(predicate->reserved == 0, HYB_ERR_INVALID, "hyb_column_scan_predicate.reserved must be 0");
  const int32_t left_type = table->column_types[predicate->left_column_id];
  const int32_t right_type = table->column_types[predicate->right_column_id];
  const bool strings = left_type == HYB_TYPE_STRING;
  // column_vs_column_table_scan_impl.cpp: Fail("Trying to compare strings and non-strings")
  HYB_CHECK(strings == (right_type == HYB_TYPE_STRING), HYB_ERR_INVALID, "Trying to compare strings and non-strings");
  HYB_CHECK(!strings || predicate->right_in_left, HYB_ERR_INVALID,
            "string column-vs-column scans need the host-built right_in_left words (hyb_dictionary_translate)");
  HYB_TRY(sync_table_descriptors(context, table));

  timing_begin(context);
  DeviceScratch scratch(context);
  PairTest* tests = nullptr;
  uint64_t translation_words = 0;
  HYB_TRY(prepare_pair_tests(context, table, predicate, strings ? kCompareInt64 : pair_compare(left_type, right_type),
                             scratch, &tests, &translation_words));
  ScanPlan plan{};
  plan.row_column = predicate->left_column_id;
  plan.prepare_launches = 1;
  plan.prepared_bytes = sizeof(uint32_t) * translation_words;
  plan.column_bytes = column_bytes_per_launch(table, predicate->left_column_id) +
                      column_bytes_per_launch(table, predicate->right_column_id);
  const PairRows::Extra extra{table->d_segments + size_t{predicate->right_column_id} * table->chunk_count(), tests};
  return run_scan<PairRows>(context, table_handle, table, filter, plan, extra, out_pos_list);
}

int hyb_table_scan_in(hyb_context* context, hyb_table_t table_handle, const hyb_in_predicate* predicate,
                      hyb_pos_list_t input_filter, hyb_pos_list_t* out_pos_list) {
  HYB_CHECK(context && predicate && out_pos_list, HYB_ERR_INVALID, "NULL argument");
  *out_pos_list = 0;
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  Table* table = nullptr;
  PosList* filter = nullptr;
  HYB_TRY(find_scan_inputs(context, table_handle, input_filter, &table, &filter));
  InForm form;
  std::vector<hyb_value> bounds;
  HYB_TRY(check_in_predicate(table, predicate, &form, bounds));
  HYB_TRY(sync_table_descriptors(context, table));

  timing_begin(context);
  DeviceScratch scratch(context);
  ChunkTest* tests = nullptr;
  InList list{};
  uint64_t list_bytes = 0;
  HYB_TRY(prepare_in_tests(context, table, predicate, form, bounds, scratch, &tests, &list, &list_bytes));
  ScanPlan plan{};
  plan.row_column = predicate->column_id;
  plan.tests = tests;
  plan.prepare_launches = 1;
  plan.prepared_bytes = list_bytes;
  plan.column_bytes = column_bytes_per_launch(table, predicate->column_id);
  // a NULL_ROW_ID reads as NULL: it matches only where NULL rows do, i.e. NOT IN over a list without a compatible element
  plan.null_row_matches = form == kInEveryRow;
  return run_scan<InRows>(context, table_handle, table, filter, plan, list, out_pos_list);
}

int hyb_table_scan_expression(hyb_context* context, hyb_table_t table_handle, const hyb_expression_scan_predicate* predicate,
                              hyb_pos_list_t input_filter, hyb_pos_list_t* out_pos_list) {
  HYB_CHECK(context && predicate && out_pos_list, HYB_ERR_INVALID, "NULL argument");
  *out_pos_list = 0;
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  Table* table = nullptr;
  PosList* filter = nullptr;
  HYB_TRY(find_scan_inputs(context, table_handle, input_filter, &table, &filter));
  auto program = std::make_unique<ExprProgram>();
  uint32_t column_ids[HYB_MAX_EXPRESSION_COLUMNS] = {};
  HYB_TRY(compile_expression(table, predicate, *program, column_ids));
  HYB_TRY(sync_table_descriptors(context, table));

  timing_begin(context);
  DeviceScratch scratch(context);
  const uint32_t chunk_count = table->chunk_count();
  for (uint32_t c = 0; c < program->column_count; ++c) {
    program->columns[c] = table->d_segments + size_t{column_ids[c]} * chunk_count;
  }
  const size_t program_bytes = offsetof(ExprProgram, nodes) + sizeof(ExprNode) * program->node_count;
  void* d_program = nullptr;
  HYB_TRY(scratch.alloc(program_bytes, &d_program));
  // pageable source: the copy is staged before cudaMemcpyAsync returns
  HYB_CUDA(cudaMemcpyAsync(d_program, program.get(), program_bytes, cudaMemcpyHostToDevice, context->stream));
  ScanPlan plan{};
  // every column NULL: the value of a NULL_ROW_ID, and of every row when the predicate reads no column (the kernel stores
  // it in the program, so it runs unfiltered too)
  HYB_TRY(probe_null_row(context, scratch, expression_null_row_kernel, static_cast<ExprProgram*>(d_program), filter != nullptr,
                         &plan.null_row_matches));
  // the first column read (any column when none is): ExprRows takes the chunks' row counts from its segments
  plan.row_column = program->column_count ? column_ids[0] : 0;
  plan.prepare_launches = 1;  // expression_null_row_kernel
  plan.prepared_bytes = program_bytes;
  for (uint32_t c = 0; c < program->column_count; ++c) plan.column_bytes += column_bytes_per_launch(table, column_ids[c]);
  return run_scan<ExprRows>(context, table_handle, table, filter, plan, static_cast<const ExprProgram*>(d_program),
                            out_pos_list);
}

int hyb_table_scan_expression_tests(hyb_context* context, hyb_table_t table_handle,
                                    const hyb_expression_scan_predicate* predicate, const hyb_expression_leaf_tests* leaf_tests,
                                    hyb_pos_list_t input_filter, hyb_pos_list_t* out_pos_list) {
  HYB_CHECK(context && predicate && leaf_tests && out_pos_list, HYB_ERR_INVALID, "NULL argument");
  *out_pos_list = 0;
  uint32_t scan_terms = 0, in_terms = 0;
  HYB_TRY(count_test_terms(predicate, leaf_tests, &scan_terms, &in_terms));
  // operand leaves only: today's predicate, today's kernel
  if (scan_terms + in_terms == 0) return hyb_table_scan_expression(context, table_handle, predicate, input_filter, out_pos_list);

  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  Table* table = nullptr;
  PosList* filter = nullptr;
  HYB_TRY(find_scan_inputs(context, table_handle, input_filter, &table, &filter));
  // host checks of every leaf before anything runs
  auto tree = std::make_unique<ExpressionTree>();
  HYB_TRY(compile_expression_tree(table, predicate, leaf_tests, tree.get()));
  HYB_TRY(sync_table_descriptors(context, table));

  timing_begin(context);
  DeviceScratch scratch(context);
  HYB_TRY(upload_expression_tree(context, table, *tree, scratch));
  const bool operands = tree->operands();
  ScanPlan plan{};
  plan.prepare_launches = tree->launches;
  if (filter) {
    HYB_TRY(probe_null_row(context, scratch,
                           operands ? expression_tests_null_row_kernel<true> : expression_tests_null_row_kernel<false>,
                           tree->device, true, &plan.null_row_matches));
    ++plan.prepare_launches;
  }
  // the first test leaf's column: TestRows takes the chunks' row counts from its segments
  plan.row_column = tree->test_columns[0];
  plan.prepared_bytes = tree->uploaded_bytes;
  // every distinct column once, whether an operand or a test leaf reads it
  const uint32_t* test_columns = tree->test_columns;
  const uint32_t test_column_count = tree->host.column_count;
  for (uint32_t c = 0; c < test_column_count; ++c) plan.column_bytes += column_bytes_per_launch(table, test_columns[c]);
  for (uint32_t c = 0; c < tree->program.column_count; ++c) {
    const uint32_t column_id = tree->column_ids[c];
    if (std::find(test_columns, test_columns + test_column_count, column_id) == test_columns + test_column_count) {
      plan.column_bytes += column_bytes_per_launch(table, column_id);
    }
  }
  HYB_TRY(operands ? run_scan<TestRows<true>>(context, table_handle, table, filter, plan, tree->device, out_pos_list)
                   : run_scan<TestRows<false>>(context, table_handle, table, filter, plan, tree->device, out_pos_list));
  context->timing.stats.path = operands ? 2 : 1;
  return HYB_OK;
}

static int ensure_pos_list_host(hyb_context* context, PosList* list) {
  if (list->host_valid) return HYB_OK;
  list->h_chunk_offsets.assign(size_t{list->chunk_count} + 1, 0);
  std::vector<uint64_t> ends(size_t{list->chunk_count} + 1);
  HYB_CUDA(cudaMemcpyAsync(ends.data(), list->d_chunk_end, sizeof(uint64_t) * ends.size(), cudaMemcpyDeviceToHost,
                           context->stream));
  HYB_CUDA(cudaStreamSynchronize(context->stream));
  uint64_t running = 0;
  for (uint32_t chunk = 0; chunk < list->chunk_count; ++chunk) {
    list->h_chunk_offsets[chunk] = running;
    if (ends[chunk] != ~uint64_t{0}) running = ends[chunk];
  }
  list->h_chunk_offsets[list->chunk_count] = running;
  list->host_valid = true;
  return HYB_OK;
}

int hyb_pos_list_info(hyb_context* context, hyb_pos_list_t handle, uint64_t* out_total, uint32_t* out_chunk_count) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* list = find_pos_list(context, handle);
  HYB_CHECK(list, HYB_ERR_NOT_FOUND, "unknown pos list handle");
  HYB_TRY(ensure_pos_list_host(context, list));
  if (out_total) *out_total = list->h_chunk_offsets.back();
  if (out_chunk_count) *out_chunk_count = list->chunk_count;
  return HYB_OK;
}

int hyb_pos_list_chunk_offsets(hyb_context* context, hyb_pos_list_t handle, uint64_t* out_chunk_offsets) {
  HYB_CHECK(context && out_chunk_offsets, HYB_ERR_INVALID, "NULL argument");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* list = find_pos_list(context, handle);
  HYB_CHECK(list, HYB_ERR_NOT_FOUND, "unknown pos list handle");
  HYB_TRY(ensure_pos_list_host(context, list));
  std::copy(list->h_chunk_offsets.begin(), list->h_chunk_offsets.end(), out_chunk_offsets);
  return HYB_OK;
}

int hyb_pos_list_copy(hyb_context* context, hyb_pos_list_t handle, uint64_t begin, uint64_t count,
                      hyb_row_id* out_row_ids) {
  HYB_CHECK(context && (out_row_ids || count == 0), HYB_ERR_INVALID, "NULL argument");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* list = find_pos_list(context, handle);
  HYB_CHECK(list, HYB_ERR_NOT_FOUND, "unknown pos list handle");
  HYB_TRY(ensure_pos_list_host(context, list));
  HYB_CHECK(begin + count <= list->h_chunk_offsets.back(), HYB_ERR_INVALID, "range exceeds the pos list");
  if (count) {
    HYB_CUDA(cudaMemcpyAsync(out_row_ids, list->d_row_ids + begin, sizeof(hyb_row_id) * count, cudaMemcpyDeviceToHost,
                             context->stream));
    HYB_CUDA(cudaStreamSynchronize(context->stream));
  }
  return HYB_OK;
}

int hyb_pos_list_device_ptr(hyb_context* context, hyb_pos_list_t handle, void** out_device_row_ids) {
  HYB_CHECK(context && out_device_row_ids, HYB_ERR_INVALID, "NULL argument");
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* list = find_pos_list(context, handle);
  HYB_CHECK(list, HYB_ERR_NOT_FOUND, "unknown pos list handle");
  *out_device_row_ids = list->d_row_ids;
  return HYB_OK;
}

int hyb_pos_list_free(hyb_context* context, hyb_pos_list_t handle) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto it = context->pos_lists.find(handle);
  HYB_CHECK(it != context->pos_lists.end(), HYB_ERR_NOT_FOUND, "unknown pos list handle");
  context->pos_lists.erase(it);
  return HYB_OK;
}

}  // extern "C"
