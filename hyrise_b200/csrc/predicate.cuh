// Per-chunk predicate tests shared by TableScan and the fused predicates of AggregateHash.
#pragma once

#include "device_utils.cuh"
#include "internal.hpp"

namespace hyb {

enum ChunkTestMode : uint32_t {
  kTestNone = 0,        // no row matches: skip the chunk's bytes
  kTestIdRange = 1,     // dictionary value-ID range
  kTestInt = 2,         // typed integer range (ValueSegment<int32/int64>, FrameOfReference)
  kTestFloat = 3,       // typed floating-point range (ValueSegment<float/double>)
  kTestNull = 4,        // IS NULL / IS NOT NULL on a null vector
  kTestIdSet = 5,       // dictionary value-ID set (LIKE): match iff value_id < dict_size and its bit in id_bits is set
  kTestInList = 6,      // [NOT] IN on a Value / FrameOfReference segment: the list's intervals (in_list.cuh)
  kTestAll = 7          // every row, NULL rows included (NOT IN over a list without a compatible element)
};

struct ChunkTest {
  uint32_t mode;
  uint32_t negate;      // NotEquals: match iff outside the range and not NULL
  uint32_t id_lo;       // kTestIdRange: match iff (value_id - id_lo) < id_span
  uint32_t id_span;
  union {
    long long int_lo;         // kTestInt: inclusive bounds
    const uint32_t* id_bits;  // kTestIdSet: device copy of the chunk's match bitmap (bit i & 31 of word i >> 5)
  };
  long long int_hi;
  double float_lo;      // kTestFloat
  double float_hi;
  uint32_t float_lo_inclusive;
  uint32_t float_hi_inclusive;
  uint32_t want_null;   // kTestNull: 1 = IS NULL, 0 = IS NOT NULL
  uint32_t pad;
};
static_assert(sizeof(ChunkTest) == 64, "scan_bulk_kernel copies a test as 4 x uint4");

__host__ __device__ __forceinline__ bool is_like_condition(int32_t condition) {
  return condition >= HYB_PRED_LIKE && condition <= HYB_PRED_NOT_LIKE_INSENSITIVE;
}


// Builds the per-chunk tests (scan.cu): on the device from value-ID bounds or literals, on the host from the dictionary
// match bitmaps of a LIKE predicate. Caller frees *out_tests and *out_bounds_scratch with device_free.
int prepare_chunk_tests(hyb_context* context, Table* table, const hyb_scan_predicate* predicate, ChunkTest** out_tests,
                        void** out_bounds_scratch);

// LIKE on a dictionary segment: value-ID `code` matches iff it is not the NULL id and its bitmap bit is set. The bitmap
// (<= 8 KB for 65 535-entry dictionaries) is gathered through L1; a tile never straddles chunks, so a CTA reads one
// chunk's bitmap. DESIGN.md §3.1 gives the measured cost against a value-ID range scan of the same selectivity.
__device__ __forceinline__ bool id_set_contains(const uint32_t* bits, uint32_t dict_size, uint32_t code) {
  return code < dict_size && ((__ldg(bits + (code >> 5)) >> (code & 31u)) & 1u);
}

// ---------------------------------------------------------------------------------------------------------------------
// Predicate evaluation for 8 consecutive rows of one segment. Returns a bit mask (bit j = row0 + j matches).
// All control flow depends on per-chunk values only, so it is uniform across a CTA (one tile = one chunk).
// ---------------------------------------------------------------------------------------------------------------------
// have_raw / raw: the segment's code vector for these rows if the caller loaded it early (load_raw_codes8).
__device__ __forceinline__ uint32_t evaluate8(const DevSegment& segment, const ChunkTest& test, uint32_t row0,
                                              bool have_raw = false, uint4 raw = uint4{0u, 0u, 0u, 0u}) {
  const uint32_t rows = segment.row_count;
  const uint32_t valid = rows - row0 >= 8 ? 0xFFu : ((1u << (rows - row0)) - 1u);
  uint32_t mask = 0;
  switch (test.mode) {
    case kTestIdRange: {
      uint32_t codes[8];
      codes8(segment, row0, have_raw, raw, codes);
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
    }
    case kTestIdSet: {
      uint32_t codes[8];
      codes8(segment, row0, have_raw, raw, codes);
#pragma unroll
      for (int j = 0; j < 8; ++j) mask |= id_set_contains(test.id_bits, segment.dict_size, codes[j]) ? (1u << j) : 0u;
      break;
    }
    case kTestInt: {
      long long values[8];
      if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) {
        uint32_t codes[8];
        codes8(segment, row0, have_raw, raw, codes);
        const int32_t minimum = __ldg(static_cast<const int32_t*>(segment.values) + row0 / HYB_FOR_BLOCK_SIZE);
#pragma unroll
        for (int j = 0; j < 8; ++j) values[j] = static_cast<int32_t>(static_cast<uint32_t>(minimum) + codes[j]);
      } else if (segment.data_type == HYB_TYPE_INT32) {
        const uint4 a = ld_stream_v4(static_cast<const int32_t*>(segment.values) + row0);
        const uint4 b = ld_stream_v4(static_cast<const int32_t*>(segment.values) + row0 + 4);
        values[0] = static_cast<int32_t>(a.x);
        values[1] = static_cast<int32_t>(a.y);
        values[2] = static_cast<int32_t>(a.z);
        values[3] = static_cast<int32_t>(a.w);
        values[4] = static_cast<int32_t>(b.x);
        values[5] = static_cast<int32_t>(b.y);
        values[6] = static_cast<int32_t>(b.z);
        values[7] = static_cast<int32_t>(b.w);
      } else {
        const auto* base = static_cast<const long long*>(segment.values) + row0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint4 v = ld_stream_v4(base + 2 * j);
          values[2 * j] = static_cast<long long>((static_cast<unsigned long long>(v.y) << 32) | v.x);
          values[2 * j + 1] = static_cast<long long>((static_cast<unsigned long long>(v.w) << 32) | v.z);
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const bool inside = values[j] >= test.int_lo && values[j] <= test.int_hi;
        mask |= (inside != static_cast<bool>(test.negate)) ? (1u << j) : 0u;
      }
      mask &= ~load_nulls8(segment.nulls, row0);
      break;
    }
    case kTestFloat: {
      double values[8];
      if (segment.data_type == HYB_TYPE_FLOAT32) {
        const uint4 a = ld_stream_v4(static_cast<const float*>(segment.values) + row0);
        const uint4 b = ld_stream_v4(static_cast<const float*>(segment.values) + row0 + 4);
        values[0] = __uint_as_float(a.x);
        values[1] = __uint_as_float(a.y);
        values[2] = __uint_as_float(a.z);
        values[3] = __uint_as_float(a.w);
        values[4] = __uint_as_float(b.x);
        values[5] = __uint_as_float(b.y);
        values[6] = __uint_as_float(b.z);
        values[7] = __uint_as_float(b.w);
      } else {
        const auto* base = static_cast<const double*>(segment.values) + row0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint4 v = ld_stream_v4(base + 2 * j);
          values[2 * j] = __longlong_as_double(static_cast<long long>((static_cast<unsigned long long>(v.y) << 32) | v.x));
          values[2 * j + 1] =
              __longlong_as_double(static_cast<long long>((static_cast<unsigned long long>(v.w) << 32) | v.z));
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const bool above = test.float_lo_inclusive ? values[j] >= test.float_lo : values[j] > test.float_lo;
        const bool below = test.float_hi_inclusive ? values[j] <= test.float_hi : values[j] < test.float_hi;
        mask |= ((above && below) != static_cast<bool>(test.negate)) ? (1u << j) : 0u;
      }
      mask &= ~load_nulls8(segment.nulls, row0);
      break;
    }
    case kTestNull: {
      const uint32_t nulls = load_nulls8(segment.nulls, row0);
      mask = test.want_null ? nulls : ~nulls;
      break;
    }
    default:
      break;
  }
  return mask & valid;
}

__device__ __forceinline__ bool evaluate1(const DevSegment& segment, const ChunkTest& test, uint32_t row) {
  switch (test.mode) {
    case kTestIdRange: {
      const uint32_t code = load_code1(segment.av, segment.vector_type, segment.bit_width, row);
      const bool inside = (code - test.id_lo) < test.id_span;
      return test.negate ? (!inside && code < segment.dict_size) : inside;
    }
    case kTestIdSet:
      return id_set_contains(test.id_bits, segment.dict_size,
                             load_code1(segment.av, segment.vector_type, segment.bit_width, row));
    case kTestInt: {
      if (segment.nulls && segment.nulls[row]) return false;
      long long value;
      if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) {
        const uint32_t code = load_code1(segment.av, segment.vector_type, segment.bit_width, row);
        const int32_t minimum = __ldg(static_cast<const int32_t*>(segment.values) + row / HYB_FOR_BLOCK_SIZE);
        value = static_cast<int32_t>(static_cast<uint32_t>(minimum) + code);
      } else if (segment.data_type == HYB_TYPE_INT32) {
        value = __ldg(static_cast<const int32_t*>(segment.values) + row);
      } else {
        value = __ldg(static_cast<const long long*>(segment.values) + row);
      }
      const bool inside = value >= test.int_lo && value <= test.int_hi;
      return inside != static_cast<bool>(test.negate);
    }
    case kTestFloat: {
      if (segment.nulls && segment.nulls[row]) return false;
      const double value = segment.data_type == HYB_TYPE_FLOAT32
                               ? static_cast<double>(__ldg(static_cast<const float*>(segment.values) + row))
                               : __ldg(static_cast<const double*>(segment.values) + row);
      const bool above = test.float_lo_inclusive ? value >= test.float_lo : value > test.float_lo;
      const bool below = test.float_hi_inclusive ? value <= test.float_hi : value < test.float_hi;
      return (above && below) != static_cast<bool>(test.negate);
    }
    case kTestNull: {
      const bool is_null = segment.nulls && segment.nulls[row];
      return test.want_null ? is_null : !is_null;
    }
    default:
      return false;
  }
}


}  // namespace hyb
