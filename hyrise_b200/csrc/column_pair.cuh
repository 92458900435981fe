// Column-vs-column predicate tests (`left <op> right` in one row), used by the TableScan pipelines of scan.cu; JoinHash's
// secondary predicates (join.cu) compare a build row with a probe row through decode1 and compare1.
//
// Restates ColumnVsColumnTableScanImpl::_typed_scan_chunk_with_iterators and the two-iterator loop of
// AbstractTableScanImpl::_scan_with_iterators<true> (abstract_table_scan_impl.hpp:56-84): a row matches iff neither side
// is NULL and the comparator (std::equal_to<void>, std::less<void>, ...) holds for the two values, i.e. after C++'s usual
// arithmetic conversions to their common type. String pairs compare value-IDs: the left ID i as 2 * i + 1, the right ID j
// as the host-built key right_in_left[j] (translate.cu), which orders against the left keys exactly like the strings.
#pragma once

#include "device_utils.cuh"
#include "internal.hpp"

namespace hyb {

enum PairMode : uint32_t {
  kPairNone = 0,       // no row can match (no rows, or one side has no dictionary entry): skip the chunk's bytes
  kPairStringIds = 1,  // string dictionaries: compare 2 * left ID + 1 with right_in_left[right ID]
  kPairDecoded = 2     // numeric: decode both sides in registers, compare in `compare`
};

enum PairCompare : uint32_t {
  kCompareInt64 = 0,   // int32 / int64 x int32 / int64: exact
  kCompareFloat = 1,   // int x float, float x float: the integer rounded to the nearest float first
  kCompareDouble = 2   // anything with a double, float x double
};

// The common type of std::less<void> and friends on two numeric column types (C++'s usual arithmetic conversions):
// TableScan's column pairs and JoinHash's secondary predicates.
inline PairCompare pair_compare(int32_t left_type, int32_t right_type) {
  const auto floating = [](int32_t type) { return type == HYB_TYPE_FLOAT32 || type == HYB_TYPE_FLOAT64; };
  if (left_type == HYB_TYPE_FLOAT64 || right_type == HYB_TYPE_FLOAT64) return kCompareDouble;
  if (floating(left_type) || floating(right_type)) return kCompareFloat;
  return kCompareInt64;
}

// The per-chunk test of a column pair (ChunkTest stays the one-column test).
struct PairTest {
  uint32_t mode;                   // PairMode
  int32_t condition;               // HYB_PRED_EQUALS .. HYB_PRED_GREATER_THAN_EQUALS
  uint32_t compare;                // PairCompare (kPairDecoded)
  uint32_t pad;
  const uint32_t* right_in_left;   // kPairStringIds: device copy of this chunk's words, one per right dictionary entry
};

// Conversions into the common type. The host pairs each type with a valid common type only, so the unused directions
// (a float into int64, a double into float) are never called.
struct AsInt64 {
  using T = long long;
  static __device__ __forceinline__ T from_i32(int32_t v) { return v; }
  static __device__ __forceinline__ T from_i64(long long v) { return v; }
  static __device__ __forceinline__ T from_f32(float) { return 0; }
  static __device__ __forceinline__ T from_f64(double) { return 0; }
};
struct AsFloat {
  using T = float;
  static __device__ __forceinline__ T from_i32(int32_t v) { return __int2float_rn(v); }
  static __device__ __forceinline__ T from_i64(long long v) { return __ll2float_rn(v); }
  static __device__ __forceinline__ T from_f32(float v) { return v; }
  static __device__ __forceinline__ T from_f64(double) { return 0.0f; }
};
struct AsDouble {
  using T = double;
  static __device__ __forceinline__ T from_i32(int32_t v) { return static_cast<double>(v); }
  static __device__ __forceinline__ T from_i64(long long v) { return __ll2double_rn(v); }
  static __device__ __forceinline__ T from_f32(float v) { return static_cast<double>(v); }
  static __device__ __forceinline__ T from_f64(double v) { return v; }
};

// Comparator of `condition` on 8 value pairs: bit j = a[j] <op> b[j]. IEEE comparisons: NaN fails every operator but !=.
template <typename T>
__device__ __forceinline__ uint32_t compare8(int32_t condition, const T (&a)[8], const T (&b)[8]) {
  uint32_t mask = 0;
  switch (condition) {
    case HYB_PRED_EQUALS:
#pragma unroll
      for (int j = 0; j < 8; ++j) mask |= a[j] == b[j] ? (1u << j) : 0u;
      break;
    case HYB_PRED_NOT_EQUALS:
#pragma unroll
      for (int j = 0; j < 8; ++j) mask |= a[j] != b[j] ? (1u << j) : 0u;
      break;
    case HYB_PRED_LESS_THAN:
#pragma unroll
      for (int j = 0; j < 8; ++j) mask |= a[j] < b[j] ? (1u << j) : 0u;
      break;
    case HYB_PRED_LESS_THAN_EQUALS:
#pragma unroll
      for (int j = 0; j < 8; ++j) mask |= a[j] <= b[j] ? (1u << j) : 0u;
      break;
    case HYB_PRED_GREATER_THAN:
#pragma unroll
      for (int j = 0; j < 8; ++j) mask |= a[j] > b[j] ? (1u << j) : 0u;
      break;
    default:  // HYB_PRED_GREATER_THAN_EQUALS
#pragma unroll
      for (int j = 0; j < 8; ++j) mask |= a[j] >= b[j] ? (1u << j) : 0u;
      break;
  }
  return mask;
}

template <typename T>
__device__ __forceinline__ bool compare1(int32_t condition, T a, T b) {
  switch (condition) {
    case HYB_PRED_EQUALS:
      return a == b;
    case HYB_PRED_NOT_EQUALS:
      return a != b;
    case HYB_PRED_LESS_THAN:
      return a < b;
    case HYB_PRED_LESS_THAN_EQUALS:
      return a <= b;
    case HYB_PRED_GREATER_THAN:
      return a > b;
    default:
      return a >= b;
  }
}

// Dictionary entry `id` (< dict_size) of a numeric dictionary segment, gathered through L1.
template <typename Conv>
__device__ __forceinline__ typename Conv::T gather_entry(const DevSegment& segment, uint32_t id) {
  switch (segment.data_type) {
    case HYB_TYPE_INT32:
      return Conv::from_i32(__ldg(static_cast<const int32_t*>(segment.values) + id));
    case HYB_TYPE_INT64:
      return Conv::from_i64(__ldg(static_cast<const long long*>(segment.values) + id));
    case HYB_TYPE_FLOAT32:
      return Conv::from_f32(__ldg(static_cast<const float*>(segment.values) + id));
    default:
      return Conv::from_f64(__ldg(static_cast<const double*>(segment.values) + id));
  }
}

// Values of rows row0 .. row0 + 7 of a Value / Dictionary / FrameOfReference segment in the common type; returns the
// NULL mask (dictionary: value-ID == dict_size; otherwise the null vector). Rows past the segment hold garbage.
template <typename Conv>
__device__ __forceinline__ uint32_t decode8(const DevSegment& segment, uint32_t row0, typename Conv::T (&out)[8]) {
  if (segment.encoding == HYB_ENC_DICTIONARY) {
    uint32_t codes[8];
    load_codes8(segment.av, segment.vector_type, segment.bit_width, row0, segment.row_count, codes);
    uint32_t nulls = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const bool is_null = codes[j] >= segment.dict_size;
      nulls |= is_null ? (1u << j) : 0u;
      out[j] = gather_entry<Conv>(segment, is_null ? 0u : codes[j]);
    }
    return nulls;
  }
  if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) {  // row0 % 8 == 0: the 8 rows share one 2048-row block
    uint32_t codes[8];
    load_codes8(segment.av, segment.vector_type, segment.bit_width, row0, segment.row_count, codes);
    const int32_t minimum = __ldg(static_cast<const int32_t*>(segment.values) + row0 / HYB_FOR_BLOCK_SIZE);
#pragma unroll
    for (int j = 0; j < 8; ++j) out[j] = Conv::from_i32(static_cast<int32_t>(static_cast<uint32_t>(minimum) + codes[j]));
    return load_nulls8(segment.nulls, row0);
  }
  if (segment.data_type == HYB_TYPE_INT32 || segment.data_type == HYB_TYPE_FLOAT32) {
    const uint4 a = ld_stream_v4(static_cast<const uint32_t*>(segment.values) + row0);
    const uint4 b = ld_stream_v4(static_cast<const uint32_t*>(segment.values) + row0 + 4);
    const uint32_t words[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    const bool integral = segment.data_type == HYB_TYPE_INT32;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      out[j] = integral ? Conv::from_i32(static_cast<int32_t>(words[j])) : Conv::from_f32(__uint_as_float(words[j]));
    }
  } else {
    const auto* base = static_cast<const unsigned long long*>(segment.values) + row0;
    const bool integral = segment.data_type == HYB_TYPE_INT64;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint4 v = ld_stream_v4(base + 2 * k);
      const long long lo = static_cast<long long>((static_cast<unsigned long long>(v.y) << 32) | v.x);
      const long long hi = static_cast<long long>((static_cast<unsigned long long>(v.w) << 32) | v.z);
      out[2 * k] = integral ? Conv::from_i64(lo) : Conv::from_f64(__longlong_as_double(lo));
      out[2 * k + 1] = integral ? Conv::from_i64(hi) : Conv::from_f64(__longlong_as_double(hi));
    }
  }
  return load_nulls8(segment.nulls, row0);
}

// One row of a segment in the common type; returns true for NULL (gather paths: position-filtered scans).
template <typename Conv>
__device__ __forceinline__ bool decode1(const DevSegment& segment, uint32_t row, typename Conv::T& out) {
  if (segment.encoding == HYB_ENC_DICTIONARY) {
    const uint32_t code = load_code1(segment.av, segment.vector_type, segment.bit_width, row);
    if (code >= segment.dict_size) return true;
    out = gather_entry<Conv>(segment, code);
    return false;
  }
  if (segment.nulls && segment.nulls[row]) return true;
  if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) {
    const uint32_t code = load_code1(segment.av, segment.vector_type, segment.bit_width, row);
    const int32_t minimum = __ldg(static_cast<const int32_t*>(segment.values) + row / HYB_FOR_BLOCK_SIZE);
    out = Conv::from_i32(static_cast<int32_t>(static_cast<uint32_t>(minimum) + code));
    return false;
  }
  switch (segment.data_type) {
    case HYB_TYPE_INT32:
      out = Conv::from_i32(__ldg(static_cast<const int32_t*>(segment.values) + row));
      break;
    case HYB_TYPE_INT64:
      out = Conv::from_i64(__ldg(static_cast<const long long*>(segment.values) + row));
      break;
    case HYB_TYPE_FLOAT32:
      out = Conv::from_f32(__ldg(static_cast<const float*>(segment.values) + row));
      break;
    default:
      out = Conv::from_f64(__ldg(static_cast<const double*>(segment.values) + row));
      break;
  }
  return false;
}

template <typename Conv>
__device__ __forceinline__ uint32_t decoded_pair8(const DevSegment& left, const DevSegment& right, int32_t condition,
                                                  uint32_t row0) {
  typename Conv::T a[8], b[8];
  const uint32_t nulls = decode8<Conv>(left, row0, a) | decode8<Conv>(right, row0, b);
  return compare8(condition, a, b) & ~nulls;
}

template <typename Conv>
__device__ __forceinline__ bool decoded_pair1(const DevSegment& left, const DevSegment& right, int32_t condition,
                                              uint32_t row) {
  typename Conv::T a, b;
  if (decode1<Conv>(left, row, a) || decode1<Conv>(right, row, b)) return false;
  return compare1(condition, a, b);
}

// 8 consecutive rows (row0 % 8 == 0) of one chunk: bit j = row0 + j matches. Control flow depends on per-chunk values
// only. The right key of a string pair is gathered through L1: a tile never straddles chunks, so a CTA reads one chunk's
// translation words (4 bytes per right dictionary entry).
__device__ __forceinline__ uint32_t evaluate8_pair(const DevSegment& left, const DevSegment& right, const PairTest& test,
                                                   uint32_t row0) {
  const uint32_t rows = left.row_count;
  const uint32_t valid = rows - row0 >= 8 ? 0xFFu : ((1u << (rows - row0)) - 1u);
  uint32_t mask = 0;
  if (test.mode == kPairStringIds) {
    uint32_t left_ids[8], right_ids[8];
    load_codes8(left.av, left.vector_type, left.bit_width, row0, rows, left_ids);
    load_codes8(right.av, right.vector_type, right.bit_width, row0, rows, right_ids);
    uint32_t left_keys[8], right_keys[8], nulls = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const bool right_null = right_ids[j] >= right.dict_size;
      nulls |= (left_ids[j] >= left.dict_size || right_null) ? (1u << j) : 0u;
      left_keys[j] = 2 * left_ids[j] + 1;
      right_keys[j] = right_null ? 0u : __ldg(test.right_in_left + right_ids[j]);
    }
    mask = compare8(test.condition, left_keys, right_keys) & ~nulls;
  } else if (test.compare == kCompareInt64) {
    mask = decoded_pair8<AsInt64>(left, right, test.condition, row0);
  } else if (test.compare == kCompareFloat) {
    mask = decoded_pair8<AsFloat>(left, right, test.condition, row0);
  } else {
    mask = decoded_pair8<AsDouble>(left, right, test.condition, row0);
  }
  return mask & valid;
}

__device__ __forceinline__ bool evaluate1_pair(const DevSegment& left, const DevSegment& right, const PairTest& test,
                                               uint32_t row) {
  switch (test.mode) {
    case kPairStringIds: {
      const uint32_t left_id = load_code1(left.av, left.vector_type, left.bit_width, row);
      const uint32_t right_id = load_code1(right.av, right.vector_type, right.bit_width, row);
      if (left_id >= left.dict_size || right_id >= right.dict_size) return false;
      return compare1(test.condition, 2 * left_id + 1, __ldg(test.right_in_left + right_id));
    }
    case kPairDecoded:
      if (test.compare == kCompareInt64) return decoded_pair1<AsInt64>(left, right, test.condition, row);
      if (test.compare == kCompareFloat) return decoded_pair1<AsFloat>(left, right, test.condition, row);
      return decoded_pair1<AsDouble>(left, right, test.condition, row);
    default:
      return false;
  }
}

}  // namespace hyb
