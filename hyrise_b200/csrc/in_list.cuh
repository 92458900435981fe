// `<column> [NOT] IN (<literal>, ...)` on Value / FrameOfReference segments, used by the TableScan pipelines of scan.cu.
//
// The host turns the list into sorted, disjoint closed intervals of the column's type (hyb_in_list_normalize, in_list.cu),
// stored as [lo, hi] pairs in the column's type. A row is decoded in
// registers (decode8 / decode1 of column_pair.cuh) and found with a branch-free binary search for the last interval whose
// lo is <= the value; it is inside iff that interval's hi is >= the value. NaN compares false with every bound, so it is
// never inside. The bounds (8 or 16 bytes per interval) are gathered through L1: every CTA searches the same few words.
#pragma once

#include "column_pair.cuh"
#include "predicate.cuh"

namespace hyb {

// The type the bounds are stored and compared in: the column's own type.
enum InCompare : uint32_t { kInInt32 = 0, kInInt64 = 1, kInFloat = 2, kInDouble = 3 };

// The list's intervals: the same for every chunk of the column.
struct InList {
  const void* bounds;       // interval_count [lo, hi] pairs of int32 / long long / float / double
  uint32_t interval_count;  // >= 1 (a list that matches no value holds one empty interval, lo > hi)
  uint32_t compare;         // InCompare
};

// int32 columns (Value, Dictionary, FrameOfReference) decode into int32: 4-byte bounds and 32-bit compares. The other
// directions are never called for an int32 column.
struct AsInt32 {
  using T = int32_t;
  static __device__ __forceinline__ T from_i32(int32_t v) { return v; }
  static __device__ __forceinline__ T from_i64(long long v) { return static_cast<int32_t>(v); }
  static __device__ __forceinline__ T from_f32(float) { return 0; }
  static __device__ __forceinline__ T from_f64(double) { return 0; }
};

template <typename T>
__device__ __forceinline__ uint32_t in_intervals8(const T* bounds, uint32_t count, const T (&values)[8]) {
  uint32_t base[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (uint32_t n = count; n > 1;) {  // uniform trip count: log2(count) steps
    const uint32_t half = n >> 1;
#pragma unroll
    for (int j = 0; j < 8; ++j) base[j] = __ldg(bounds + 2 * (base[j] + half)) <= values[j] ? base[j] + half : base[j];
    n -= half;
  }
  uint32_t mask = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const bool inside = __ldg(bounds + 2 * base[j]) <= values[j] && values[j] <= __ldg(bounds + 2 * base[j] + 1);
    mask |= inside ? (1u << j) : 0u;
  }
  return mask;
}

template <typename T>
__device__ __forceinline__ bool in_intervals1(const T* bounds, uint32_t count, T value) {
  uint32_t base = 0;
  for (uint32_t n = count; n > 1;) {
    const uint32_t half = n >> 1;
    base = __ldg(bounds + 2 * (base + half)) <= value ? base + half : base;
    n -= half;
  }
  return __ldg(bounds + 2 * base) <= value && value <= __ldg(bounds + 2 * base + 1);
}

template <typename Conv>
__device__ __forceinline__ uint32_t in_list_typed8(const DevSegment& segment, const InList& list, uint32_t row0,
                                                   uint32_t& nulls) {
  typename Conv::T values[8];
  nulls = decode8<Conv>(segment, row0, values);
  return in_intervals8(static_cast<const typename Conv::T*>(list.bounds), list.interval_count, values);
}

// 8 consecutive rows (row0 % 8 == 0) of a Value / FrameOfReference segment: bit j = row0 + j matches IN (negate: NOT IN).
// NULL rows never match.
__device__ __forceinline__ uint32_t evaluate8_in(const DevSegment& segment, const ChunkTest& test, const InList& list,
                                                 uint32_t row0) {
  const uint32_t rows = segment.row_count;
  const uint32_t valid = rows - row0 >= 8 ? 0xFFu : ((1u << (rows - row0)) - 1u);
  uint32_t nulls = 0, inside;
  if (list.compare == kInInt32) {
    inside = in_list_typed8<AsInt32>(segment, list, row0, nulls);
  } else if (list.compare == kInInt64) {
    inside = in_list_typed8<AsInt64>(segment, list, row0, nulls);
  } else if (list.compare == kInFloat) {
    inside = in_list_typed8<AsFloat>(segment, list, row0, nulls);
  } else {
    inside = in_list_typed8<AsDouble>(segment, list, row0, nulls);
  }
  return (test.negate ? ~inside : inside) & ~nulls & valid;
}

__device__ __forceinline__ bool evaluate1_in(const DevSegment& segment, const ChunkTest& test, const InList& list,
                                             uint32_t row) {
  bool inside;
  if (list.compare == kInInt32) {
    int32_t value;
    if (decode1<AsInt32>(segment, row, value)) return false;
    inside = in_intervals1(static_cast<const int32_t*>(list.bounds), list.interval_count, value);
  } else if (list.compare == kInInt64) {
    long long value;
    if (decode1<AsInt64>(segment, row, value)) return false;
    inside = in_intervals1(static_cast<const long long*>(list.bounds), list.interval_count, value);
  } else if (list.compare == kInFloat) {
    float value;
    if (decode1<AsFloat>(segment, row, value)) return false;
    inside = in_intervals1(static_cast<const float*>(list.bounds), list.interval_count, value);
  } else {
    double value;
    if (decode1<AsDouble>(segment, row, value)) return false;
    inside = in_intervals1(static_cast<const double*>(list.bounds), list.interval_count, value);
  }
  return inside != static_cast<bool>(test.negate);
}

}  // namespace hyb
