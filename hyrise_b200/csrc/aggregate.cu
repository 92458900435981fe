// AggregateHash on the device, with the TableScan predicates and the Projection arithmetic that precede it in a TPC-H
// plan fused into the same pass.
//
// Replaces AggregateHash::_on_execute (src/lib/operators/aggregate_hash.cpp:1180-1372): _partition_by_groupby_keys
// (:661-948), get_or_add_result (:317-403), _aggregate_segment (:605-655) and the output writers (:56-230, :421-537).
// The reference walks chunks and aggregates sequentially on one thread; here every row is handled once:
//
//   aggregate_fast_kernel<W, G, C>   the TPC-H shape: at most G <= 8 groups, SUM / AVG / COUNT over columns and over one
//       product chain col0 (x) f1(col1) (x) f2(col2) ... (Q1: price, price*(1-disc), price*(1-disc)*(1+tax); Q6:
//       price*disc). One streaming pass: 128-bit loads of value-IDs, predicates as bit masks (same code as TableScan),
//       dictionary decode in registers, float arithmetic with the reference's type rules (non-fused __fmul_rn /
//       __fsub_rn), group lookup in a CTA-shared table of <= G keys, per-thread double / int64 accumulators in
//       registers, one deterministic tree reduction per CTA, partials merged in CTA order on the host.
//       HBM traffic = the bytes of the referenced columns (+ their per-chunk dictionaries), each read once.
//   aggregate_general_kernel         everything else (MIN/MAX, arbitrary arithmetic, many groups, position-filtered
//       input): one thread per row, RPN interpreter, global open-addressing table keyed by the group-by values,
//       atomic accumulators. Falls back from the fast kernel when more than G groups show up.
//
// Group order and representative rows follow the reference: first appearance in row order — or ascending key with the
// NULL group first and the LAST row as representative when the immediate-key shortcut applies (:781-804, :367).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <numeric>

#include "bulk_copy.cuh"
#include "device_utils.cuh"
#include "internal.hpp"
#include "peer.hpp"
#include "expression.cuh"
#include "expression_scan.cuh"
#include "predicate.cuh"

namespace hyb {

constexpr int kAggThreads = 256;
constexpr int kAggWarps = kAggThreads / 32;
constexpr int kAggTileRows = 4096;
constexpr int kMaxKeyWords = HYB_MAX_GROUPBY_COLUMNS;

// ---------------------------------------------------------------------------------------------------------------------
// Shared device helpers
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
  x ^= x >> 33;
  x *= 0xFF51AFD7ED558CCDull;
  x ^= x >> 33;
  x *= 0xC4CEB9FE1A85EC53ull;
  x ^= x >> 33;
  return x;
}

// One AggregateKeyEntry (aggregate_hash.cpp:737-925). int32 -> value - INT32_MIN + 1, strings -> the per-dictionary
// codes the shim computed with the reference's scheme, other types -> their bit pattern (only equality matters).
__device__ __forceinline__ unsigned long long key_entry_from_code(const DevSegment& segment, uint32_t code_or_row,
                                                                  bool is_dictionary_code, bool& is_null) {
  is_null = false;
  if (is_dictionary_code) {
    const uint32_t value_id = code_or_row;
    if (value_id >= segment.dict_size) {
      is_null = true;
      return 0;
    }
    if (segment.dict_codes) return __ldg(segment.dict_codes + value_id);
    switch (segment.data_type) {
      case HYB_TYPE_INT32:
        return static_cast<unsigned long long>(static_cast<long long>(__ldg(static_cast<const int32_t*>(segment.values) + value_id)) + 2147483648ll) + 1ull;
      case HYB_TYPE_INT64:
        return static_cast<unsigned long long>(__ldg(static_cast<const long long*>(segment.values) + value_id));
      case HYB_TYPE_FLOAT32: {
        const float v = __ldg(static_cast<const float*>(segment.values) + value_id);
        return __float_as_uint(v == 0.0f ? 0.0f : v);
      }
      default: {
        const double v = __ldg(static_cast<const double*>(segment.values) + value_id);
        return static_cast<unsigned long long>(__double_as_longlong(v == 0.0 ? 0.0 : v));
      }
    }
  }
  return 0;
}

__device__ __forceinline__ unsigned long long key_entry_at(const DevSegment& segment, uint32_t row, bool& is_null) {
  if (segment.encoding == HYB_ENC_DICTIONARY) {
    const uint32_t value_id = load_code1(segment.av, segment.vector_type, segment.bit_width, row);
    return key_entry_from_code(segment, value_id, true, is_null);
  }
  is_null = segment.nulls && segment.nulls[row];
  if (is_null) return 0;
  if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) {
    const uint32_t code = load_code1(segment.av, segment.vector_type, segment.bit_width, row);
    const int32_t minimum = __ldg(static_cast<const int32_t*>(segment.values) + row / HYB_FOR_BLOCK_SIZE);
    const int32_t value = static_cast<int32_t>(static_cast<uint32_t>(minimum) + code);
    return static_cast<unsigned long long>(static_cast<long long>(value) + 2147483648ll) + 1ull;
  }
  switch (segment.data_type) {
    case HYB_TYPE_INT32:
      return static_cast<unsigned long long>(static_cast<long long>(__ldg(static_cast<const int32_t*>(segment.values) + row)) + 2147483648ll) + 1ull;
    case HYB_TYPE_INT64:
      return static_cast<unsigned long long>(__ldg(static_cast<const long long*>(segment.values) + row));
    case HYB_TYPE_FLOAT32: {
      const float v = __ldg(static_cast<const float*>(segment.values) + row);
      return __float_as_uint(v == 0.0f ? 0.0f : v);
    }
    default: {
      const double v = __ldg(static_cast<const double*>(segment.values) + row);
      return static_cast<unsigned long long>(__double_as_longlong(v == 0.0 ? 0.0 : v));
    }
  }
}

__device__ __forceinline__ DevScalar scalar_at(const DevSegment& segment, uint32_t row) {
  DevScalar s;
  s.type = segment.data_type;
  s.i64 = 0;
  uint32_t index = row;
  if (segment.encoding == HYB_ENC_DICTIONARY) {
    index = load_code1(segment.av, segment.vector_type, segment.bit_width, row);
    s.is_null = index >= segment.dict_size;
    if (s.is_null) return s;
  } else {
    s.is_null = segment.nulls && segment.nulls[row];
    if (s.is_null) return s;
    if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) {
      const uint32_t code = load_code1(segment.av, segment.vector_type, segment.bit_width, row);
      const int32_t minimum = __ldg(static_cast<const int32_t*>(segment.values) + row / HYB_FOR_BLOCK_SIZE);
      s.i32 = static_cast<int32_t>(static_cast<uint32_t>(minimum) + code);
      return s;
    }
  }
  switch (segment.data_type) {
    case HYB_TYPE_INT32:
      s.i32 = __ldg(static_cast<const int32_t*>(segment.values) + index);
      break;
    case HYB_TYPE_INT64:
      s.i64 = __ldg(static_cast<const long long*>(segment.values) + index);
      break;
    case HYB_TYPE_FLOAT32:
      s.f32 = __ldg(static_cast<const float*>(segment.values) + index);
      break;
    default:
      s.f64 = __ldg(static_cast<const double*>(segment.values) + index);
      break;
  }
  return s;
}

// ---------------------------------------------------------------------------------------------------------------------
// Plan (device-resident, read-only)
// ---------------------------------------------------------------------------------------------------------------------
struct DevExprNode {
  int32_t op;
  uint32_t column;  // index into AggregatePlan::columns
  int32_t literal_type;
  hyb_value literal;
};

struct DevAggregate {
  int32_t function;
  uint32_t node_count;
  int32_t input_type;
  int32_t result_type;
  DevExprNode nodes[HYB_MAX_EXPR_NODES];
};

struct AggregatePlan {
  // input positions
  const uint2* tile_map;       // unfiltered
  const hyb_row_id* filter;    // filtered
  const unsigned long long* chunk_row_start;
  unsigned long long position_count;
  uint32_t tile_count;
  uint32_t chunk_count;
  // fused predicates
  uint32_t predicate_count;
  const DevSegment* predicate_segments[HYB_MAX_FUSED_PREDICATES];
  const ChunkTest* predicate_tests[HYB_MAX_FUSED_PREDICATES];
  // group-by
  uint32_t groupby_count;
  const DevSegment* group_segments[HYB_MAX_GROUPBY_COLUMNS];
  // aggregates
  uint32_t aggregate_count;
  uint32_t column_count;
  const DevSegment* columns[HYB_MAX_AGGREGATES * 4];
  DevAggregate aggregates[HYB_MAX_AGGREGATES];
  // expression tree (kTreeRows sweeps only)
  const TestProgram* tree;
};

__device__ DevScalar evaluate_expression(const AggregatePlan& plan, const DevAggregate& aggregate, uint32_t chunk,
                                         uint32_t row) {
  DevScalar stack[HYB_MAX_EXPR_NODES];
  int top = 0;
  for (uint32_t n = 0; n < aggregate.node_count; ++n) {
    const DevExprNode& node = aggregate.nodes[n];
    if (node.op == HYB_EXPR_COLUMN) {
      stack[top++] = scalar_at(plan.columns[node.column][chunk], row);
    } else if (node.op == HYB_EXPR_LITERAL) {
      DevScalar s;
      s.type = node.literal_type;
      s.is_null = false;
      s.i64 = 0;
      if (node.literal_type == HYB_TYPE_INT32) s.i32 = node.literal.i32;
      if (node.literal_type == HYB_TYPE_INT64) s.i64 = node.literal.i64;
      if (node.literal_type == HYB_TYPE_FLOAT32) s.f32 = node.literal.f32;
      if (node.literal_type == HYB_TYPE_FLOAT64) s.f64 = node.literal.f64;
      stack[top++] = s;
    } else {
      const DevScalar b = stack[--top];
      const DevScalar a = stack[--top];
      stack[top++] = apply_arithmetic(node.op, a, b);
    }
  }
  return stack[0];
}

// ---------------------------------------------------------------------------------------------------------------------
// General path
// ---------------------------------------------------------------------------------------------------------------------
struct GroupTable {
  uint32_t capacity_mask;  // capacity - 1 (power of two)
  uint32_t key_words;      // max(groupby_count, 1)
  unsigned long long* hashes;    // 0 = empty
  uint32_t* states;              // 2 = key words published
  unsigned long long* keys;      // capacity * key_words
  uint32_t* null_masks;          // capacity
  unsigned long long* rows;      // capacity: COUNT(*)
  unsigned long long* min_position;
  unsigned long long* max_position;
  unsigned long long* accumulators;  // aggregate_count * capacity (double / int64 / ordered min-max encodings)
  unsigned long long* counts;        // aggregate_count * capacity (non-NULL inputs)
  // aggregate_count * capacity: position << 1 | sign bit of the first -0.0 / +0.0 a floating-point MIN / MAX met. The
  // ordered encoding holds both zeros as +0.0 (they compare equal); the reference keeps the first of equal values.
  unsigned long long* zero_first;
  uint32_t* control;                 // [0] groups inserted, [1] overflow
  // STDDEV_SAMP plans only (nullptr otherwise): 3 * aggregate_count * capacity doubles, per aggregate {mean, Σd, Σd²}
  // with d = x - mean (the second sweep of the corrected two-pass method).
  double* moments;
};

__device__ __forceinline__ unsigned long long ordered_from_double(double value) {
  const unsigned long long bits = static_cast<unsigned long long>(__double_as_longlong(value));
  return (bits >> 63) ? ~bits : (bits | 0x8000000000000000ull);
}
__device__ __forceinline__ unsigned long long ordered_from_int64(long long value) {
  return static_cast<unsigned long long>(value) ^ 0x8000000000000000ull;
}

// kDistinctSet: the table is a set of COUNT(DISTINCT) entries — no null masks, and `*inserted` tells whether this call
// added the key (exactly one caller per key sees true).
template <bool kDistinctSet = false>
__device__ uint32_t find_or_insert_group(const GroupTable& table, const unsigned long long* key, uint32_t null_mask,
                                         unsigned long long hash, bool* inserted_here = nullptr) {
  if constexpr (kDistinctSet) {
    // A set that asked to regrow is rerun anyway; stop filling it, or a set far smaller than the distinct values fills
    // up and every later insert probes all of it.
    if (*reinterpret_cast<volatile uint32_t*>(table.control + 1)) return 0xFFFFFFFFu;
  }
  uint32_t slot = static_cast<uint32_t>(hash >> 17) & table.capacity_mask;
  for (uint32_t probes = 0; probes <= table.capacity_mask; ++probes) {
    unsigned long long current = ld_volatile_u64(table.hashes + slot);
    if (current == 0) {
      current = atomicCAS(table.hashes + slot, 0ull, hash);
      if (current == 0) {
        for (uint32_t w = 0; w < table.key_words; ++w) table.keys[static_cast<size_t>(slot) * table.key_words + w] = key[w];
        if constexpr (!kDistinctSet) table.null_masks[slot] = null_mask;
        __threadfence();
        *reinterpret_cast<volatile uint32_t*>(table.states + slot) = 2;
        const uint32_t inserted = atomicAdd(table.control, 1u) + 1;
        if (inserted > (table.capacity_mask >> 1)) table.control[1] = 1;  // load factor > 0.5: ask for a bigger table
        if constexpr (kDistinctSet) *inserted_here = true;
        return slot;
      }
    }
    if (current == hash) {
      while (*reinterpret_cast<volatile uint32_t*>(table.states + slot) != 2) {
      }
      __threadfence();
      bool equal = kDistinctSet || *reinterpret_cast<volatile uint32_t*>(table.null_masks + slot) == null_mask;
      for (uint32_t w = 0; w < table.key_words && equal; ++w) {
        equal = ld_volatile_u64(table.keys + static_cast<size_t>(slot) * table.key_words + w) == key[w];
      }
      if (equal) return slot;
    }
    slot = (slot + 1) & table.capacity_mask;
  }
  table.control[1] = 1;
  return 0xFFFFFFFFu;
}

// Lookup-only probe of a group that an earlier kernel on the stream inserted and published.
__device__ uint32_t find_group(const GroupTable& table, const unsigned long long* key, uint32_t null_mask,
                               unsigned long long hash) {
  uint32_t slot = static_cast<uint32_t>(hash >> 17) & table.capacity_mask;
  for (uint32_t probes = 0; probes <= table.capacity_mask; ++probes) {
    const unsigned long long current = table.hashes[slot];
    if (current == 0) break;
    if (current == hash && table.null_masks[slot] == null_mask) {
      bool equal = true;
      for (uint32_t w = 0; w < table.key_words && equal; ++w) {
        equal = table.keys[static_cast<size_t>(slot) * table.key_words + w] == key[w];
      }
      if (equal) return slot;
    }
    slot = (slot + 1) & table.capacity_mask;
  }
  return 0xFFFFFFFFu;
}

// The value word a COUNT(DISTINCT) set holds: the int64 value, the bits of the value as double with -0.0 folded into
// +0.0, or the string's chunk-independent dictionary code. Equal words <=> equal values under std::equal_to, except NaN,
// which the caller counts without inserting (NaN != NaN, so every NaN row is a new value of the reference's set).
__device__ __forceinline__ unsigned long long distinct_word(const AggregatePlan& plan, const DevAggregate& aggregate,
                                                           uint32_t chunk, uint32_t row, bool& is_null, bool& is_nan) {
  is_nan = false;
  if (aggregate.input_type == HYB_TYPE_STRING) {
    return key_entry_at(plan.columns[aggregate.nodes[0].column][chunk], row, is_null);
  }
  const DevScalar value = evaluate_expression(plan, aggregate, chunk, row);
  is_null = value.is_null;
  if (value.type == HYB_TYPE_INT32 || value.type == HYB_TYPE_INT64) {
    return static_cast<unsigned long long>(scalar_to_int64(value));
  }
  const double as_double = scalar_to_double(value);
  is_nan = as_double != as_double;
  return static_cast<unsigned long long>(__double_as_longlong(as_double == 0.0 ? 0.0 : as_double));
}

// Sweeps of aggregate_general_kernel. kPlain is the only one plans without COUNT(DISTINCT) / STDDEV_SAMP launch.
// kTreeRows added to a sweep: a row must also satisfy the plan's expression tree (hyb_aggregate_hash_expression).
enum GeneralSweep : int { kPlain = 0, kWithDistinct = 1, kDeviations = 2, kTreeRows = 4 };

// kPlain / kWithDistinct: insert the groups and accumulate; STDDEV_SAMP gathers count and sum as AVG does, and
// COUNT(DISTINCT) inserts {aggregate, group slot, value word} into `distinct` and counts in the group's accumulator when
// this row inserted it. kDeviations: the same rows again after stddev_mean_kernel; each row finds its group with a
// lookup-only probe and adds d = x - mean and d² to the STDDEV_SAMP moments. kSweep | kTreeRows: the same sweep over the
// rows the plan's expression tree selects.
template <int kSweep>
__global__ void __launch_bounds__(kAggThreads) aggregate_general_kernel(const AggregatePlan* __restrict__ plan_ptr,
                                                                        const GroupTable table, const GroupTable distinct) {
  const AggregatePlan& plan = *plan_ptr;
  const uint32_t capacity = table.capacity_mask + 1;
  for (uint32_t tile = blockIdx.x; tile < plan.tile_count; tile += gridDim.x) {
    for (uint32_t index = threadIdx.x; index < kAggTileRows; index += kAggThreads) {
      uint32_t chunk, row;
      unsigned long long position;
      if (plan.tile_map) {
        const uint2 info = __ldg(plan.tile_map + tile);
        chunk = info.x;
        row = (info.y & 0x7FFFFFFFu) + index;
        const DevSegment& first = plan.groupby_count      ? plan.group_segments[0][chunk]
                                  : plan.column_count     ? plan.columns[0][chunk]
                                  : plan.predicate_count  ? plan.predicate_segments[0][chunk]
                                                          : plan.group_segments[0][chunk];
        if (row >= first.row_count) continue;
        position = __ldg(plan.chunk_row_start + chunk) + row;
      } else {
        position = static_cast<unsigned long long>(tile) * kAggTileRows + index;
        if (position >= plan.position_count) continue;
        const hyb_row_id row_id = plan.filter[position];
        chunk = row_id.chunk_id;
        row = row_id.chunk_offset;
      }
      bool keep = true;
      for (uint32_t p = 0; p < plan.predicate_count && keep; ++p) {
        keep = evaluate1(plan.predicate_segments[p][chunk], plan.predicate_tests[p][chunk], row);
      }
      if constexpr ((kSweep & kTreeRows) != 0) {
        const TestProgram& tree = *plan.tree;
        if (keep) keep = tree.operand_count ? evaluate1_tests<true>(tree, chunk, row) : evaluate1_tests<false>(tree, chunk, row);
      }
      if (!keep) continue;

      unsigned long long key[kMaxKeyWords];
      uint32_t null_mask = 0;
      unsigned long long hash = 0x9E3779B97F4A7C15ull;
      for (uint32_t g = 0; g < plan.groupby_count; ++g) {
        bool is_null;
        key[g] = key_entry_at(plan.group_segments[g][chunk], row, is_null);
        if (is_null) null_mask |= 1u << g;
        hash = mix64(hash ^ key[g]) + (is_null ? 0x51ED270B3Full : 0ull);
      }
      if (plan.groupby_count == 0) key[0] = 0;
      hash = mix64(hash) | 1ull;
      if constexpr ((kSweep & ~kTreeRows) == kDeviations) {
        const uint32_t slot = find_group(table, key, null_mask, hash);
        if (slot == 0xFFFFFFFFu) continue;  // cannot happen: the first sweep inserted every group of these rows
        for (uint32_t a = 0; a < plan.aggregate_count; ++a) {
          const DevAggregate& aggregate = plan.aggregates[a];
          if (aggregate.function != HYB_AGG_STDDEV_SAMP) continue;
          const DevScalar value = evaluate_expression(plan, aggregate, chunk, row);
          if (value.is_null) continue;
          double* moments = table.moments + static_cast<size_t>(a) * 3 * capacity + slot;
          const double d = scalar_to_double(value) - moments[0];
          atomicAdd(moments + capacity, d);
          atomicAdd(moments + 2 * static_cast<size_t>(capacity), d * d);
        }
        continue;
      }
      const uint32_t slot = find_or_insert_group(table, key, null_mask, hash);
      if (slot == 0xFFFFFFFFu) continue;
      atomicAdd(table.rows + slot, 1ull);
      atomicMin(table.min_position + slot, position);
      atomicMax(table.max_position + slot, position);

      for (uint32_t a = 0; a < plan.aggregate_count; ++a) {
        const DevAggregate& aggregate = plan.aggregates[a];
        if (aggregate.function == HYB_AGG_COUNT_STAR) continue;
        if constexpr ((kSweep & ~kTreeRows) == kWithDistinct) {
          if (aggregate.function == HYB_AGG_COUNT_DISTINCT) {
            bool is_null, is_nan;
            const unsigned long long word = distinct_word(plan, aggregate, chunk, row, is_null, is_nan);
            if (is_null) continue;
            unsigned long long* distinct_count = table.accumulators + static_cast<size_t>(a) * capacity + slot;
            if (is_nan) {
              atomicAdd(distinct_count, 1ull);
              continue;
            }
            const unsigned long long entry[2] = {(static_cast<unsigned long long>(a) << 32) | slot, word};
            bool inserted = false;
            find_or_insert_group<true>(distinct, entry, 0, mix64(mix64(entry[0] + 0x9E3779B97F4A7C15ull) ^ word) | 1ull,
                                       &inserted);
            if (inserted) atomicAdd(distinct_count, 1ull);
            continue;
          }
        }
        const DevScalar value = evaluate_expression(plan, aggregate, chunk, row);
        if (value.is_null) continue;
        unsigned long long* accumulator = table.accumulators + static_cast<size_t>(a) * capacity + slot;
        atomicAdd(table.counts + static_cast<size_t>(a) * capacity + slot, 1ull);
        if constexpr ((kSweep & ~kTreeRows) == kWithDistinct) {
          if (aggregate.function == HYB_AGG_STDDEV_SAMP) {
            // The first sweep gathers the sum for the mean in double for every argument type, as the reference converts
            // each value to double before its update: an int64 sum could wrap. Partial sums k * v of int32 values stay
            // exact below 2^22 rows, of float values below 2^29, so a constant group's mean is exactly its value.
            atomicAdd(reinterpret_cast<double*>(accumulator), scalar_to_double(value));
            continue;
          }
        }
        const bool integral = value.type == HYB_TYPE_INT32 || value.type == HYB_TYPE_INT64;
        switch (aggregate.function) {
          case HYB_AGG_SUM:
          case HYB_AGG_AVG:
            if (integral) {
              atomicAdd(accumulator, static_cast<unsigned long long>(scalar_to_int64(value)));
            } else {
              atomicAdd(reinterpret_cast<double*>(accumulator), scalar_to_double(value));
            }
            break;
          case HYB_AGG_MIN:
          case HYB_AGG_MAX: {
            unsigned long long ordered;
            if (integral) {
              ordered = ordered_from_int64(scalar_to_int64(value));
            } else {
              double as_double = scalar_to_double(value);
              if (as_double == 0.0) {
                atomicMin(table.zero_first + static_cast<size_t>(a) * capacity + slot,
                          (position << 1) | (__double_as_longlong(as_double) < 0 ? 1ull : 0ull));
                as_double = 0.0;
              }
              ordered = ordered_from_double(as_double);
            }
            if (aggregate.function == HYB_AGG_MIN) {
              atomicMin(accumulator, ordered);
            } else {
              atomicMax(accumulator, ordered);
            }
            break;
          }
          default:
            break;
        }
      }
    }
  }
}

// Between the two sweeps of a STDDEV_SAMP plan: mean = sum / count per occupied slot, on the device (the sum is a
// double for every argument type). Bit a of `stddev_mask` marks a STDDEV_SAMP aggregate.
__global__ void stddev_mean_kernel(const GroupTable table, uint32_t aggregate_count, uint32_t stddev_mask) {
  const uint32_t capacity = table.capacity_mask + 1;
  for (uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x; slot < capacity; slot += gridDim.x * blockDim.x) {
    if (table.hashes[slot] == 0) continue;
    for (uint32_t a = 0; a < aggregate_count; ++a) {
      if (!((stddev_mask >> a) & 1)) continue;
      const unsigned long long count = table.counts[static_cast<size_t>(a) * capacity + slot];
      if (count == 0) continue;
      const double sum = __longlong_as_double(static_cast<long long>(table.accumulators[static_cast<size_t>(a) * capacity + slot]));
      table.moments[static_cast<size_t>(a) * 3 * capacity + slot] = sum / static_cast<double>(count);
    }
  }
}

// The group table is sized for the worst case (2 slots per input row, at most 2^20 to start with); what leaves the
// device is only the occupied slots: this kernel packs them (order irrelevant: the host orders groups by their first row
// or, with immediate keys, by key) into arrays of `groups` entries with the layout of the table itself.
__global__ void aggregate_compact_kernel(const GroupTable table, uint32_t aggregate_count, uint32_t groups,
                                         unsigned long long* __restrict__ out_words, uint32_t* __restrict__ out_null_masks,
                                         uint32_t* __restrict__ cursor) {
  const uint32_t capacity = table.capacity_mask + 1;
  const uint32_t key_words = table.key_words;
  unsigned long long* out_hashes = out_words;
  unsigned long long* out_keys = out_hashes + groups;
  unsigned long long* out_rows = out_keys + static_cast<size_t>(groups) * key_words;
  unsigned long long* out_min = out_rows + groups;
  unsigned long long* out_max = out_min + groups;
  unsigned long long* out_accumulators = out_max + groups;
  unsigned long long* out_counts = out_accumulators + static_cast<size_t>(groups) * aggregate_count;
  unsigned long long* out_zero_first = out_counts + static_cast<size_t>(groups) * aggregate_count;
  // STDDEV_SAMP plans: {Σd, Σd²} per aggregate follow the zero_first words
  double* out_moments = reinterpret_cast<double*>(out_zero_first + static_cast<size_t>(groups) * aggregate_count);
  for (uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x; slot < capacity; slot += gridDim.x * blockDim.x) {
    const unsigned long long hash = table.hashes[slot];
    if (hash == 0) continue;
    const uint32_t at = atomicAdd(cursor, 1u);
    if (at >= groups) continue;  // cannot happen: `groups` is the table's own insert counter
    out_hashes[at] = hash;
    for (uint32_t w = 0; w < key_words; ++w) out_keys[static_cast<size_t>(at) * key_words + w] = table.keys[static_cast<size_t>(slot) * key_words + w];
    out_rows[at] = table.rows[slot];
    out_min[at] = table.min_position[slot];
    out_max[at] = table.max_position[slot];
    for (uint32_t a = 0; a < aggregate_count; ++a) {
      out_accumulators[static_cast<size_t>(a) * groups + at] = table.accumulators[static_cast<size_t>(a) * capacity + slot];
      out_counts[static_cast<size_t>(a) * groups + at] = table.counts[static_cast<size_t>(a) * capacity + slot];
      out_zero_first[static_cast<size_t>(a) * groups + at] = table.zero_first[static_cast<size_t>(a) * capacity + slot];
      if (table.moments) {
        const double* moments = table.moments + static_cast<size_t>(a) * 3 * capacity + slot;
        out_moments[(static_cast<size_t>(a) * 2) * groups + at] = moments[capacity];
        out_moments[(static_cast<size_t>(a) * 2 + 1) * groups + at] = moments[2 * static_cast<size_t>(capacity)];
      }
    }
    out_null_masks[at] = table.null_masks[slot];
  }
}

// String MIN / MAX: the general kernel accumulated the ordered encoding of the extreme order rank (the column's
// StringColumnView turns its dictionaries into rank words). Before the occupied slots are packed, each such accumulator
// becomes the hyb_dictionary_position {chunk_id, value_id} of the first dictionary entry holding that rank.
struct StringExtremes {
  const unsigned long long* first_entry[HYB_MAX_AGGREGATES];  // per aggregate: chunk << 32 | value-ID by rank, or nullptr
};

__global__ void string_extreme_kernel(const GroupTable table, uint32_t aggregate_count,
                                      const __grid_constant__ StringExtremes extremes) {
  const uint32_t capacity = table.capacity_mask + 1;
  for (uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x; slot < capacity; slot += gridDim.x * blockDim.x) {
    if (table.hashes[slot] == 0) continue;
    for (uint32_t a = 0; a < aggregate_count; ++a) {
      if (!extremes.first_entry[a] || table.counts[static_cast<size_t>(a) * capacity + slot] == 0) continue;
      unsigned long long* accumulator = table.accumulators + static_cast<size_t>(a) * capacity + slot;
      const uint32_t rank = static_cast<uint32_t>(*accumulator ^ 0x8000000000000000ull);
      const unsigned long long entry = extremes.first_entry[a][rank];
      *accumulator = (entry >> 32) | (entry << 32);
    }
  }
}

// Once per hyb_table_set_string_order: the first {chunk, value-ID} (in chunk order) of every rank, as chunk << 32 |
// value-ID so that atomicMin keeps the first. One CTA per chunk.
__global__ void string_order_first_entry_kernel(const uint32_t* __restrict__ ranks, const uint64_t* __restrict__ chunk_begin,
                                                uint32_t chunk_count, unsigned long long* __restrict__ first_entry) {
  for (uint32_t chunk = blockIdx.x; chunk < chunk_count; chunk += gridDim.x) {
    const uint64_t begin = chunk_begin[chunk], end = chunk_begin[chunk + 1];
    for (uint64_t entry = begin + threadIdx.x; entry < end; entry += blockDim.x) {
      atomicMin(first_entry + ranks[entry], (static_cast<unsigned long long>(chunk) << 32) | (entry - begin));
    }
  }
}

__global__ void gather_row_ids_kernel(const unsigned long long* __restrict__ positions, uint32_t count,
                                      const hyb_row_id* __restrict__ filter, hyb_row_id* __restrict__ out) {
  const uint32_t index = blockIdx.x * blockDim.x + threadIdx.x;
  if (index < count) out[index] = filter[positions[index]];
}

// ---------------------------------------------------------------------------------------------------------------------
// Fast path
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kFastMaxColumns = 4;
enum AffineKind : int32_t { kIdentity = 0, kLiteralMinusColumn = 1, kLiteralPlusColumn = 2, kColumnMinusLiteral = 3, kColumnPlusLiteral = 4 };

struct FastPlan {
  const DevSegment* size_segments;  // any column of the table: row count per chunk
  const uint2* tile_map;
  const unsigned long long* chunk_row_start;
  uint32_t tile_count;
  uint32_t predicate_count;
  const DevSegment* predicate_segments[HYB_MAX_FUSED_PREDICATES];
  const ChunkTest* predicate_tests[HYB_MAX_FUSED_PREDICATES];
  uint32_t groupby_count;
  const DevSegment* group_segments[HYB_MAX_GROUPBY_COLUMNS];
  const DevSegment* value_segments[kFastMaxColumns];
  int32_t affine_kind[kFastMaxColumns];
  double literal[kFastMaxColumns];
  uint32_t need_raw_mask;   // bit i: accumulate column i itself
  uint32_t need_product_mask;  // bit i: accumulate f0(col0) * ... * fi(coli)
  // per-CTA partials
  unsigned long long* partial_hash;      // [cta][G]
  unsigned long long* partial_keys;      // [cta][G][kMaxKeyWords]
  uint32_t* partial_null_mask;           // [cta][G]
  unsigned long long* partial_rows;      // [cta][G]
  unsigned long long* partial_min_position;
  unsigned long long* partial_max_position;
  unsigned long long* partial_raw;       // [cta][G][C] (double or int64 bits)
  unsigned long long* partial_product;   // [cta][G][C]
  unsigned long long* partial_raw_nulls;      // [cta][G][C]
  unsigned long long* partial_product_nulls;  // [cta][G][C]
  uint32_t* overflow;                    // set when a CTA sees more than G groups
};

template <int W>
struct WorkType;
template <>
struct WorkType<0> {
  using Value = float;
  using Accumulator = double;
};
template <>
struct WorkType<1> {
  using Value = double;
  using Accumulator = double;
};
template <>
struct WorkType<2> {
  using Value = long long;
  using Accumulator = long long;
};

template <int W>
__device__ __forceinline__ typename WorkType<W>::Value typed_load(const void* base, uint8_t data_type, uint32_t index) {
  if constexpr (W == 0) {
    return __ldg(static_cast<const float*>(base) + index);
  } else if constexpr (W == 1) {
    return __ldg(static_cast<const double*>(base) + index);
  } else {
    return data_type == HYB_TYPE_INT32 ? static_cast<long long>(__ldg(static_cast<const int32_t*>(base) + index))
                                       : __ldg(static_cast<const long long*>(base) + index);
  }
}

// Values of 8 consecutive rows of a value column in the working type + NULL bits.
template <int W>
__device__ __forceinline__ void load_values8(const DevSegment& segment, uint32_t row0, typename WorkType<W>::Value (&values)[8],
                                             uint32_t& null_bits) {
  using Value = typename WorkType<W>::Value;
  null_bits = 0;
  if (segment.encoding == HYB_ENC_DICTIONARY) {
    uint32_t codes[8];
    load_codes8(segment.av, segment.vector_type, segment.bit_width, row0, segment.row_count, codes);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const bool is_null = codes[j] >= segment.dict_size;
      null_bits |= is_null ? (1u << j) : 0u;
      values[j] = is_null ? Value{} : typed_load<W>(segment.values, segment.data_type, codes[j]);
    }
    return;
  }
  null_bits = load_nulls8(segment.nulls, row0);
  if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) {
    if constexpr (W == 2) {
      uint32_t codes[8];
      load_codes8(segment.av, segment.vector_type, segment.bit_width, row0, segment.row_count, codes);
      const int32_t minimum = __ldg(static_cast<const int32_t*>(segment.values) + row0 / HYB_FOR_BLOCK_SIZE);
#pragma unroll
      for (int j = 0; j < 8; ++j) values[j] = static_cast<int32_t>(static_cast<uint32_t>(minimum) + codes[j]);
    }
    return;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    values[j] = (row0 + j < segment.row_count) ? typed_load<W>(segment.values, segment.data_type, row0 + j) : Value{};
  }
}

// Factor of the product chain as a + b * value with b = +-1: one FMA, and bit-identical to the reference's separate
// subtraction / addition because b * value is exact (lit - col == fma(-1, col, lit), col - lit == fma(1, col, -lit)).
template <int W>
__device__ __forceinline__ typename WorkType<W>::Value apply_affine(typename WorkType<W>::Value a, typename WorkType<W>::Value b,
                                                                    typename WorkType<W>::Value value) {
  if constexpr (W == 0) {
    return __fmaf_rn(b, value, a);
  } else if constexpr (W == 1) {
    return __fma_rn(b, value, a);
  } else {
    return value;
  }
}

template <int W>
__device__ __forceinline__ typename WorkType<W>::Value multiply(typename WorkType<W>::Value a, typename WorkType<W>::Value b) {
  if constexpr (W == 0) {
    return __fmul_rn(a, b);
  } else if constexpr (W == 1) {
    return __dmul_rn(a, b);
  } else {
    return a * b;
  }
}

template <typename T>
__device__ __forceinline__ T warp_reduce_add(T value) {
#pragma unroll
  for (int delta = 16; delta > 0; delta >>= 1) value += __shfl_xor_sync(kFullMask, value, delta);
  return value;
}

// Element j of a register-resident 8-array for a run-time j. Indexing such an array directly (a[j]) in a rolled loop
// makes the compiler place the WHOLE array in local memory for its entire lifetime — measured as LDL/STL round trips on
// every access of the hot path — so the rare rolled loops go through these select chains instead.
template <typename T>
__device__ __forceinline__ T pick8(const T (&array)[8], int j) {
  T result = array[0];
#pragma unroll
  for (int k = 1; k < 8; ++k) result = (j == k) ? array[k] : result;
  return result;
}
template <typename T>
__device__ __forceinline__ void put8(T (&array)[8], int j, T value) {
#pragma unroll
  for (int k = 0; k < 8; ++k) array[k] = (j == k) ? value : array[k];
}

constexpr int kEarlyPredicates = 2;   // fused predicates / group-by columns whose loads are hoisted to the top of an
constexpr int kEarlyGroups = 2;       // iteration (the rest load at their point of use)
constexpr int kFastThreads = 128;
constexpr int kFastWarps = kFastThreads / 32;
constexpr int kFastRowsPerWarp = kAggTileRows / kFastWarps;   // 1024 contiguous rows per warp and tile
constexpr int kFastIterations = kFastRowsPerWarp / 256;       // 8 rows per thread per iteration
constexpr int kStagedDictionary = 256;                        // dictionaries up to this size are staged in shared memory
constexpr int kMaxCombos = 256;                              // product of (dictionary size + 1) over the group-by columns
constexpr uint8_t kComboUnresolved = 0xFF;
constexpr uint8_t kComboOverflow = 0xFE;

// acc += value where the row's group equals g. A predicated add on purpose: written as `if (group == g) acc[g] += v`
// the compiler folds the chain into an indexed access and moves the accumulators from registers to local memory; as a
// select (group == g ? v : 0) every add costs two extra SEL instructions.
__device__ __forceinline__ void add_where(double& accumulator, double value, int group, int g) {
  asm("{\n\t.reg .pred p;\n\tsetp.eq.s32 p, %2, %3;\n\t@p add.rn.f64 %0, %0, %1;\n\t}"
      : "+d"(accumulator)
      : "d"(value), "r"(group), "r"(g));
}
__device__ __forceinline__ void add_where(long long& accumulator, long long value, int group, int g) {
  asm("{\n\t.reg .pred p;\n\tsetp.eq.s32 p, %2, %3;\n\t@p add.s64 %0, %0, %1;\n\t}"
      : "+l"(accumulator)
      : "l"(value), "r"(group), "r"(g));
}

// kTree: a row must also satisfy the expression tree `tree` (hyb_aggregate_hash_expression); its 8-bit mask joins the
// fused predicates' mask before the group lookup.
template <int W, int G, int C, bool kTree>
__device__ __forceinline__ void aggregate_fast_rows(const FastPlan* __restrict__ plan_ptr, const TestProgram* __restrict__ tree) {
  using Value = typename WorkType<W>::Value;
  using Accumulator = typename WorkType<W>::Accumulator;
  const FastPlan& plan = *plan_ptr;

  // CTA-wide group table (<= G distinct keys), filled on first sight
  __shared__ unsigned long long s_hash[G];
  __shared__ unsigned long long s_keys[G][kMaxKeyWords];
  __shared__ uint32_t s_null_mask[G];
  __shared__ unsigned long long s_null_counts[2][G][C];  // [raw | product] NULL inputs (rare path)
  // per-tile staging
  __shared__ DevSegment s_value_segment[C];
  __shared__ DevSegment s_group_segment[G == 1 ? 1 : HYB_MAX_GROUPBY_COLUMNS];
  __shared__ Value s_dictionary[C][kStagedDictionary];
  __shared__ uint8_t s_dictionary_staged[C];
  __shared__ uint8_t s_combo_group[G == 1 ? 4 : kMaxCombos];
  __shared__ uint32_t s_combo_stride[G == 1 ? 1 : HYB_MAX_GROUPBY_COLUMNS];
  __shared__ uint32_t s_use_combos;
  __shared__ Accumulator s_reduce[kFastWarps];
  __shared__ unsigned long long s_reduce_u64[kFastWarps];

  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x < G) {
    s_hash[threadIdx.x] = 0;
    s_null_mask[threadIdx.x] = 0;
    for (int w = 0; w < kMaxKeyWords; ++w) s_keys[threadIdx.x][w] = 0;
    for (int c = 0; c < C; ++c) {
      s_null_counts[0][threadIdx.x][c] = 0;
      s_null_counts[1][threadIdx.x][c] = 0;
    }
  }

  Accumulator raw_sum[G][C], product_sum[G][C];
  uint32_t rows[G];                 // a thread sees far fewer than 2^32 rows
  unsigned long long first_position[G], last_position[G];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    rows[g] = 0;
    first_position[g] = ~0ull;
    last_position[g] = 0;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      raw_sum[g][c] = Accumulator{};
      product_sum[g][c] = Accumulator{};
    }
  }
  Value affine_a[C], affine_b[C];
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const Value literal = static_cast<Value>(plan.literal[c]);
    const int32_t kind = plan.affine_kind[c];
    affine_a[c] = (kind == kLiteralMinusColumn || kind == kLiteralPlusColumn || kind == kColumnPlusLiteral) ? literal
                  : kind == kColumnMinusLiteral                                                             ? -literal
                                                                                                            : Value{};
    affine_b[c] = kind == kLiteralMinusColumn ? Value(-1) : Value(1);
  }
  const uint32_t need_raw_mask = plan.need_raw_mask, need_product_mask = plan.need_product_mask;
  const uint32_t groupby_count = plan.groupby_count;

  // Static tile assignment in units of kTilesPerUnit consecutive tiles, units strided over the CTAs. Static keeps the
  // summation order reproducible; consecutive tiles of a unit come from the same chunk, so descriptors, dictionaries and
  // the combo table are staged once per unit instead of once per tile (the staging is a chain of dependent global loads
  // and barriers, ~4 us, that the row work cannot hide); striding the units keeps the CTAs of a wave on neighbouring
  // memory (fully blocked assignment — one chunk range per CTA — measured 40 % slower on bandwidth-heavy queries).
  constexpr uint32_t kTilesPerUnit = 4;
  uint32_t staged_chunk = 0xFFFFFFFFu;
  const uint32_t unit_count = (plan.tile_count + kTilesPerUnit - 1) / kTilesPerUnit;
  for (uint32_t unit = blockIdx.x; unit < unit_count; unit += gridDim.x)
  for (uint32_t tile = unit * kTilesPerUnit; tile < min(plan.tile_count, (unit + 1) * kTilesPerUnit); ++tile) {
    const uint2 info = __ldg(plan.tile_map + tile);
    const uint32_t chunk = info.x;
    const uint32_t tile_row0 = info.y & 0x7FFFFFFFu;
    const unsigned long long chunk_first_position = __ldg(plan.chunk_row_start + chunk);
    const uint32_t chunk_rows = plan.size_segments[chunk].row_count;

    if (chunk != staged_chunk) {
    staged_chunk = chunk;
    // ---- per-chunk staging: segment descriptors, small dictionaries, the combo -> group table ----------------------
    __syncthreads();  // previous tile done with the staged data
    if (threadIdx.x < C && plan.value_segments[threadIdx.x]) {
      s_value_segment[threadIdx.x] = plan.value_segments[threadIdx.x][chunk];
    }
    if (G > 1 && threadIdx.x >= 32 && threadIdx.x < 32 + groupby_count) {
      s_group_segment[threadIdx.x - 32] = plan.group_segments[threadIdx.x - 32][chunk];
    }
    __syncthreads();
    if constexpr (G > 1) {
      if (threadIdx.x == 0) {
        uint32_t combos = 1;
        bool usable = true;
        for (uint32_t q = 0; q < groupby_count; ++q) {
          const DevSegment& segment = s_group_segment[q];
          usable = usable && segment.encoding == HYB_ENC_DICTIONARY && segment.vector_type == HYB_VEC_FIXED_1B;
          s_combo_stride[q] = combos;
          combos = usable ? combos * (segment.dict_size + 1) : combos;
          usable = usable && combos <= kMaxCombos;
        }
        s_use_combos = usable ? combos : 0;
      }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) {
      if (plan.value_segments[c] == nullptr) continue;
      const DevSegment& segment = s_value_segment[c];
      const bool staged = segment.encoding == HYB_ENC_DICTIONARY && segment.dict_size <= kStagedDictionary;
      if (threadIdx.x == 0) s_dictionary_staged[c] = staged;
      if (staged) {
        for (uint32_t i = threadIdx.x; i < segment.dict_size; i += kFastThreads) {
          s_dictionary[c][i] = typed_load<W>(segment.values, segment.data_type, i);
        }
      }
    }
    __syncthreads();
    if constexpr (G > 1) {
      // Resolve every value-ID combination of this chunk against the groups the CTA already knows (lookup only: a
      // combination that never occurs must not claim a slot). After the first tiles all real groups are known, so
      // rows take the per-row slow path only on first sightings.
      for (uint32_t combination = threadIdx.x; combination < s_use_combos; combination += kFastThreads) {
        unsigned long long hash = 0x9E3779B97F4A7C15ull;
        uint32_t rest = combination;
        for (uint32_t q = 0; q < groupby_count; ++q) {
          const DevSegment& segment = s_group_segment[q];
          const uint32_t value_id = rest % (segment.dict_size + 1);
          rest /= segment.dict_size + 1;
          bool is_null;
          const unsigned long long entry = key_entry_from_code(segment, value_id, true, is_null);
          hash = mix64(hash ^ entry) + (is_null ? 0x51ED270B3Full : 0ull);
        }
        hash = mix64(hash) | 1ull;
        uint8_t group = kComboUnresolved;
        for (int g = 0; g < G; ++g) {
          if (*reinterpret_cast<volatile unsigned long long*>(&s_hash[g]) == hash) group = static_cast<uint8_t>(g);
        }
        s_combo_group[combination] = group;
      }
      __syncthreads();
    }
    }  // staging
    const bool use_combos = G > 1 && s_use_combos != 0;

#pragma unroll 1
    for (int it = 0; it < kFastIterations; ++it) {
      const uint32_t row0 = tile_row0 + warp * kFastRowsPerWarp + it * 256 + lane * 8;
      if (row0 >= chunk_rows) continue;
      // ---- early loads: an iteration costs two DRAM round trips — all predicate columns, then (for threads with a
      // surviving row) all group-by and value columns — instead of one per column; see device_utils.cuh. Static
      // indexes only (a run-time index would move the arrays to local memory).
      uint4 raw_predicate[kEarlyPredicates];
      bool early_predicate[kEarlyPredicates];
#pragma unroll
      for (int p = 0; p < kEarlyPredicates; ++p) {
        early_predicate[p] = false;
        raw_predicate[p] = uint4{0u, 0u, 0u, 0u};
        if (static_cast<uint32_t>(p) < plan.predicate_count) {
          const DevSegment& segment = plan.predicate_segments[p][chunk];
          const uint32_t mode = plan.predicate_tests[p][chunk].mode;
          early_predicate[p] = raw_codes_loadable(segment) && (mode == kTestIdRange || mode == kTestIdSet || mode == kTestInt);
          raw_predicate[p] = early_predicate[p] ? load_raw_codes8(segment, row0) : uint4{0u, 0u, 0u, 0u};
        }
      }
      uint32_t mask = chunk_rows - row0 >= 8 ? 0xFFu : ((1u << (chunk_rows - row0)) - 1u);
#pragma unroll
      for (int p = 0; p < kEarlyPredicates; ++p) {
        if (static_cast<uint32_t>(p) < plan.predicate_count) {
          const ChunkTest& test = plan.predicate_tests[p][chunk];
          mask &= test.mode == kTestNone ? 0u
                                         : evaluate8(plan.predicate_segments[p][chunk], test, row0, early_predicate[p],
                                                     raw_predicate[p]);
        }
      }
      for (uint32_t p = kEarlyPredicates; p < plan.predicate_count && mask; ++p) {
        const ChunkTest& test = plan.predicate_tests[p][chunk];
        mask &= test.mode == kTestNone ? 0u : evaluate8(plan.predicate_segments[p][chunk], test, row0);
      }
      if constexpr (kTree) {
        if (mask) {
          mask &= tree->operand_count ? evaluate8_tests<true>(*tree, chunk, row0, chunk_rows)
                                      : evaluate8_tests<false>(*tree, chunk, row0, chunk_rows);
        }
      }
      if (mask == 0) continue;
      // second round trip: group-by and value columns, only for threads with a surviving row
      uint2 raw_group[kEarlyGroups];
      if constexpr (G > 1) {
        if (use_combos) {
#pragma unroll
          for (int q = 0; q < kEarlyGroups; ++q) {
            if (static_cast<uint32_t>(q) < groupby_count) {
              raw_group[q] = ld_stream_v2(static_cast<const uint8_t*>(s_group_segment[q].av) + row0);
            }
          }
        }
      }
      uint4 raw_value[C];
      bool early_value[C];
#pragma unroll
      for (int c = 0; c < C; ++c) {
        early_value[c] = false;
        raw_value[c] = uint4{0u, 0u, 0u, 0u};
        if (plan.value_segments[c] != nullptr) {
          const DevSegment& segment = s_value_segment[c];
          early_value[c] = segment.encoding == HYB_ENC_DICTIONARY && raw_codes_loadable(segment);
          raw_value[c] = early_value[c] ? load_raw_codes8(segment, row0) : uint4{0u, 0u, 0u, 0u};
        }
      }

      // ---- group of each row ----------------------------------------------------------------------------------------
      int32_t group_of[8];
      if constexpr (G == 1) {
#pragma unroll
        for (int j = 0; j < 8; ++j) group_of[j] = ((mask >> j) & 1u) ? 0 : -1;
        if (s_hash[0] == 0) s_hash[0] = 1;  // benign race: every writer stores the same value
      } else {
        uint32_t combo[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          combo[j] = 0;
          group_of[j] = -1;
        }
        if (use_combos) {
#pragma unroll
          for (int q = 0; q < kEarlyGroups; ++q) {
            if (static_cast<uint32_t>(q) < groupby_count) {
              const uint2 packed = raw_group[q];
              const uint32_t stride = s_combo_stride[q];
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                combo[j] += ((packed.x >> (8 * j)) & 0xFFu) * stride;
                combo[4 + j] += ((packed.y >> (8 * j)) & 0xFFu) * stride;
              }
            }
          }
          for (uint32_t q = kEarlyGroups; q < groupby_count; ++q) {
            const uint2 packed = ld_stream_v2(static_cast<const uint8_t*>(s_group_segment[q].av) + row0);
            const uint32_t stride = s_combo_stride[q];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              combo[j] += ((packed.x >> (8 * j)) & 0xFFu) * stride;
              combo[4 + j] += ((packed.y >> (8 * j)) & 0xFFu) * stride;
            }
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if ((mask >> j) & 1u) group_of[j] = s_combo_group[combo[j]];
          }
        }
        // slow path: rows whose combination has not been seen in this tile (or every row when combos are unusable)
        bool any_unresolved = !use_combos;
#pragma unroll
        for (int j = 0; j < 8; ++j) any_unresolved = any_unresolved || group_of[j] >= static_cast<int32_t>(kComboOverflow);
        if (any_unresolved)
#pragma unroll 1
        for (int j = 0; j < 8; ++j) {
          if (!((mask >> j) & 1u)) continue;
          const int32_t known = pick8(group_of, j);
          const uint32_t combination = pick8(combo, j);
          if (use_combos && known != kComboUnresolved) {
            if (known == kComboOverflow) {
              put8(group_of, j, int32_t{-1});
              mask &= ~(1u << j);
            }
            continue;
          }
          unsigned long long entries[kMaxKeyWords];
          uint32_t null_mask = 0;
          unsigned long long hash = 0x9E3779B97F4A7C15ull;
          for (uint32_t q = 0; q < groupby_count; ++q) {
            bool is_null;
            entries[q] = key_entry_at(s_group_segment[q], row0 + j, is_null);
            if (is_null) null_mask |= 1u << q;
            hash = mix64(hash ^ entries[q]) + (is_null ? 0x51ED270B3Full : 0ull);
          }
          hash = mix64(hash) | 1ull;
          int32_t found = -1;
          for (int g = 0; g < G && found < 0; ++g) {
            unsigned long long current = *reinterpret_cast<volatile unsigned long long*>(&s_hash[g]);
            if (current == 0ull) {
              current = atomicCAS(&s_hash[g], 0ull, hash);
              if (current == 0ull) {
                for (uint32_t q = 0; q < groupby_count; ++q) s_keys[g][q] = entries[q];
                s_null_mask[g] = null_mask;
                found = g;
              }
            }
            if (current == hash) found = g;
          }
          if (found < 0) {
            *plan.overflow = 1;  // more than G groups: the host reruns with a bigger G or the general kernel
            mask &= ~(1u << j);
            if (use_combos) s_combo_group[combination] = kComboOverflow;
          } else if (use_combos) {
            s_combo_group[combination] = static_cast<uint8_t>(found);
          }
          put8(group_of, j, found);
        }
      }

      // ---- rows / first / last position per group, once per iteration through hit masks ---------------------------
      {
        const unsigned long long base_position = chunk_first_position + row0;
#pragma unroll
        for (int g = 0; g < G; ++g) {
          uint32_t hits = 0;
#pragma unroll
          for (int j = 0; j < 8; ++j) hits |= (group_of[j] == g) ? (1u << j) : 0u;
          if (hits) {
            if (rows[g] == 0) first_position[g] = base_position + (__ffs(hits) - 1);
            last_position[g] = base_position + (31 - __clz(hits));
            rows[g] += __popc(hits);
          }
        }
      }

      // ---- value columns: raw sums and the running product ------------------------------------------------------------
      Value product[8];
      uint32_t product_nulls = 0;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        if (plan.value_segments[c] == nullptr) continue;
        const DevSegment& segment = s_value_segment[c];
        Value values[8];
        uint32_t null_bits = 0;
        if (segment.encoding == HYB_ENC_DICTIONARY) {
          uint32_t codes[8];
          codes8(segment, row0, early_value[c], raw_value[c], codes);
          if (segment.pad & kSegmentMayContainNulls) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const bool is_null = codes[j] >= segment.dict_size;
              null_bits |= is_null ? (1u << j) : 0u;
              codes[j] = is_null ? 0u : codes[j];
            }
          } else if (row0 + 8 > segment.row_count) {
#pragma unroll
            for (int j = 0; j < 8; ++j) codes[j] = row0 + j < segment.row_count ? codes[j] : 0u;
          }
          if (s_dictionary_staged[c]) {
#pragma unroll
            for (int j = 0; j < 8; ++j) values[j] = s_dictionary[c][codes[j]];
          } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) values[j] = typed_load<W>(segment.values, segment.data_type, codes[j]);
          }
        } else {
          load_values8<W>(segment, row0, values, null_bits);
        }
        const bool need_raw = (need_raw_mask >> c) & 1u;
        const bool need_product = (need_product_mask >> c) & 1u;
        const bool in_chain = (need_product_mask >> c) != 0;  // some product at or after this column
        if (in_chain) {
          product_nulls |= null_bits;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const Value factor = apply_affine<W>(affine_a[c], affine_b[c], values[j]);
            product[j] = c == 0 ? factor : multiply<W>(product[j], factor);
          }
        }
        if (need_raw) {
          if (null_bits == 0) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const Accumulator value = static_cast<Accumulator>(values[j]);
#pragma unroll
              for (int g = 0; g < G; ++g) add_where(raw_sum[g][c], value, group_of[j], g);
            }
          } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int32_t group = ((null_bits >> j) & 1u) ? -1 : group_of[j];
              const Accumulator value = static_cast<Accumulator>(values[j]);
#pragma unroll
              for (int g = 0; g < G; ++g) add_where(raw_sum[g][c], value, group, g);
            }
          }
        }
        if (need_product) {
          if (product_nulls == 0) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const Accumulator value = static_cast<Accumulator>(product[j]);
#pragma unroll
              for (int g = 0; g < G; ++g) add_where(product_sum[g][c], value, group_of[j], g);
            }
          } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int32_t group = ((product_nulls >> j) & 1u) ? -1 : group_of[j];
              const Accumulator value = static_cast<Accumulator>(product[j]);
#pragma unroll
              for (int g = 0; g < G; ++g) add_where(product_sum[g][c], value, group, g);
            }
          }
        }
        if ((need_raw && (null_bits & mask)) || (need_product && (product_nulls & mask))) {
#pragma unroll 1
          for (int j = 0; j < 8; ++j) {
            const int32_t group = pick8(group_of, j);
            if (!((mask >> j) & 1u) || group < 0) continue;
            if (need_raw && ((null_bits >> j) & 1u)) atomicAdd(&s_null_counts[0][group][c], 1ull);
            if (need_product && ((product_nulls >> j) & 1u)) atomicAdd(&s_null_counts[1][group][c], 1ull);
          }
        }
      }
    }
  }

  // CTA reduction in a fixed order: lanes (butterfly), then warps.
  __syncthreads();
  const size_t cta = blockIdx.x;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const unsigned long long total_rows = warp_reduce_add(static_cast<unsigned long long>(rows[g]));
    unsigned long long low = first_position[g], high = last_position[g];
#pragma unroll
    for (int delta = 16; delta > 0; delta >>= 1) {
      low = min(low, __shfl_xor_sync(kFullMask, low, delta));
      high = max(high, __shfl_xor_sync(kFullMask, high, delta));
    }
    if (lane == 0) s_reduce_u64[warp] = total_rows;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long sum = 0;
      for (int w = 0; w < kFastWarps; ++w) sum += s_reduce_u64[w];
      plan.partial_rows[cta * G + g] = sum;
    }
    __syncthreads();
    if (lane == 0) s_reduce_u64[warp] = low;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long value = ~0ull;
      for (int w = 0; w < kFastWarps; ++w) value = min(value, s_reduce_u64[w]);
      plan.partial_min_position[cta * G + g] = value;
    }
    __syncthreads();
    if (lane == 0) s_reduce_u64[warp] = high;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long value = 0;
      for (int w = 0; w < kFastWarps; ++w) value = max(value, s_reduce_u64[w]);
      plan.partial_max_position[cta * G + g] = value;
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < C; ++c) {
#pragma unroll
      for (int which = 0; which < 2; ++which) {
        const Accumulator lane_sum = warp_reduce_add(which == 0 ? raw_sum[g][c] : product_sum[g][c]);
        if (lane == 0) s_reduce[warp] = lane_sum;
        __syncthreads();
        if (threadIdx.x == 0) {
          Accumulator sum{};
          for (int w = 0; w < kFastWarps; ++w) sum += s_reduce[w];
          unsigned long long bits;
          memcpy(&bits, &sum, sizeof(bits));
          (which == 0 ? plan.partial_raw : plan.partial_product)[(cta * G + g) * C + c] = bits;
        }
        __syncthreads();
      }
    }
  }
  if (threadIdx.x < G) {
    const int g = threadIdx.x;
    plan.partial_hash[cta * G + g] = s_hash[g];
    plan.partial_null_mask[cta * G + g] = s_null_mask[g];
    for (int w = 0; w < kMaxKeyWords; ++w) plan.partial_keys[(cta * G + g) * kMaxKeyWords + w] = s_keys[g][w];
    for (int c = 0; c < C; ++c) {
      plan.partial_raw_nulls[(cta * G + g) * C + c] = s_null_counts[0][g][c];
      plan.partial_product_nulls[(cta * G + g) * C + c] = s_null_counts[1][g][c];
    }
  }
}

template <int W, int G, int C, int kMinBlocks>
__global__ void __launch_bounds__(kFastThreads, kMinBlocks) aggregate_fast_kernel(const FastPlan* __restrict__ plan_ptr) {
  aggregate_fast_rows<W, G, C, false>(plan_ptr, nullptr);
}

template <int W, int G, int C, int kMinBlocks>
__global__ void __launch_bounds__(kFastThreads, kMinBlocks) aggregate_fast_tree_kernel(const FastPlan* __restrict__ plan_ptr,
                                                                                       const TestProgram* __restrict__ tree) {
  aggregate_fast_rows<W, G, C, true>(plan_ptr, tree);
}

}  // namespace hyb

#include "aggregate_stream.cuh"

namespace hyb {

// A kernel of aggregate_fast_kernel (parameter: the plan) or aggregate_fast_tree_kernel (the plan and the tree).
using FastKernel = const void*;

// Resident CTAs per SM the register allocation is capped for: 3 (170 registers) measured best for Q1 — 2 leaves too few
// warps to hide latency (+24 %), 4 spills the accumulators (+30 %).
constexpr int kFastMinBlocks = 3;

template <int W, int G, int C>
static FastKernel fast_kernel_for_min_blocks(bool tree) {
  return tree ? reinterpret_cast<FastKernel>(aggregate_fast_tree_kernel<W, G, C, kFastMinBlocks>)
              : reinterpret_cast<FastKernel>(aggregate_fast_kernel<W, G, C, kFastMinBlocks>);
}

template <int W, int G>
static FastKernel fast_kernel_for_columns(int columns, bool tree) {
  switch (columns) {
    case 1:
      return fast_kernel_for_min_blocks<W, G, 1>(tree);
    case 2:
      return fast_kernel_for_min_blocks<W, G, 2>(tree);
    default:
      return fast_kernel_for_min_blocks<W, G, 4>(tree);
  }
}

template <int W>
static FastKernel fast_kernel_for_groups(int groups, int columns, bool tree) {
  switch (groups) {
    case 1:
      return fast_kernel_for_columns<W, 1>(columns, tree);
    case 4:
      return fast_kernel_for_columns<W, 4>(columns, tree);
    default:
      return fast_kernel_for_columns<W, 8>(columns, tree);
  }
}

static FastKernel fast_kernel(int work_type, int groups, int columns, bool tree) {
  switch (work_type) {
    case 0:
      return fast_kernel_for_groups<0>(groups, columns, tree);
    case 1:
      return fast_kernel_for_groups<1>(groups, columns, tree);
    default:
      return fast_kernel_for_groups<2>(groups, columns, tree);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------------------------------
struct HostGroup {
  std::vector<uint64_t> key;
  uint32_t null_mask = 0;
  uint64_t rows = 0;
  uint64_t min_position = ~uint64_t{0};
  uint64_t max_position = 0;
  std::vector<uint64_t> accumulators;  // per aggregate (bits)
  std::vector<uint64_t> counts;        // per aggregate
  // distributed aggregation: positions are global and the rows behind them are named directly (they may live on another rank)
  bool has_global_rows = false;
  hyb_row_id row_min{}, row_max{};
};

struct AggregateExchange {
  PeerGroup* group;
  uint32_t chunk_id_base;
  uint64_t position_base;
};

static int expression_type(const Table* table, const hyb_aggregate_def& def, int32_t* out_type) {
  std::vector<int32_t> stack;
  for (uint32_t n = 0; n < def.node_count; ++n) {
    const auto& node = def.nodes[n];
    if (node.op == HYB_EXPR_COLUMN) {
      HYB_CHECK(node.column_id < table->column_count, HYB_ERR_INVALID, "expression column out of range");
      const int32_t type = table->column_types[node.column_id];
      HYB_CHECK(type != HYB_TYPE_STRING, HYB_ERR_UNSUPPORTED, "aggregates over string columns stay on the CPU operator");
      stack.push_back(type < 0 ? HYB_TYPE_INT32 : type);
    } else if (node.op == HYB_EXPR_LITERAL) {
      HYB_CHECK(node.literal_type >= HYB_TYPE_INT32 && node.literal_type <= HYB_TYPE_FLOAT64, HYB_ERR_INVALID,
                "bad literal type");
      stack.push_back(node.literal_type);
    } else {
      HYB_CHECK(node.op != HYB_EXPR_MOD && node.op != HYB_EXPR_NULL, HYB_ERR_UNSUPPORTED,
                "modulo and NULL literals in aggregate programs run on the CPU operator");
      HYB_CHECK(node.op >= HYB_EXPR_ADD && node.op <= HYB_EXPR_DIV, HYB_ERR_INVALID, "bad expression op");
      HYB_CHECK(stack.size() >= 2, HYB_ERR_INVALID, "malformed expression");
      const int32_t b = stack.back();
      stack.pop_back();
      const int32_t a = stack.back();
      stack.pop_back();
      stack.push_back(expression_common_type(a, b));
    }
  }
  HYB_CHECK(stack.size() == 1, HYB_ERR_INVALID, "malformed expression");
  *out_type = stack[0];
  return HYB_OK;
}

static int32_t aggregate_result_type(int32_t function, int32_t input_type) {  // window_function_traits.hpp:14-77
  const bool integral = input_type == HYB_TYPE_INT32 || input_type == HYB_TYPE_INT64;
  switch (function) {
    case HYB_AGG_COUNT:
    case HYB_AGG_COUNT_STAR:
    case HYB_AGG_COUNT_DISTINCT:
      return HYB_TYPE_INT64;
    case HYB_AGG_SUM:
      return integral ? HYB_TYPE_INT64 : HYB_TYPE_FLOAT64;
    case HYB_AGG_AVG:
    case HYB_AGG_STDDEV_SAMP:
      return HYB_TYPE_FLOAT64;
    default:
      return input_type;
  }
}

// ---- fast-path planning: recognise `col`, and left-nested products of {col, lit (+|-) col, col (+|-) lit} -----------
struct Factor {
  uint32_t column;
  int32_t kind;
  double literal;
  int32_t literal_type = HYB_TYPE_INT32;
  bool operator==(const Factor& other) const {
    return column == other.column && kind == other.kind && (kind == kIdentity || literal == other.literal);
  }
};

static double literal_as_double(const hyb_expr_node& node) {
  switch (node.literal_type) {
    case HYB_TYPE_INT32:
      return node.literal.i32;
    case HYB_TYPE_INT64:
      return static_cast<double>(node.literal.i64);
    case HYB_TYPE_FLOAT32:
      return node.literal.f32;
    default:
      return node.literal.f64;
  }
}

// Parses the RPN program into a chain of factors; false if it is not of the supported shape.
static bool parse_product_chain(const hyb_aggregate_def& def, std::vector<Factor>* chain) {
  struct Item {
    enum { kLiteral, kFactor, kChain } what;
    double literal = 0;
    int32_t literal_type = 0;
    std::vector<Factor> factors;
  };
  std::vector<Item> stack;
  for (uint32_t n = 0; n < def.node_count; ++n) {
    const auto& node = def.nodes[n];
    if (node.op == HYB_EXPR_COLUMN) {
      Item item;
      item.what = Item::kFactor;
      item.factors.push_back(Factor{node.column_id, kIdentity, 0.0, HYB_TYPE_INT32});
      stack.push_back(item);
    } else if (node.op == HYB_EXPR_LITERAL) {
      Item item;
      item.what = Item::kLiteral;
      item.literal = literal_as_double(node);
      item.literal_type = node.literal_type;
      stack.push_back(item);
    } else {
      if (stack.size() < 2) return false;
      Item b = stack.back();
      stack.pop_back();
      Item a = stack.back();
      stack.pop_back();
      Item result;
      if (node.op == HYB_EXPR_ADD || node.op == HYB_EXPR_SUB) {
        const bool plus = node.op == HYB_EXPR_ADD;
        if (a.what == Item::kLiteral && b.what == Item::kFactor && b.factors[0].kind == kIdentity) {
          result.what = Item::kFactor;
          result.factors.push_back(Factor{b.factors[0].column, plus ? kLiteralPlusColumn : kLiteralMinusColumn, a.literal, a.literal_type});
        } else if (b.what == Item::kLiteral && a.what == Item::kFactor && a.factors[0].kind == kIdentity) {
          result.what = Item::kFactor;
          result.factors.push_back(Factor{a.factors[0].column, plus ? kColumnPlusLiteral : kColumnMinusLiteral, b.literal, b.literal_type});
        } else {
          return false;
        }
      } else if (node.op == HYB_EXPR_MUL) {
        if (a.what == Item::kLiteral || b.what == Item::kLiteral) return false;
        if (b.what != Item::kFactor) return false;  // only left-nested products: (a * b) * c
        result.what = Item::kChain;
        result.factors = a.factors;
        result.factors.push_back(b.factors[0]);
      } else {
        return false;
      }
      stack.push_back(result);
    }
  }
  if (stack.size() != 1 || stack[0].what == Item::kLiteral) return false;
  *chain = stack[0].factors;
  return true;
}

struct FastMapping {
  bool is_count_star = false;
  bool uses_product = false;
  uint32_t column_slot = 0;  // index into the canonical column list
};

struct FastPlanHost {
  bool possible = false;
  int work_type = 0;  // 0 float, 1 double, 2 int64
  std::vector<Factor> columns;  // canonical order: the product chain first, then stand-alone columns
  uint32_t chain_length = 0;
  uint32_t need_raw_mask = 0, need_product_mask = 0;
  std::vector<FastMapping> mapping;  // per aggregate
};

static FastPlanHost plan_fast_path(const Table* table, const hyb_aggregate_query* query) {
  FastPlanHost plan;
  if (query->filter) return plan;
  std::vector<std::vector<Factor>> chains(query->aggregate_count);
  std::vector<Factor> longest;
  for (uint32_t a = 0; a < query->aggregate_count; ++a) {
    const auto& def = query->aggregates[a];
    if (def.function == HYB_AGG_COUNT_STAR) continue;
    if (def.function != HYB_AGG_SUM && def.function != HYB_AGG_AVG && def.function != HYB_AGG_COUNT) return plan;
    if (!parse_product_chain(def, &chains[a])) return plan;
    const bool is_plain_column = chains[a].size() == 1 && chains[a][0].kind == kIdentity;
    if (!is_plain_column && chains[a].size() > longest.size()) longest = chains[a];
  }
  // every non-trivial chain must be a prefix of the longest one
  for (uint32_t a = 0; a < query->aggregate_count; ++a) {
    const auto& chain = chains[a];
    const bool is_plain_column = chain.size() == 1 && chain[0].kind == kIdentity;
    if (chain.empty() || is_plain_column) continue;
    if (chain.size() > longest.size()) return plan;
    for (size_t i = 0; i < chain.size(); ++i) {
      if (!(chain[i] == longest[i])) return plan;
    }
  }
  plan.columns = longest;
  plan.chain_length = static_cast<uint32_t>(longest.size());
  // a column may appear only once in the chain (keeps the column <-> slot mapping unique)
  for (size_t i = 0; i < longest.size(); ++i) {
    for (size_t j = i + 1; j < longest.size(); ++j) {
      if (longest[i].column == longest[j].column) return plan;
    }
  }
  plan.mapping.resize(query->aggregate_count);
  for (uint32_t a = 0; a < query->aggregate_count; ++a) {
    const auto& def = query->aggregates[a];
    auto& mapping = plan.mapping[a];
    if (def.function == HYB_AGG_COUNT_STAR) {
      mapping.is_count_star = true;
      continue;
    }
    const auto& chain = chains[a];
    const bool is_plain_column = chain.size() == 1 && chain[0].kind == kIdentity;
    if (is_plain_column) {
      size_t slot = plan.columns.size();
      for (size_t i = 0; i < plan.columns.size(); ++i) {
        if (plan.columns[i].column == chain[0].column) slot = i;
      }
      if (slot == plan.columns.size()) plan.columns.push_back(chain[0]);
      // chain position 0 with identity kind: the product P_1 equals the raw column, either accumulator works
      mapping.column_slot = static_cast<uint32_t>(slot);
      plan.need_raw_mask |= 1u << slot;
    } else {
      mapping.uses_product = true;
      mapping.column_slot = static_cast<uint32_t>(chain.size() - 1);
      plan.need_product_mask |= 1u << (chain.size() - 1);
    }
  }
  if (plan.columns.size() > kFastMaxColumns) return plan;
  // one working type: all value columns share a type; arithmetic only on float / double columns
  int32_t type = -1;
  for (const auto& factor : plan.columns) {
    const int32_t column_type = table->column_types[factor.column];
    if (column_type == HYB_TYPE_STRING) return plan;
    const int32_t normalised = column_type == HYB_TYPE_INT32 ? HYB_TYPE_INT64 : column_type;
    if (type < 0) type = normalised;
    if (type != normalised) return plan;
  }
  if (type < 0) type = HYB_TYPE_INT64;  // COUNT(*) only
  if (type == HYB_TYPE_INT64 && plan.chain_length > 0) return plan;
  if (type == HYB_TYPE_INT64) {
    // int32 and int64 columns must not be mixed inside one FrameOfReference / value decode path: they are not (checked
    // per segment at decode time through data_type), nothing to do.
  }
  // The fast kernels evaluate `literal (+|-) column` in the columns' type. The reference promotes per operation with
  // std::common_type (expression_utils.cpp:172-205): a double literal next to a float column makes the factor — and every
  // product after it — double, which only the general kernel's interpreter reproduces. Integer literals keep the
  // column type (float o int -> float).
  if (type == HYB_TYPE_FLOAT32) {
    for (const auto& factor : plan.columns) {
      if (factor.kind != kIdentity && factor.literal_type == HYB_TYPE_FLOAT64) return plan;
    }
  }
  plan.work_type = type == HYB_TYPE_FLOAT32 ? 0 : type == HYB_TYPE_FLOAT64 ? 1 : 2;
  plan.possible = true;
  return plan;
}

// ---- streaming kernel: host-side eligibility + shared-memory layout ----------------------------------------------------
struct StreamLayout {
  bool possible = false;
  StreamPlan plan{};        // everything but plan.fast
  size_t dynamic_bytes = 0;
};

// Registry of the compile-time row-loop shapes (aggregate_stream.cuh): W, G, C, shape word. The layout-generic instantiations
// (shape 0) cover every eligible plan; these add the fixed-width layouts dbgen's lineitem yields for the TPC-H Q1 / Q6 plans
// (the shapes of the reference's own headline queries) — anything else a deployment runs hot is one line here.
//   Q1: l_shipdate (2-byte value-IDs) range test | 2 group-by columns | l_extendedprice (2-byte IDs, dictionary in global
//       memory), 1 - l_discount, 1 + l_tax, l_quantity (1-byte IDs, staged dictionaries); sums: price, disc, qty raw + 2 products
//   Q6: l_shipdate, l_discount, l_quantity range tests | no group-by | sum(l_extendedprice * l_discount)
constexpr uint64_t kShapeTpchQ1 =
    shape_counts(1, 2) | shape_predicate(0, 2, 0) | shape_value(0, 2, kValueGlobalDictionary, kIdentity, true) |
    shape_value(1, 1, kValueStagedDictionary, kLiteralMinusColumn, true) |
    shape_value(2, 1, kValueStagedDictionary, kLiteralPlusColumn, false) | shape_value(3, 1, kValueStagedDictionary, kIdentity, true) |
    shape_products(0b0110);
constexpr uint64_t kShapeTpchQ6 = shape_counts(3, 0) | shape_predicate(0, 2, 0) | shape_predicate(1, 1, 0) | shape_predicate(2, 1, 0) |
                                  shape_value(0, 2, kValueGlobalDictionary, kIdentity, false) |
                                  shape_value(1, 1, kValueStagedDictionary, kIdentity, false) | shape_products(0b0010);
#define HYB_STREAM_SHAPES(X) \
  X(0, 4, 4, kShapeTpchQ1)   \
  X(0, 1, 2, kShapeTpchQ6)

// The shape word of a plan, 0 if the word cannot express it (more predicates than it has room for, encoded int tests, ...).
static uint64_t stream_shape_of(const StreamPlan& plan, const FastPlan& fast, uint32_t column_count) {
  if (fast.predicate_count > kShapeMaxPredicates || fast.groupby_count > 7 || column_count > 4) return 0;
  uint64_t shape = shape_counts(fast.predicate_count, fast.groupby_count) | shape_products(fast.need_product_mask);
  for (uint32_t p = 0; p < fast.predicate_count; ++p) {
    uint32_t mode_code;
    if (plan.predicate_mode[p] == kTestIdRange) {
      mode_code = 0;
    } else if (plan.predicate_mode[p] == kTestInt && plan.predicate_encoding[p] == HYB_ENC_UNENCODED) {
      mode_code = 1;
    } else if (plan.predicate_mode[p] == kTestFloat) {
      mode_code = 2;
    } else {
      return 0;
    }
    shape |= shape_predicate(static_cast<int>(p), plan.predicate_width[p], mode_code);
  }
  for (uint32_t c = 0; c < column_count; ++c) {
    if (fast.value_segments[c] == nullptr) continue;
    shape |= shape_value(static_cast<int>(c), plan.value_width[c], plan.value_kind[c], fast.affine_kind[c], (fast.need_raw_mask >> c) & 1u);
  }
  return shape;
}

template <int W>
static void* stream_kernel_for(int groups, int columns, uint64_t shape, bool* is_static) {
  *is_static = true;
#define HYB_STREAM_MATCH(SW, SG, SC, SHAPE) \
  if (W == SW && groups == SG && columns == SC && shape == SHAPE) return reinterpret_cast<void*>(aggregate_stream_static_kernel<SW, SG, SC, SHAPE>);
  HYB_STREAM_SHAPES(HYB_STREAM_MATCH)
#undef HYB_STREAM_MATCH
  *is_static = false;
  if (groups == 1) {
    return columns == 1   ? reinterpret_cast<void*>(aggregate_stream_kernel<W, 1, 1>)
           : columns == 2 ? reinterpret_cast<void*>(aggregate_stream_kernel<W, 1, 2>)
                          : reinterpret_cast<void*>(aggregate_stream_kernel<W, 1, 4>);
  }
  return columns == 1   ? reinterpret_cast<void*>(aggregate_stream_kernel<W, 4, 1>)
         : columns == 2 ? reinterpret_cast<void*>(aggregate_stream_kernel<W, 4, 2>)
                        : reinterpret_cast<void*>(aggregate_stream_kernel<W, 4, 4>);
}

static StreamLayout stream_layout_for(const Table* table, const hyb_aggregate_query* query, const FastPlanHost& fast,
                                      uint32_t stage_count, bool tree) {
  StreamLayout layout;
  if (fast.work_type == 2 || table->row_count() >= 0xFFFFFFF0ull) return layout;
  // an expression tree is evaluated by the register-tile and general kernels only
  if (tree) return layout;
  // a single int32 group-by column may take the immediate-key order, which needs the LAST row of every group
  if (query->groupby_count == 1 && table->column_types[query->groupby_column_ids[0]] == HYB_TYPE_INT32) return layout;
  // the row loop decodes a dictionary predicate as a value-ID range (predicate_mode below); LIKE needs the id-set test of
  // the register-tile and general kernels
  for (uint32_t p = 0; p < query->predicate_count; ++p) {
    if (is_like_condition(query->predicates[p].condition)) return layout;
  }
  const uint32_t chunk_count = table->chunk_count();
  std::vector<uint32_t> staged;  // distinct referenced columns
  const auto slot_of = [&](uint32_t column) -> uint32_t {
    for (size_t i = 0; i < staged.size(); ++i) {
      if (staged[i] == column) return static_cast<uint32_t>(i);
    }
    staged.push_back(column);
    return static_cast<uint32_t>(staged.size() - 1);
  };
  std::vector<uint32_t> predicate_slot(query->predicate_count), group_slot(query->groupby_count), value_slot(fast.columns.size());
  for (uint32_t p = 0; p < query->predicate_count; ++p) predicate_slot[p] = slot_of(query->predicates[p].column_id);
  for (uint32_t g = 0; g < query->groupby_count; ++g) group_slot[g] = slot_of(query->groupby_column_ids[g]);
  for (size_t c = 0; c < fast.columns.size(); ++c) value_slot[c] = slot_of(fast.columns[c].column);
  if (staged.size() > kStreamMaxColumns) return layout;

  const auto stream_width = [](const DevSegment& segment) -> uint32_t {
    if (segment.encoding == HYB_ENC_UNENCODED) return static_cast<uint32_t>(data_type_size(segment.data_type));
    return segment.vector_type == HYB_VEC_FIXED_1B ? 1u : segment.vector_type == HYB_VEC_FIXED_2B ? 2u
           : segment.vector_type == HYB_VEC_FIXED_4B ? 4u : 0u;
  };
  const size_t value_size = fast.work_type == 0 ? sizeof(float) : sizeof(double);
  std::vector<uint32_t> max_width(staged.size(), 0);
  std::vector<uint32_t> max_dictionary(table->column_count, 0);
  for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
    const DevSegment* segments = &table->segments[size_t{chunk} * table->column_count];
    for (size_t i = 0; i < staged.size(); ++i) {
      const DevSegment& segment = segments[staged[i]];
      const uint32_t width = stream_width(segment);
      if (width == 0 || width > 4 || segment.nulls || (segment.pad & kSegmentMayContainNulls)) return layout;
      // one encoding per column: the row loop is compiled for the launch constants (narrower vectors are widened per tile)
      if (segment.encoding != table->segments[staged[i]].encoding) return layout;
      max_width[i] = std::max(max_width[i], width);
      max_dictionary[staged[i]] = std::max(max_dictionary[staged[i]], segment.dict_size);
    }
    uint64_t combos = 1;
    for (uint32_t g = 0; g < query->groupby_count; ++g) {
      const DevSegment& segment = segments[query->groupby_column_ids[g]];
      if (segment.encoding != HYB_ENC_DICTIONARY || segment.vector_type != HYB_VEC_FIXED_1B || segment.dict_size == 0) return layout;
      if (!segment.dict_codes && segment.data_type == HYB_TYPE_STRING) return layout;
      combos *= segment.dict_size;
    }
    if (combos > kMaxCombos) return layout;
    for (const auto& factor : fast.columns) {
      const DevSegment& segment = segments[factor.column];
      const bool right_type = segment.data_type == (fast.work_type == 0 ? HYB_TYPE_FLOAT32 : HYB_TYPE_FLOAT64);
      if (!right_type) return layout;
      if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) return layout;
      if (segment.encoding == HYB_ENC_UNENCODED && fast.work_type != 0) return layout;
    }
  }
  // stage = column slices | small dictionaries of the value columns | key data of the group-by dictionaries | header
  StreamPlan& plan = layout.plan;
  uint32_t offset = 0;
  plan.column_count = static_cast<uint32_t>(staged.size());
  for (size_t i = 0; i < staged.size(); ++i) {
    plan.columns[i].segments = table->d_segments + size_t{staged[i]} * chunk_count;
    plan.columns[i].slot_offset = offset;
    plan.column_width[i] = max_width[i];
    offset += kStreamTileRows * max_width[i];
  }
  // launch constants: widest vector / largest dictionary of a column over all chunks, the (uniform) encoding
  const DevSegment* first = &table->segments[0];
  for (uint32_t p = 0; p < query->predicate_count; ++p) {
    const DevSegment& segment = first[query->predicates[p].column_id];
    const int32_t condition = query->predicates[p].condition;
    const bool null_check = condition == HYB_PRED_IS_NULL || condition == HYB_PRED_IS_NOT_NULL;
    plan.predicate_offset[p] = plan.columns[predicate_slot[p]].slot_offset;
    plan.predicate_width[p] = max_width[predicate_slot[p]];
    plan.predicate_encoding[p] = segment.encoding;
    plan.predicate_mode[p] = segment.encoding == HYB_ENC_DICTIONARY ? kTestIdRange
                             : null_check                            ? kTestNull
                             : (segment.data_type == HYB_TYPE_FLOAT32 || segment.data_type == HYB_TYPE_FLOAT64) ? kTestFloat
                                                                                                                 : kTestInt;
  }
  for (uint32_t g = 0; g < query->groupby_count; ++g) plan.group_offset[g] = plan.columns[group_slot[g]].slot_offset;
  for (size_t c = 0; c < fast.columns.size(); ++c) {
    const DevSegment& segment = first[fast.columns[c].column];
    plan.value_offset[c] = plan.columns[value_slot[c]].slot_offset;
    plan.value_width[c] = max_width[value_slot[c]];
    plan.value_kind[c] = segment.encoding != HYB_ENC_DICTIONARY                              ? kValueBits
                         : max_dictionary[fast.columns[c].column] <= kStagedDictionary ? kValueStagedDictionary
                                                                                       : kValueGlobalDictionary;
    plan.dictionary_offset[c] = offset;
    offset += static_cast<uint32_t>(kStagedDictionary * value_size);
  }
  for (uint32_t g = 0; g < query->groupby_count; ++g) {
    plan.group_words_offset[g] = offset;
    offset += kMaxCombos * 8 + 16;
  }
  offset = (offset + 127u) & ~127u;
  plan.info_offset = offset;
  offset += (static_cast<uint32_t>(sizeof(StreamStageInfo)) + 127u) & ~127u;
  plan.stage_bytes = offset;
  plan.stage_count = std::min<uint32_t>(std::max<uint32_t>(stage_count, 2), kStreamMaxStages);
  while (plan.stage_count > 2 && size_t{plan.stage_count} * plan.stage_bytes > kStreamMaxDynamicBytes) --plan.stage_count;
  layout.dynamic_bytes = size_t{plan.stage_count} * plan.stage_bytes;
  if (layout.dynamic_bytes > kStreamMaxDynamicBytes) return layout;
  layout.possible = true;
  return layout;
}

static hyb_row_id position_to_row_id_host(const Table* table, uint64_t position) {
  const auto& starts = table->chunk_row_start;
  const auto it = std::upper_bound(starts.begin(), starts.end(), position);
  const uint32_t chunk = static_cast<uint32_t>(it - starts.begin()) - 1;
  return hyb_row_id{chunk, static_cast<uint32_t>(position - starts[chunk])};
}

static double double_from_ordered(uint64_t ordered) {
  const uint64_t bits = (ordered >> 63) ? (ordered & 0x7FFFFFFFFFFFFFFFull) : ~ordered;
  double value;
  std::memcpy(&value, &bits, sizeof(value));
  return value;
}

}  // namespace hyb

using namespace hyb;

static int exchange_partial_groups(hyb_context* context, const AggregateExchange& exchange, const Table* table,
                                   const hyb_aggregate_query* query, const std::vector<int32_t>& input_types,
                                   std::vector<HostGroup>* groups, bool* out_needs_partitioning);

static int exchange_partial_groups_partitioned(hyb_context* context, const AggregateExchange& exchange, const Table* table,
                                               const hyb_aggregate_query* query, const std::vector<int32_t>& input_types,
                                               std::vector<HostGroup>* groups, int* out_immediate);

// The INT32 dictionary descriptors of a string column (Table::StringColumnView) with `words` as per-chunk dictionaries:
// chunk c's dictionary starts at words + word_begin[c] (word_begin == nullptr: every chunk reads `words` itself).
static int build_string_view_segments(hyb_context* context, Table* table, uint32_t column, Table::StringColumnView* view,
                                      const uint64_t* word_begin) {
  const uint32_t chunk_count = table->chunk_count();
  std::vector<DevSegment> segments(chunk_count);
  for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
    DevSegment segment = table->segments[size_t{chunk} * table->column_count + column];
    HYB_CHECK(segment.encoding == HYB_ENC_DICTIONARY, HYB_ERR_UNSUPPORTED, "string aggregates need dictionary segments");
    segment.data_type = HYB_TYPE_INT32;  // dict_codes stay: COUNT(DISTINCT) of the same column reads them
    segment.values = view->d_words + (word_begin ? word_begin[chunk] : 0);
    segments[chunk] = segment;
  }
  HYB_TRY(device_alloc(context, sizeof(DevSegment) * std::max<uint32_t>(chunk_count, 1), reinterpret_cast<void**>(&view->d_segments)));
  if (chunk_count) {
    HYB_CUDA(cudaMemcpyAsync(view->d_segments, segments.data(), sizeof(DevSegment) * chunk_count, cudaMemcpyHostToDevice,
                             context->stream));
  }
  HYB_CUDA(cudaStreamSynchronize(context->stream));
  return HYB_OK;
}

// The view a string MIN / MAX (`need_order`) or COUNT reads. COUNT without attached ranks gets zero words: it tests the
// value-ID against the NULL value-ID only.
static int string_column_view(hyb_context* context, Table* table, uint32_t column, bool need_order,
                              Table::StringColumnView** out_view) {
  auto it = table->string_views.find(column);
  if (it == table->string_views.end()) {
    HYB_CHECK(!need_order, HYB_ERR_UNSUPPORTED,
              "MIN / MAX over string column " + std::to_string(column) + " needs hyb_table_set_string_order");
    auto view = std::make_shared<Table::StringColumnView>();
    view->owner = context;
    uint32_t max_dictionary = 0;
    for (uint32_t chunk = 0; chunk < table->chunk_count(); ++chunk) {
      max_dictionary = std::max(max_dictionary, table->segments[size_t{chunk} * table->column_count + column].dict_size);
    }
    HYB_TRY(device_alloc(context, sizeof(uint32_t) * (size_t{max_dictionary} + 1), reinterpret_cast<void**>(&view->d_words)));
    HYB_CUDA(cudaMemsetAsync(view->d_words, 0, sizeof(uint32_t) * (size_t{max_dictionary} + 1), context->stream));
    HYB_TRY(build_string_view_segments(context, table, column, view.get(), nullptr));
    it = table->string_views.emplace(column, std::move(view)).first;
  }
  HYB_CHECK(!need_order || it->second->ordered, HYB_ERR_UNSUPPORTED,
            "MIN / MAX over string column " + std::to_string(column) + " needs hyb_table_set_string_order");
  *out_view = it->second.get();
  return HYB_OK;
}

extern "C" int hyb_table_set_string_order(hyb_context* context, hyb_table_t handle, uint32_t column, const uint32_t* ranks,
                                          uint64_t count) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* table = find_table(context, handle);
  HYB_CHECK(table, HYB_ERR_NOT_FOUND, "unknown table handle");
  HYB_CHECK(column < table->column_count && table->column_types[column] == HYB_TYPE_STRING, HYB_ERR_INVALID,
            "not a string column");
  const uint32_t chunk_count = table->chunk_count();
  std::vector<uint64_t> word_begin(size_t{chunk_count} + 1, 0);
  for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
    const DevSegment& segment = table->segments[size_t{chunk} * table->column_count + column];
    HYB_CHECK(segment.encoding == HYB_ENC_DICTIONARY, HYB_ERR_INVALID, "not a string dictionary column");
    word_begin[chunk + 1] = word_begin[chunk] + segment.dict_size;
  }
  HYB_CHECK(count == word_begin.back(), HYB_ERR_INVALID,
            "expected " + std::to_string(word_begin.back()) + " rank words (one per dictionary entry), got " + std::to_string(count));
  HYB_CHECK(ranks || count == 0, HYB_ERR_INVALID, "ranks is NULL");
  uint32_t max_rank = 0;
  for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
    for (uint64_t word = word_begin[chunk]; word < word_begin[chunk + 1]; ++word) {
      // dense ranks stay below the word count; that also bounds the rank -> first entry table by it
      HYB_CHECK(ranks[word] < (1u << 31) && ranks[word] < count, HYB_ERR_INVALID,
                "rank words must be below 2^31 and below their count");
      HYB_CHECK(word == word_begin[chunk] || ranks[word] > ranks[word - 1], HYB_ERR_INVALID,
                "rank words must be strictly increasing within chunk " + std::to_string(chunk));
      max_rank = std::max(max_rank, ranks[word]);
    }
  }
  HYB_TRY(sync_table_descriptors(context, table));  // before the view: a pending descriptor sync drops views
  auto view = std::make_shared<Table::StringColumnView>();
  view->owner = context;
  view->ordered = true;
  view->word_count = count;
  const uint64_t distinct_bound = count ? uint64_t{max_rank} + 1 : 1;
  HYB_TRY(device_alloc(context, sizeof(uint32_t) * std::max<uint64_t>(count, 1), reinterpret_cast<void**>(&view->d_words)));
  HYB_TRY(device_alloc(context, sizeof(unsigned long long) * distinct_bound, reinterpret_cast<void**>(&view->d_first_entry)));
  uint64_t* d_word_begin = nullptr;
  HYB_TRY(device_alloc(context, sizeof(uint64_t) * word_begin.size(), reinterpret_cast<void**>(&d_word_begin)));
  DeviceScratch scratch(context);
  scratch.adopt(d_word_begin);
  if (count) HYB_CUDA(cudaMemcpyAsync(view->d_words, ranks, sizeof(uint32_t) * count, cudaMemcpyHostToDevice, context->stream));
  HYB_CUDA(cudaMemcpyAsync(d_word_begin, word_begin.data(), sizeof(uint64_t) * word_begin.size(), cudaMemcpyHostToDevice,
                           context->stream));
  HYB_CUDA(cudaMemsetAsync(view->d_first_entry, 0xFF, sizeof(unsigned long long) * distinct_bound, context->stream));
  if (chunk_count) {
    string_order_first_entry_kernel<<<std::min<uint32_t>(chunk_count, context->sm_count * 8), 256, 0, context->stream>>>(
        view->d_words, d_word_begin, chunk_count, view->d_first_entry);
    HYB_CUDA(cudaGetLastError());
  }
  HYB_TRY(build_string_view_segments(context, table, column, view.get(), word_begin.data()));
  table->string_views[column] = std::move(view);
  return HYB_OK;
}

// Per (table, query shape): what the descriptor walk found. See Table::plan_memo.
struct AggregatePlanMemo {
  uint64_t algorithmic_bytes = 0;
  bool has_stream_layout = false;
  uint32_t stream_stages = 0;
  StreamLayout stream_layout;
};

static std::string aggregate_signature(const hyb_aggregate_query* query) {
  std::string signature = "agg";
  const auto add = [&](const void* data, size_t bytes) { signature.append(static_cast<const char*>(data), bytes); };
  add(&query->predicate_count, sizeof(query->predicate_count));
  for (uint32_t p = 0; p < query->predicate_count; ++p) {
    add(&query->predicates[p].column_id, sizeof(uint32_t));
    add(&query->predicates[p].condition, sizeof(int32_t));
  }
  add(&query->groupby_count, sizeof(query->groupby_count));
  for (uint32_t g = 0; g < query->groupby_count; ++g) add(&query->groupby_column_ids[g], sizeof(uint32_t));
  add(&query->aggregate_count, sizeof(query->aggregate_count));
  for (uint32_t a = 0; a < query->aggregate_count; ++a) {
    const auto& def = query->aggregates[a];
    add(&def.function, sizeof(def.function));
    add(&def.node_count, sizeof(def.node_count));
    for (uint32_t n = 0; n < def.node_count; ++n) add(&def.nodes[n], sizeof(def.nodes[n]));
  }
  return signature;
}

// Whether an aggregate's expression reads a string column of `table` (a column out of range is rejected when it is typed).
static bool has_string_argument(const Table* table, const hyb_aggregate_def& def) {
  return std::any_of(def.nodes, def.nodes + def.node_count, [&](const auto& node) {
    return node.op == HYB_EXPR_COLUMN && node.column_id < table->column_count &&
           table->column_types[node.column_id] == HYB_TYPE_STRING;
  });
}

struct AggregateTypes {
  std::vector<int32_t> input_types, result_types;
  // MIN / MAX / COUNT of a bare string column: the column's INT32 view (order ranks, or zeros for COUNT)
  std::vector<Table::StringColumnView*> string_views;
};

// Validates the aggregates (ANY already stripped) and the group-by columns, and types every aggregate.
static int type_aggregates(hyb_context* context, Table* table, const hyb_aggregate_query* query, AggregateTypes* out) {
  const uint32_t aggregate_count = query->aggregate_count;
  const uint32_t chunk_count = table->chunk_count();
  out->input_types.assign(aggregate_count, HYB_TYPE_INT64);
  out->result_types.assign(aggregate_count, HYB_TYPE_INT64);
  out->string_views.assign(aggregate_count, nullptr);
  for (uint32_t a = 0; a < aggregate_count; ++a) {
    const auto& def = query->aggregates[a];
    HYB_CHECK(def.function >= HYB_AGG_MIN && def.function <= HYB_AGG_STDDEV_SAMP, HYB_ERR_UNSUPPORTED,
              "aggregate function " + std::to_string(def.function) + " runs on the CPU operator");
    if (def.function == HYB_AGG_COUNT_STAR) continue;
    HYB_CHECK(def.node_count >= 1 && def.node_count <= HYB_MAX_EXPR_NODES, HYB_ERR_INVALID, "bad expression length");
    const bool string_argument = has_string_argument(table, def);
    if (string_argument && def.function == HYB_AGG_STDDEV_SAMP) {
      HYB_CHECK(false, HYB_ERR_INVALID, "STDDEV_SAMP is not defined for strings");
    }
    if (string_argument && def.function == HYB_AGG_COUNT_DISTINCT) {
      // A bare column whose dictionaries carry the chunk-independent codes string group-by uses: equal codes <=> equal
      // strings, so the codes stand in for the values.
      HYB_CHECK(def.node_count == 1 && def.nodes[0].op == HYB_EXPR_COLUMN, HYB_ERR_UNSUPPORTED,
                "COUNT(DISTINCT) over a string expression runs on the CPU operator");
      for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
        const auto& segment = table->segments[size_t{chunk} * table->column_count + def.nodes[0].column_id];
        HYB_CHECK(segment.encoding == HYB_ENC_DICTIONARY && segment.dict_codes, HYB_ERR_UNSUPPORTED,
                  "COUNT(DISTINCT) over a string column needs dictionary_codes in its segments");
      }
      out->input_types[a] = HYB_TYPE_STRING;
      out->result_types[a] = HYB_TYPE_INT64;
      continue;
    }
    const bool bare_column = def.node_count == 1 && def.nodes[0].op == HYB_EXPR_COLUMN;
    if (string_argument && bare_column &&
        (def.function == HYB_AGG_MIN || def.function == HYB_AGG_MAX || def.function == HYB_AGG_COUNT)) {
      HYB_TRY(string_column_view(context, table, def.nodes[0].column_id, def.function != HYB_AGG_COUNT,
                                 &out->string_views[a]));
      out->input_types[a] = HYB_TYPE_STRING;
      out->result_types[a] = def.function == HYB_AGG_COUNT ? HYB_TYPE_INT64 : HYB_TYPE_STRING;
      continue;
    }
    HYB_TRY(expression_type(table, def, &out->input_types[a]));
    out->result_types[a] = aggregate_result_type(def.function, out->input_types[a]);
  }
  for (uint32_t g = 0; g < query->groupby_count; ++g) {
    const uint32_t column = query->groupby_column_ids[g];
    HYB_CHECK(column < table->column_count, HYB_ERR_INVALID, "group-by column out of range");
    if (table->column_types[column] == HYB_TYPE_STRING) {
      for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
        HYB_CHECK(table->segments[size_t{chunk} * table->column_count + column].dict_codes, HYB_ERR_UNSUPPORTED,
                  "grouping by a string column needs dictionary_codes in its segments");
      }
    }
  }
  return HYB_OK;
}

struct FusedPredicates {
  std::vector<ChunkTest*> tests;      // per fused predicate
  const TestProgram* tree = nullptr;  // the expression tree's programs (hyb_aggregate_hash_expression), or none
  uint32_t launches = 0;              // the kernels that built the tests
};

// The fused predicates' per-chunk tests and the expression tree's tests and programs, all owned by `scratch`.
static int prepare_fused_predicates(hyb_context* context, Table* table, const hyb_aggregate_query* query,
                                    ExpressionTree* tree, DeviceScratch& scratch, FusedPredicates* out) {
  out->tests.assign(query->predicate_count, nullptr);
  for (uint32_t p = 0; p < query->predicate_count; ++p) {
    void* bounds = nullptr;
    HYB_TRY(prepare_chunk_tests(context, table, &query->predicates[p], &out->tests[p], &bounds));
    scratch.adopt(out->tests[p]);
    scratch.adopt(bounds);
    ++out->launches;
  }
  if (tree) {
    HYB_TRY(upload_expression_tree(context, table, *tree, scratch));
    out->tree = tree->device;
    out->launches += tree->launches;
  }
  return HYB_OK;
}

// The rank words string MIN / MAX read as their dictionaries, each view once (`ordered_only`: views with ranks only).
static uint64_t rank_word_bytes(const AggregateTypes& types, bool ordered_only) {
  std::vector<const Table::StringColumnView*> ranked;
  uint64_t bytes = 0;
  for (size_t a = 0; a < types.string_views.size(); ++a) {
    const Table::StringColumnView* view = types.string_views[a];
    if (view && (!ordered_only || view->ordered) && types.result_types[a] == HYB_TYPE_STRING &&
        std::find(ranked.begin(), ranked.end(), view) == ranked.end()) {
      ranked.push_back(view);
      bytes += sizeof(uint32_t) * view->word_count;
    }
  }
  return bytes;
}

// hyb_operator_stats::algorithmic_bytes: every referenced column once (kept in the memo), or one RowID per position of
// a filtered input; plus the expression tree's uploads and, on filtered inputs, the rank words.
static uint64_t aggregate_algorithmic_bytes(const Table* table, const hyb_aggregate_query* query, const ExpressionTree* tree,
                                            const AggregateTypes& types, const PosList* filter, uint64_t position_count,
                                            AggregatePlanMemo* memo) {
  if (memo->algorithmic_bytes == 0) {
    // bytes of every referenced column, each counted once
    std::vector<uint32_t> referenced;
    for (uint32_t p = 0; p < query->predicate_count; ++p) referenced.push_back(query->predicates[p].column_id);
    for (uint32_t g = 0; g < query->groupby_count; ++g) referenced.push_back(query->groupby_column_ids[g]);
    if (tree) {
      referenced.insert(referenced.end(), tree->test_columns, tree->test_columns + tree->host.column_count);
      referenced.insert(referenced.end(), tree->column_ids, tree->column_ids + tree->program.column_count);
    }
    for (uint32_t a = 0; a < query->aggregate_count; ++a) {
      for (uint32_t n = 0; n < query->aggregates[a].node_count; ++n) {
        if (query->aggregates[a].nodes[n].op == HYB_EXPR_COLUMN) referenced.push_back(query->aggregates[a].nodes[n].column_id);
      }
    }
    std::sort(referenced.begin(), referenced.end());
    referenced.erase(std::unique(referenced.begin(), referenced.end()), referenced.end());
    for (const uint32_t column : referenced) {
      for (uint32_t chunk = 0; chunk < table->chunk_count(); ++chunk) {
        const auto& segment = table->segments[size_t{chunk} * table->column_count + column];
        if (segment.encoding == HYB_ENC_UNENCODED) {
          memo->algorithmic_bytes += data_type_size(segment.data_type) * segment.row_count;
        } else {
          memo->algorithmic_bytes += vector_bytes(segment.vector_type, segment.bit_width, segment.row_count);
          if (segment.encoding == HYB_ENC_DICTIONARY && segment.data_type != HYB_TYPE_STRING) {
            memo->algorithmic_bytes += data_type_size(segment.data_type) * segment.dict_size;
          }
          if (segment.encoding == HYB_ENC_FRAME_OF_REFERENCE) {
            memo->algorithmic_bytes += sizeof(int32_t) * ((segment.row_count + HYB_FOR_BLOCK_SIZE - 1) / HYB_FOR_BLOCK_SIZE);
          }
        }
        if (segment.nulls) memo->algorithmic_bytes += segment.row_count;
      }
    }
    memo->algorithmic_bytes += rank_word_bytes(types, true);  // string MIN / MAX read the column's rank words
  }
  uint64_t bytes = filter ? position_count * sizeof(hyb_row_id) : memo->algorithmic_bytes;
  if (tree) bytes += tree->uploaded_bytes;       // the leaves' tests, bitmaps and intervals, and the programs
  if (filter) bytes += rank_word_bytes(types, false);  // string MIN / MAX read their rank words on filtered inputs too
  return bytes;
}

// What both kernels' plans read besides their own fields: the fused predicates' segments and tests, the group-by segments.
template <typename Plan>
static void plan_inputs(const Table* table, const hyb_aggregate_query* query, const FusedPredicates& fused, Plan* plan) {
  const uint32_t chunk_count = table->chunk_count();
  plan->chunk_row_start = reinterpret_cast<const unsigned long long*>(table->d_chunk_row_start);
  plan->predicate_count = query->predicate_count;
  for (uint32_t p = 0; p < query->predicate_count; ++p) {
    plan->predicate_segments[p] = table->d_segments + size_t{query->predicates[p].column_id} * chunk_count;
    plan->predicate_tests[p] = fused.tests[p];
  }
  plan->groupby_count = query->groupby_count;
  for (uint32_t g = 0; g < query->groupby_count; ++g) {
    plan->group_segments[g] = table->d_segments + size_t{query->groupby_column_ids[g]} * chunk_count;
  }
}

// This rank's groups, the kernel they came from (hyb_operator_stats::path), the launches so far and the timed span.
struct AggregateOutcome {
  bool done = false;
  std::vector<HostGroup> groups;
  uint32_t path = HYB_AGG_PATH_NONE;
  uint32_t launches = 0;
  bool kernel_timed = false;
};

// Offsets (64-bit words) in the fast path's partials block of `entries` (CTA x group slot) entries and C value columns.
// The copy back to the host covers all `words`; the device FastPlan follows them.
struct FastPartials {
  size_t hash, keys, rows, min_position, max_position, raw, product, raw_nulls, product_nulls, null_mask, overflow, words;
  FastPartials(size_t entries, size_t C)
      : hash(0), keys(hash + entries), rows(keys + entries * kMaxKeyWords), min_position(rows + entries),
        max_position(min_position + entries), raw(max_position + entries), product(raw + entries * C),
        raw_nulls(product + entries * C), product_nulls(raw_nulls + entries * C), null_mask(product_nulls + entries * C),
        overflow(null_mask + (entries + 1) / 2), words(overflow + 1) {}
};

// Merges the per-CTA partials in CTA order (deterministic). false: two groups share a 64-bit hash.
static bool merge_fast_partials(const hyb_aggregate_query* query, const FastPlanHost& fast, const std::vector<uint64_t>& host,
                                const FastPartials& layout, size_t entries, int C, std::vector<HostGroup>* groups) {
  struct Merged {
    uint64_t hash;
    std::vector<uint64_t> key;
    uint32_t null_mask;
    uint64_t rows = 0, min_position = ~uint64_t{0}, max_position = 0;
    std::vector<double> raw_f, product_f;
    std::vector<int64_t> raw_i;
    std::vector<uint64_t> raw_nulls, product_nulls;
  };
  const auto* null_masks = reinterpret_cast<const uint32_t*>(&host[layout.null_mask]);
  std::vector<Merged> merged;
  bool consistent = true;
  for (size_t entry = 0; entry < entries; ++entry) {
    const uint64_t hash = host[layout.hash + entry];
    if (hash == 0 || host[layout.rows + entry] == 0) continue;
    const uint64_t* key_words = &host[layout.keys + entry * kMaxKeyWords];
    std::vector<uint64_t> key(key_words, key_words + std::max<uint32_t>(query->groupby_count, 1));
    Merged* target = nullptr;
    for (auto& m : merged) {
      if (m.hash == hash) {
        if (m.key != key || m.null_mask != null_masks[entry]) consistent = false;  // 64-bit hash collision
        target = &m;
      }
    }
    if (!target) {
      merged.emplace_back();
      target = &merged.back();
      target->hash = hash;
      target->key = key;
      target->null_mask = null_masks[entry];
      target->raw_f.assign(C, 0.0);
      target->product_f.assign(C, 0.0);
      target->raw_i.assign(C, 0);
      target->raw_nulls.assign(C, 0);
      target->product_nulls.assign(C, 0);
    }
    target->rows += host[layout.rows + entry];
    target->min_position = std::min(target->min_position, host[layout.min_position + entry]);
    target->max_position = std::max(target->max_position, host[layout.max_position + entry]);
    for (int c = 0; c < C; ++c) {
      const size_t at = entry * C + c;
      if (fast.work_type == 2) {
        target->raw_i[c] += static_cast<int64_t>(host[layout.raw + at]);
      } else {
        double raw, product;
        std::memcpy(&raw, &host[layout.raw + at], sizeof(double));
        std::memcpy(&product, &host[layout.product + at], sizeof(double));
        target->raw_f[c] += raw;
        target->product_f[c] += product;
      }
      target->raw_nulls[c] += host[layout.raw_nulls + at];
      target->product_nulls[c] += host[layout.product_nulls + at];
    }
  }
  if (!consistent) return false;
  for (const auto& m : merged) {
    HostGroup group;
    group.key = m.key;
    group.null_mask = m.null_mask;
    group.rows = m.rows;
    group.min_position = m.min_position;
    group.max_position = m.max_position;
    group.accumulators.assign(query->aggregate_count, 0);
    group.counts.assign(query->aggregate_count, 0);
    for (uint32_t a = 0; a < query->aggregate_count; ++a) {
      const auto& mapping = fast.mapping[a];
      if (mapping.is_count_star) {
        group.counts[a] = m.rows;
        continue;
      }
      const uint32_t slot = mapping.column_slot;
      const uint64_t nulls = mapping.uses_product ? m.product_nulls[slot] : m.raw_nulls[slot];
      group.counts[a] = m.rows - nulls;
      if (fast.work_type == 2) {
        const int64_t sum = m.raw_i[slot];
        std::memcpy(&group.accumulators[a], &sum, sizeof(sum));
      } else {
        const double sum = mapping.uses_product ? m.product_f[slot] : m.raw_f[slot];
        std::memcpy(&group.accumulators[a], &sum, sizeof(sum));
      }
    }
    groups->push_back(std::move(group));
  }
  return true;
}

// The low-cardinality kernels over unfiltered inputs. Attempts in order: the TMA-staged streaming kernel when the layout
// allows it (<= 4 groups), then the register-tile kernel with 4 and 8 group slots; a kernel that meets more groups than
// it has slots raises `overflow`. out->done stays false when no attempt holds the groups or two groups share a hash.
static int run_fast_path(hyb_context* context, Table* table, const hyb_aggregate_query* query, const FusedPredicates& fused,
                         AggregatePlanMemo* memo, AggregateOutcome* out) {
  const FastPlanHost fast = plan_fast_path(table, query);
  const uint32_t chunk_count = table->chunk_count();
  if (!fast.possible || chunk_count == 0) return HYB_OK;
  cudaStream_t stream = context->stream;
  const int C = fast.columns.size() <= 1 ? 1 : fast.columns.size() <= 2 ? 2 : 4;
  struct Attempt {
    bool stream;
    int groups;
  };
  std::vector<Attempt> attempts;
  StreamLayout stream_layout;
  if (context->options.aggregate_stream) {
    if (!memo->has_stream_layout || memo->stream_stages != context->options.aggregate_stages) {
      memo->stream_layout = stream_layout_for(table, query, fast, context->options.aggregate_stages, fused.tree != nullptr);
      memo->stream_stages = context->options.aggregate_stages;
      memo->has_stream_layout = true;
    }
    stream_layout = memo->stream_layout;
  }
  if (stream_layout.possible) attempts.push_back({true, query->groupby_count == 0 ? 1 : 4});
  if (query->groupby_count == 0) {
    attempts.push_back({false, 1});
  } else {
    attempts.push_back({false, 4});
    attempts.push_back({false, 8});
  }
  for (const Attempt attempt : attempts) {
    const uint2* tile_map = nullptr;
    uint32_t tile_count = 0;
    HYB_TRY(get_tile_map(context, table, attempt.stream ? kStreamTileRows : kAggTileRows, &tile_map, &tile_count));
    const int G = attempt.groups;
    const FastKernel kernel = fast_kernel(fast.work_type, G, C, fused.tree != nullptr);
    uint32_t grid = 1;
    if (attempt.stream) {
      // one persistent CTA per SM; its tiles are kStreamRounds contiguous runs, the runs strided over the CTAs
      grid = std::max<uint32_t>(1, std::min<uint32_t>(tile_count, context->sm_count));
    } else {
      int blocks_per_sm = 1;
      HYB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kernel, kFastThreads, 0));
      // one wave of resident CTAs: the static tile striding must not queue CTAs behind each other
      grid = std::max<uint32_t>(1, std::min<uint32_t>(tile_count, context->sm_count * std::max(blocks_per_sm, 1)));
    }
    FastPlan host_plan{};
    plan_inputs(table, query, fused, &host_plan);
    host_plan.size_segments = table->d_segments;
    host_plan.tile_map = tile_map;
    host_plan.tile_count = tile_count;
    for (size_t c = 0; c < fast.columns.size(); ++c) {
      host_plan.value_segments[c] = table->d_segments + size_t{fast.columns[c].column} * chunk_count;
      host_plan.affine_kind[c] = fast.columns[c].kind;
      host_plan.literal[c] = fast.columns[c].literal;
    }
    host_plan.need_raw_mask = fast.need_raw_mask;
    host_plan.need_product_mask = fast.need_product_mask;
    const size_t entries = size_t{grid} * G;
    const FastPartials layout(entries, C);
    std::vector<uint64_t> host(layout.words);
    {
      DeviceScratch scratch(context);  // this attempt's partials and plan
      const size_t bytes = sizeof(uint64_t) * layout.words + sizeof(FastPlan) + 64;
      void* block = nullptr;
      HYB_TRY(scratch.alloc(bytes, &block));
      HYB_CUDA(cudaMemsetAsync(block, 0, bytes, stream));
      auto* partials = static_cast<unsigned long long*>(block);
      host_plan.partial_hash = partials + layout.hash;
      host_plan.partial_keys = partials + layout.keys;
      host_plan.partial_rows = partials + layout.rows;
      host_plan.partial_min_position = partials + layout.min_position;
      host_plan.partial_max_position = partials + layout.max_position;
      host_plan.partial_raw = partials + layout.raw;
      host_plan.partial_product = partials + layout.product;
      host_plan.partial_raw_nulls = partials + layout.raw_nulls;
      host_plan.partial_product_nulls = partials + layout.product_nulls;
      host_plan.partial_null_mask = reinterpret_cast<uint32_t*>(partials + layout.null_mask);
      host_plan.overflow = reinterpret_cast<uint32_t*>(partials + layout.overflow);
      auto* device_plan = reinterpret_cast<FastPlan*>(partials + layout.words);
      if (attempt.stream) {
        StreamPlan stream_plan = stream_layout.plan;
        stream_plan.fast = host_plan;
        stream_plan.unit_tiles = std::max<uint32_t>(1, (tile_count + grid * kStreamRounds - 1) / (grid * kStreamRounds));
        const uint64_t shape = context->options.aggregate_static_shapes ? stream_shape_of(stream_plan, host_plan, static_cast<uint32_t>(C)) : 0;
        bool static_shape = false;
        void* stream_kernel = fast.work_type == 0 ? stream_kernel_for<0>(G, C, shape, &static_shape)
                                                  : stream_kernel_for<1>(G, C, shape, &static_shape);
        if (context->options.trace) {
          std::fprintf(stderr, "[hyb] aggregate_stream_kernel<%d, %d, %d> shape %#llx (%s)\n", fast.work_type, G, C,
                       static_cast<unsigned long long>(shape), static_shape ? "static instantiation" : "layout-generic");
        }
        HYB_CUDA(cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(stream_layout.dynamic_bytes)));
        void* arguments[] = {&stream_plan};
        timing_kernel_begin(context);
        HYB_CUDA(cudaLaunchKernel(stream_kernel, dim3(grid), dim3(kStreamThreads), arguments, stream_layout.dynamic_bytes, stream));
        timing_kernel_end(context);
        out->path = static_shape ? HYB_AGG_PATH_STREAM_STATIC : HYB_AGG_PATH_STREAM_GENERIC;
      } else {
        HYB_CUDA(cudaMemcpyAsync(device_plan, &host_plan, sizeof(FastPlan), cudaMemcpyHostToDevice, stream));
        const TestProgram* tree_program = fused.tree;
        void* arguments[] = {&device_plan, &tree_program};  // aggregate_fast_kernel takes the first only
        timing_kernel_begin(context);
        HYB_CUDA(cudaLaunchKernel(kernel, dim3(grid), dim3(kFastThreads), arguments, 0, stream));
        timing_kernel_end(context);
        out->path = G <= 4 ? HYB_AGG_PATH_TILE_G4 : HYB_AGG_PATH_TILE_G8;
      }
      out->kernel_timed = true;
      HYB_CUDA(cudaGetLastError());
      ++out->launches;
      HYB_CUDA(cudaMemcpyAsync(host.data(), block, sizeof(uint64_t) * layout.words, cudaMemcpyDeviceToHost, stream));
      HYB_CUDA(cudaStreamSynchronize(stream));
    }
    const uint32_t overflow = *reinterpret_cast<const uint32_t*>(&host[layout.overflow]);
    if (overflow) continue;  // more groups than this instantiation holds
    out->done = merge_fast_partials(query, fast, host, layout, entries, C, &out->groups);
    break;  // a hash collision falls through to the general path
  }
  return HYB_OK;
}

// One sweep of aggregate_general_kernel over the plan's rows; with an expression tree, its kTreeRows form.
template <int kSweep>
static void launch_general_sweep(bool tree, uint32_t grid, cudaStream_t stream, const AggregatePlan* plan,
                                 const GroupTable& group_table, const GroupTable& distinct_table) {
  if (tree) {
    aggregate_general_kernel<kSweep | kTreeRows><<<grid, kAggThreads, 0, stream>>>(plan, group_table, distinct_table);
  } else {
    aggregate_general_kernel<kSweep><<<grid, kAggThreads, 0, stream>>>(plan, group_table, distinct_table);
  }
}

// The groups of aggregate_compact_kernel's packed copy of `slots` slots; MIN / MAX and STDDEV_SAMP get their values.
static void parse_packed_groups(const hyb_aggregate_query* query, const AggregateTypes& types, const uint64_t* words,
                                uint64_t slots, uint32_t key_words, size_t compact_words, std::vector<HostGroup>* groups) {
  const uint32_t aggregate_count = query->aggregate_count;
  const uint64_t* h_hashes = words;
  const uint64_t* h_keys = h_hashes + slots;
  const uint64_t* h_rows = h_keys + slots * key_words;
  const uint64_t* h_min = h_rows + slots;
  const uint64_t* h_max = h_min + slots;
  const uint64_t* h_acc = h_max + slots;
  const uint64_t* h_counts = h_acc + slots * aggregate_count;
  const uint64_t* h_zero_first = h_counts + slots * aggregate_count;
  const uint64_t* h_moments = h_zero_first + slots * aggregate_count;  // STDDEV_SAMP plans: {Σd, Σd²} per aggregate
  const uint32_t* h_null_masks = reinterpret_cast<const uint32_t*>(words + compact_words);
  for (uint64_t slot = 0; slot < slots; ++slot) {
    if (h_hashes[slot] == 0) continue;
    HostGroup group;
    group.key.assign(h_keys + slot * key_words, h_keys + (slot + 1) * key_words);
    group.null_mask = h_null_masks[slot];
    group.rows = h_rows[slot];
    group.min_position = h_min[slot];
    group.max_position = h_max[slot];
    group.accumulators.resize(aggregate_count);
    group.counts.resize(aggregate_count);
    for (uint32_t a = 0; a < aggregate_count; ++a) {
      group.accumulators[a] = h_acc[size_t{a} * slots + slot];
      group.counts[a] = query->aggregates[a].function == HYB_AGG_COUNT_STAR ? group.rows : h_counts[size_t{a} * slots + slot];
      const int32_t function = query->aggregates[a].function;
      if (function == HYB_AGG_STDDEV_SAMP && group.counts[a] > 1) {
        // M2 = Σd² - (Σd)² / n; rounding may leave it a hair below 0 where Welford's M2 cannot go. Only a negative M2
        // is clamped: a NaN (a NaN or an infinity in the group) stays NaN, as in the reference's Welford.
        double sum_d, sum_d2;
        std::memcpy(&sum_d, h_moments + (size_t{a} * 2) * slots + slot, sizeof(double));
        std::memcpy(&sum_d2, h_moments + (size_t{a} * 2 + 1) * slots + slot, sizeof(double));
        const double n = static_cast<double>(group.counts[a]);
        double m2 = sum_d2 - sum_d * sum_d / n;
        if (m2 < 0.0) m2 = 0.0;
        const double deviation = std::sqrt(m2 / (n - 1.0));
        std::memcpy(&group.accumulators[a], &deviation, sizeof(deviation));
      }
      const int32_t input_type = types.input_types[a];
      if ((function == HYB_AGG_MIN || function == HYB_AGG_MAX) && group.counts[a] > 0 && input_type != HYB_TYPE_STRING) {
        if (input_type == HYB_TYPE_INT32 || input_type == HYB_TYPE_INT64) {
          group.accumulators[a] ^= 0x8000000000000000ull;
        } else {
          double value = double_from_ordered(group.accumulators[a]);
          if (value == 0.0 && (h_zero_first[size_t{a} * slots + slot] & 1)) value = -0.0;  // the first zero was -0.0
          std::memcpy(&group.accumulators[a], &value, sizeof(value));
        }
      }
    }
    groups->push_back(std::move(group));
  }
}

// The hash table kernel over any input. Grows the group table (and the COUNT(DISTINCT) set) by 8x until the kernel
// finds no overflow, then runs the STDDEV_SAMP and string MIN / MAX passes and packs the occupied slots for the host.
static int run_general_path(hyb_context* context, Table* table, const hyb_aggregate_query* query, const PosList* filter,
                            uint64_t position_count, const AggregateTypes& types, const FusedPredicates& fused,
                            AggregateOutcome* out) {
  cudaStream_t stream = context->stream;
  const uint32_t aggregate_count = query->aggregate_count;
  const bool tree = fused.tree != nullptr;
  const uint32_t chunk_count = table->chunk_count();
  AggregatePlan host_plan{};
  if (filter) {
    host_plan.filter = filter->d_row_ids;
    host_plan.tile_count = static_cast<uint32_t>((position_count + kAggTileRows - 1) / kAggTileRows);
  } else {
    HYB_TRY(get_tile_map(context, table, kAggTileRows, &host_plan.tile_map, &host_plan.tile_count));
  }
  plan_inputs(table, query, fused, &host_plan);
  host_plan.position_count = position_count;
  host_plan.chunk_count = chunk_count;
  if (query->groupby_count == 0) host_plan.group_segments[0] = table->d_segments;  // sizes chunks when nothing else does
  host_plan.aggregate_count = aggregate_count;
  host_plan.tree = fused.tree;
  std::vector<uint32_t> plan_columns;
  for (uint32_t a = 0; a < query->aggregate_count; ++a) {
    const auto& def = query->aggregates[a];
    auto& device_aggregate = host_plan.aggregates[a];
    device_aggregate.function = def.function;
    device_aggregate.node_count = def.function == HYB_AGG_COUNT_STAR ? 0 : def.node_count;
    device_aggregate.input_type = types.input_types[a];
    device_aggregate.result_type = types.result_types[a];
    for (uint32_t n = 0; n < device_aggregate.node_count; ++n) {
      auto& node = device_aggregate.nodes[n];
      node.op = def.nodes[n].op;
      node.literal_type = def.nodes[n].literal_type;
      node.literal = def.nodes[n].literal;
      if (node.op == HYB_EXPR_COLUMN) {
        auto it = std::find(plan_columns.begin(), plan_columns.end(), def.nodes[n].column_id);
        if (it == plan_columns.end()) {
          plan_columns.push_back(def.nodes[n].column_id);
          it = plan_columns.end() - 1;
        }
        node.column = static_cast<uint32_t>(it - plan_columns.begin());
      }
    }
  }
  HYB_CHECK(plan_columns.size() <= HYB_MAX_AGGREGATES * 4, HYB_ERR_UNSUPPORTED, "too many distinct aggregate columns");
  host_plan.column_count = static_cast<uint32_t>(plan_columns.size());
  for (size_t c = 0; c < plan_columns.size(); ++c) {
    host_plan.columns[c] = table->d_segments + size_t{plan_columns[c]} * chunk_count;
  }
  // a string column that a MIN / MAX / COUNT reads is its INT32 view for every aggregate of the plan (the view keeps
  // the dictionary codes a COUNT(DISTINCT) of the same column reads)
  StringExtremes string_extremes{};
  bool has_string_extremes = false;
  for (uint32_t a = 0; a < aggregate_count; ++a) {
    if (!types.string_views[a]) continue;
    host_plan.columns[host_plan.aggregates[a].nodes[0].column] = types.string_views[a]->d_segments;
    if (types.result_types[a] == HYB_TYPE_STRING) {
      string_extremes.first_entry[a] = types.string_views[a]->d_first_entry;
      has_string_extremes = true;
    }
  }
  DeviceScratch plan_scratch(context);
  AggregatePlan* device_plan = nullptr;
  HYB_TRY(plan_scratch.alloc_array(1, &device_plan));
  HYB_CUDA(cudaMemcpyAsync(device_plan, &host_plan, sizeof(AggregatePlan), cudaMemcpyHostToDevice, stream));
  HYB_CUDA(cudaStreamSynchronize(stream));  // host_plan is on the stack

  uint64_t capacity = 1024;
  while (capacity < std::min<uint64_t>(position_count * 2, uint64_t{1} << 20)) capacity <<= 1;
  uint64_t distinct_capacity = capacity;  // the COUNT(DISTINCT) set starts at the group table's size
  const uint32_t key_words = std::max<uint32_t>(query->groupby_count, 1);
  uint32_t distinct_mask = 0, stddev_mask = 0;
  for (uint32_t a = 0; a < aggregate_count; ++a) {
    if (query->aggregates[a].function == HYB_AGG_COUNT_DISTINCT) distinct_mask |= 1u << a;
    if (query->aggregates[a].function == HYB_AGG_STDDEV_SAMP) stddev_mask |= 1u << a;
  }
  const uint32_t grid = std::max<uint32_t>(1, std::min<uint32_t>(host_plan.tile_count, context->sm_count * 8));
  out->path = HYB_AGG_PATH_GENERAL;
  while (!out->done) {
    // more {group, value} pairs than a set of 2^31 slots holds at load factor 0.5: the CPU operator counts them
    HYB_CHECK(distinct_capacity <= (uint64_t{1} << 31), HYB_ERR_UNSUPPORTED, "COUNT(DISTINCT) set would exceed 2^31 slots");
    HYB_CHECK(capacity <= (uint64_t{1} << 31), HYB_ERR_OOM, "group table would exceed 2^31 slots");
    // moments: {mean, Σd, Σd²} per aggregate and slot on the device; the packed copy carries {Σd, Σd²}
    const size_t moment_words = stddev_mask ? 3 * size_t{aggregate_count} : 0;
    const size_t per_slot_words = 1 + key_words + 3 + 3 * size_t{aggregate_count} + (stddev_mask ? 2 * size_t{aggregate_count} : 0);
    const size_t bytes = sizeof(uint64_t) * capacity * (1 + key_words + 3 + 3 * size_t{aggregate_count} + moment_words) +
                         sizeof(uint32_t) * capacity * 2 + 64;
    DeviceScratch iteration(context);  // the group table and the compact buffer
    void* table_block = nullptr;
    HYB_TRY(iteration.alloc(bytes, &table_block));
    HYB_CUDA(cudaMemsetAsync(table_block, 0, bytes, stream));
    GroupTable group_table{};
    group_table.capacity_mask = static_cast<uint32_t>(capacity - 1);
    group_table.key_words = key_words;
    auto* cursor = static_cast<unsigned long long*>(table_block);
    group_table.hashes = cursor;
    cursor += capacity;
    group_table.keys = cursor;
    cursor += capacity * key_words;
    group_table.rows = cursor;
    cursor += capacity;
    group_table.min_position = cursor;
    cursor += capacity;
    group_table.max_position = cursor;
    cursor += capacity;
    group_table.accumulators = cursor;
    cursor += capacity * aggregate_count;
    group_table.counts = cursor;
    cursor += capacity * aggregate_count;
    group_table.zero_first = cursor;
    cursor += capacity * aggregate_count;
    if (stddev_mask) {
      group_table.moments = reinterpret_cast<double*>(cursor);
      cursor += capacity * moment_words;
    }
    group_table.states = reinterpret_cast<uint32_t*>(cursor);
    group_table.null_masks = group_table.states + capacity;
    group_table.control = group_table.null_masks + capacity;
    // {groups inserted, overflow} of both tables: these words decide whether the tables were big enough
    uint32_t table_control[2] = {0, 0}, distinct_control[2] = {0, 0};
    // The COUNT(DISTINCT) set: hashes, {aggregate << 32 | group slot, value word} keys, states and its control words.
    // Only the first sweep reads it; it is freed once its control words are read.
    GroupTable distinct_table{};
    {
      DeviceScratch distinct_scratch(context);
      if (distinct_mask) {
        const size_t distinct_bytes = sizeof(uint64_t) * distinct_capacity * 3 + sizeof(uint32_t) * distinct_capacity + 64;
        void* distinct_block = nullptr;
        HYB_TRY(distinct_scratch.alloc(distinct_bytes, &distinct_block));
        HYB_CUDA(cudaMemsetAsync(distinct_block, 0, distinct_bytes, stream));
        distinct_table.capacity_mask = static_cast<uint32_t>(distinct_capacity - 1);
        distinct_table.key_words = 2;
        distinct_table.hashes = static_cast<unsigned long long*>(distinct_block);
        distinct_table.keys = distinct_table.hashes + distinct_capacity;
        distinct_table.states = reinterpret_cast<uint32_t*>(distinct_table.keys + distinct_capacity * 2);
        distinct_table.control = distinct_table.states + distinct_capacity;
      }
      HYB_CUDA(cudaMemsetAsync(group_table.min_position, 0xFF, sizeof(uint64_t) * capacity, stream));
      for (uint32_t a = 0; a < aggregate_count; ++a) {
        if (query->aggregates[a].function == HYB_AGG_MIN) {
          HYB_CUDA(cudaMemsetAsync(group_table.accumulators + size_t{a} * capacity, 0xFF, sizeof(uint64_t) * capacity, stream));
        }
        if (query->aggregates[a].function == HYB_AGG_MIN || query->aggregates[a].function == HYB_AGG_MAX) {
          HYB_CUDA(cudaMemsetAsync(group_table.zero_first + size_t{a} * capacity, 0xFF, sizeof(uint64_t) * capacity, stream));
        }
      }
      if (!out->kernel_timed) timing_kernel_begin(context);
      if (host_plan.tile_count) {
        if (distinct_mask || stddev_mask) {
          launch_general_sweep<kWithDistinct>(tree, grid, stream, device_plan, group_table, distinct_table);
        } else {
          launch_general_sweep<kPlain>(tree, grid, stream, device_plan, group_table, distinct_table);
        }
        HYB_CUDA(cudaGetLastError());
        ++out->launches;
      }
      if (!out->kernel_timed) timing_kernel_end(context);
      out->kernel_timed = true;
      HYB_CUDA(cudaMemcpyAsync(table_control, group_table.control, sizeof(table_control), cudaMemcpyDeviceToHost, stream));
      if (distinct_mask) {
        HYB_CUDA(cudaMemcpyAsync(distinct_control, distinct_table.control, sizeof(distinct_control), cudaMemcpyDeviceToHost,
                                 stream));
      }
      HYB_CUDA(cudaStreamSynchronize(stream));
    }
    if (table_control[1] || distinct_control[1]) {
      if (table_control[1]) capacity <<= 3;
      if (distinct_control[1]) distinct_capacity <<= 3;
      out->path = HYB_AGG_PATH_GENERAL_REGROWN;
      continue;
    }
    const uint32_t slot_grid =
        static_cast<uint32_t>(std::min<uint64_t>((capacity + 255) / 256, static_cast<uint64_t>(context->sm_count) * 16));
    if (stddev_mask && table_control[0]) {
      // corrected two-pass variance: the means, then the deviations of the same rows from them
      timing_kernel_begin(context);
      stddev_mean_kernel<<<slot_grid, 256, 0, stream>>>(group_table, aggregate_count, stddev_mask);
      HYB_CUDA(cudaGetLastError());
      launch_general_sweep<kDeviations>(tree, grid, stream, device_plan, group_table, distinct_table);
      HYB_CUDA(cudaGetLastError());
      timing_kernel_end(context);
      out->launches += 2;
    }
    if (has_string_extremes && table_control[0]) {
      string_extreme_kernel<<<slot_grid, 256, 0, stream>>>(group_table, aggregate_count, string_extremes);
      HYB_CUDA(cudaGetLastError());
      ++out->launches;
    }
    // pack the occupied slots on the device; only they travel to the host
    const uint64_t group_slots = table_control[0];
    const size_t compact_words = std::max<uint64_t>(group_slots, 1) * per_slot_words;
    const size_t compact_bytes = sizeof(uint64_t) * compact_words + sizeof(uint32_t) * std::max<uint64_t>(group_slots, 1) + 64;
    void* compact = nullptr;
    HYB_TRY(iteration.alloc(compact_bytes, &compact));
    auto* compact_null_masks = reinterpret_cast<uint32_t*>(static_cast<unsigned long long*>(compact) + compact_words);
    uint32_t* compact_cursor = compact_null_masks + std::max<uint64_t>(group_slots, 1);
    HYB_CUDA(cudaMemsetAsync(compact_cursor, 0, sizeof(uint32_t), stream));
    if (group_slots) {
      aggregate_compact_kernel<<<slot_grid, 256, 0, stream>>>(group_table, aggregate_count, static_cast<uint32_t>(group_slots),
                                                              static_cast<unsigned long long*>(compact), compact_null_masks,
                                                              compact_cursor);
      HYB_CUDA(cudaGetLastError());
      ++out->launches;
    }
    std::vector<uint8_t> host(compact_bytes);
    HYB_CUDA(cudaMemcpyAsync(host.data(), compact, compact_bytes, cudaMemcpyDeviceToHost, stream));
    HYB_CUDA(cudaStreamSynchronize(stream));
    parse_packed_groups(query, types, reinterpret_cast<const uint64_t*>(host.data()), group_slots, key_words, compact_words,
                        &out->groups);
    out->done = true;
  }
  return HYB_OK;
}

// Orders the groups like the reference and builds the result: representative RowIDs, value and NULL columns.
// `forced_immediate` >= 0: the partitioned exchange chose the order from all ranks' groups.
static int materialise_aggregate_result(hyb_context* context, const Table* table, const hyb_aggregate_query* query,
                                        const PosList* filter, bool exchanged, const AggregateTypes& types,
                                        int forced_immediate, std::vector<HostGroup>& groups, uint32_t* launches,
                                        std::unique_ptr<AggregateResult>* out_result) {
  cudaStream_t stream = context->stream;
  const uint32_t aggregate_count = query->aggregate_count;
  uint64_t input_rows = 0;
  for (const auto& group : groups) input_rows += group.rows;
  bool immediate = false;
  if (forced_immediate >= 0) {
    immediate = forced_immediate != 0;  // partitioned exchange: decided on the statistics of ALL ranks' groups
  } else if (query->groupby_count == 1 && table->column_types[query->groupby_column_ids[0]] == HYB_TYPE_INT32) {
    // immediate key shortcut (aggregate_hash.cpp:781-804)
    uint64_t min_key = ~uint64_t{0}, max_key = 0;
    for (const auto& group : groups) {
      if (group.null_mask) continue;
      min_key = std::min(min_key, group.key[0]);
      max_key = std::max(max_key, group.key[0]);
    }
    immediate = max_key > 0 && static_cast<double>(max_key - min_key) < static_cast<double>(input_rows) * 1.2;
  }
  if (immediate) {
    std::sort(groups.begin(), groups.end(), [](const HostGroup& a, const HostGroup& b) {
      if ((a.null_mask != 0) != (b.null_mask != 0)) return a.null_mask != 0;  // NULL group first
      return a.key[0] < b.key[0];
    });
  } else {
    std::sort(groups.begin(), groups.end(),
              [](const HostGroup& a, const HostGroup& b) { return a.min_position < b.min_position; });
  }

  auto result = std::make_unique<AggregateResult>();
  result->table = query->table;
  const bool synthesize_empty_row = query->groupby_count == 0 && aggregate_count > 0 && groups.empty();  // (:1395-1405)
  const size_t group_count = synthesize_empty_row ? 1 : groups.size();
  result->group_count = group_count;
  result->used_immediate_keys = immediate ? 1 : 0;
  result->row_ids.resize(group_count);
  if (synthesize_empty_row) {
    result->row_ids[0] = hyb_row_id{HYB_INVALID_CHUNK_ID, HYB_INVALID_CHUNK_OFFSET};
  } else if (!groups.empty()) {
    std::vector<uint64_t> positions(groups.size());
    for (size_t g = 0; g < groups.size(); ++g) {
      positions[g] = immediate ? groups[g].max_position : groups[g].min_position;
      // no group-by + COUNT(*) first: the reference stores RowID{0, 0} (aggregate_hash.cpp:1097-1102); any non-NULL
      // RowID is equivalent since no group-by column is written.
    }
    if (filter) {
      DeviceScratch scratch(context);
      unsigned long long* d_positions = nullptr;
      hyb_row_id* d_rows = nullptr;
      HYB_TRY(scratch.alloc_array(positions.size(), &d_positions));
      HYB_TRY(scratch.alloc_array(positions.size(), &d_rows));
      HYB_CUDA(cudaMemcpyAsync(d_positions, positions.data(), sizeof(uint64_t) * positions.size(), cudaMemcpyHostToDevice, stream));
      gather_row_ids_kernel<<<static_cast<uint32_t>((positions.size() + 255) / 256), 256, 0, stream>>>(
          d_positions, static_cast<uint32_t>(positions.size()), filter->d_row_ids, d_rows);
      HYB_CUDA(cudaGetLastError());
      HYB_CUDA(cudaMemcpyAsync(result->row_ids.data(), d_rows, sizeof(hyb_row_id) * positions.size(), cudaMemcpyDeviceToHost, stream));
      HYB_CUDA(cudaStreamSynchronize(stream));
      ++*launches;
    } else if (exchanged) {
      for (size_t g = 0; g < groups.size(); ++g) result->row_ids[g] = immediate ? groups[g].row_max : groups[g].row_min;
    } else {
      for (size_t g = 0; g < groups.size(); ++g) result->row_ids[g] = position_to_row_id_host(table, positions[g]);
    }
  }
  result->columns.resize(aggregate_count);
  for (uint32_t a = 0; a < aggregate_count; ++a) {
    const auto& def = query->aggregates[a];
    const int32_t result_type = types.result_types[a];
    auto& column = result->columns[a];
    column.value_type = result_type;
    const size_t element = (result_type == HYB_TYPE_INT32 || result_type == HYB_TYPE_FLOAT32) ? 4 : 8;
    column.values.assign(group_count * element, 0);
    column.nulls.assign(group_count, 0);
    const bool integral = types.input_types[a] == HYB_TYPE_INT32 || types.input_types[a] == HYB_TYPE_INT64;
    for (size_t g = 0; g < group_count; ++g) {
      const uint64_t count = synthesize_empty_row ? 0 : groups[g].counts[a];
      const uint64_t bits = synthesize_empty_row ? 0 : groups[g].accumulators[a];
      uint8_t* out = column.values.data() + g * element;
      if (def.function == HYB_AGG_COUNT || def.function == HYB_AGG_COUNT_STAR) {
        const int64_t value = static_cast<int64_t>(count);
        std::memcpy(out, &value, sizeof(value));
        continue;
      }
      if (def.function == HYB_AGG_COUNT_DISTINCT) {  // the accumulator counted the distinct values; never NULL
        std::memcpy(out, &bits, 8);
        continue;
      }
      if (count == 0 || (def.function == HYB_AGG_STDDEV_SAMP && count < 2)) {  // VAR_SAMP of one value is NULL
        column.nulls[g] = 1;
        continue;
      }
      switch (def.function) {
        case HYB_AGG_SUM:
        case HYB_AGG_STDDEV_SAMP:
          std::memcpy(out, &bits, 8);  // int64 sum or double sum / deviation, already in the result representation
          break;
        case HYB_AGG_AVG: {
          double sum;
          if (integral) {
            int64_t as_int;
            std::memcpy(&as_int, &bits, sizeof(as_int));
            sum = static_cast<double>(as_int);
          } else {
            std::memcpy(&sum, &bits, sizeof(sum));
          }
          const double average = sum / static_cast<double>(count);
          std::memcpy(out, &average, sizeof(average));
          break;
        }
        default: {  // MIN / MAX in the column type
          if (result_type == HYB_TYPE_STRING || result_type == HYB_TYPE_INT64) {
            std::memcpy(out, &bits, 8);  // strings: the hyb_dictionary_position string_extreme_kernel wrote
          } else if (result_type == HYB_TYPE_INT32) {
            const int32_t value = static_cast<int32_t>(static_cast<int64_t>(bits));
            std::memcpy(out, &value, sizeof(value));
          } else {
            double as_double;
            std::memcpy(&as_double, &bits, sizeof(as_double));
            if (result_type == HYB_TYPE_FLOAT32) {
              const float value = static_cast<float>(as_double);
              std::memcpy(out, &value, sizeof(value));
            } else {
              std::memcpy(out, &as_double, sizeof(as_double));
            }
          }
          break;
        }
      }
    }
  }
  *out_result = std::move(result);
  return HYB_OK;
}

// hyb_aggregate_hash with context->mutex held. `exchange` != nullptr: the groups of this rank are partial; they are
// exchanged with the peer group's ranks and merged before the result is ordered and materialised. `tree` != nullptr: a
// compiled expression tree (hyb_aggregate_hash_expression) every aggregated row must also satisfy.
static int aggregate_hash_locked(hyb_context* context, const hyb_aggregate_query* query, hyb_aggregate_result_t* out_result,
                                 const AggregateExchange* exchange, ExpressionTree* tree = nullptr) {
  auto* table = find_table(context, query->table);
  HYB_CHECK(table, HYB_ERR_NOT_FOUND, "unknown table handle");
  PosList* filter = nullptr;
  if (query->filter) {
    filter = find_pos_list(context, query->filter);
    HYB_CHECK(filter, HYB_ERR_NOT_FOUND, "unknown filter handle");
    HYB_CHECK(filter->table == query->table, HYB_ERR_INVALID, "filter belongs to a different table");
    HYB_CHECK(!filter->may_hold_null_rows, HYB_ERR_UNSUPPORTED,
              "aggregating a PosList with NULL_ROW_IDs (an outer join's output) runs on the CPU operator");
  }
  HYB_TRY(sync_table_descriptors(context, table));

  // ---- ANY: a group-by column the shim writes from the representative RowIDs (write_groupby_output, :421-537) -------
  // It adds no accumulator: the other aggregates run exactly as without it (an all-ANY query is the group-by-only call,
  // the reference's DISTINCT path), and its column of the result only names its type. It is checked before the others.
  const uint32_t aggregate_count = query->aggregate_count;
  std::vector<hyb_aggregate_def> kept;
  std::vector<int32_t> any_types(aggregate_count, -1);
  for (uint32_t a = 0; a < aggregate_count; ++a) {
    const auto& def = query->aggregates[a];
    if (def.function != HYB_AGG_ANY) {
      kept.push_back(def);
      continue;
    }
    HYB_CHECK(def.node_count == 1 && def.nodes[0].op == HYB_EXPR_COLUMN && def.nodes[0].column_id < table->column_count,
              HYB_ERR_INVALID, "ANY takes a single column of the input table");
    any_types[a] = table->column_types[def.nodes[0].column_id];
  }
  hyb_aggregate_query reduced = *query;
  reduced.aggregate_count = static_cast<uint32_t>(kept.size());
  reduced.aggregates = kept.data();
  query = &reduced;  // the rest of the call never sees ANY

  AggregateTypes types;
  HYB_TRY(type_aggregates(context, table, query, &types));
  timing_begin(context);
  AggregateOutcome outcome;
  uint64_t position_count = table->row_count();
  uint64_t algorithmic_bytes = 0;
  {
    DeviceScratch predicate_scratch(context);  // the fused tests and the tree: no kernel reads them after the general path
    FusedPredicates fused;
    HYB_TRY(prepare_fused_predicates(context, table, query, tree, predicate_scratch, &fused));
    outcome.launches = fused.launches;
    if (filter) HYB_TRY(pos_list_total(context, filter, &position_count));
    auto& slot = table->plan_memo[tree ? aggregate_signature(query) + "tree" + expression_tree_signature(*tree)
                                       : aggregate_signature(query)];
    if (!slot) slot = std::make_shared<AggregatePlanMemo>();
    const auto memo = std::static_pointer_cast<AggregatePlanMemo>(slot);
    algorithmic_bytes = aggregate_algorithmic_bytes(table, query, tree, types, filter, position_count, memo.get());
    HYB_TRY(run_fast_path(context, table, query, fused, memo.get(), &outcome));
    if (!outcome.done) HYB_TRY(run_general_path(context, table, query, filter, position_count, types, fused, &outcome));
  }

  int forced_immediate = -1;
  if (exchange) {
    HYB_CHECK(!filter, HYB_ERR_UNSUPPORTED, "distributed aggregation of position-filtered inputs is not on the GPU path");
    // Low cardinality: one 32 KB block per rank, replicated result. A rank whose partial groups do not fit sends its block's
    // header alone; every rank sees that in the same set of blocks and all of them switch to the partitioned exchange.
    bool needs_partitioning = false;
    HYB_TRY(exchange_partial_groups(context, *exchange, table, query, types.input_types, &outcome.groups, &needs_partitioning));
    if (needs_partitioning) {
      HYB_TRY(exchange_partial_groups_partitioned(context, *exchange, table, query, types.input_types, &outcome.groups,
                                                  &forced_immediate));
    }
  }

  std::unique_ptr<AggregateResult> result;
  HYB_TRY(materialise_aggregate_result(context, table, query, filter, exchange != nullptr, types, forced_immediate,
                                       outcome.groups, &outcome.launches, &result));
  if (!outcome.kernel_timed) {
    timing_kernel_begin(context);
    timing_kernel_end(context);
  }
  timing_end(context, outcome.launches, algorithmic_bytes, filter ? position_count : table->row_count(), result->group_count);
  context->timing.stats.path = outcome.path;

  if (kept.size() < aggregate_count) {  // the ANY columns back in their slots
    std::vector<AggregateColumn> columns(aggregate_count);
    for (uint32_t a = 0, next = 0; a < aggregate_count; ++a) {
      if (any_types[a] >= 0) {
        columns[a].value_type = any_types[a];
        columns[a].is_any = true;
      } else {
        columns[a] = std::move(result->columns[next++]);
      }
    }
    result->columns = std::move(columns);
  }
  const auto handle = context->next_handle++;
  context->aggregate_results.emplace(handle, std::move(result));
  *out_result = handle;
  return HYB_OK;
}

// ---- distributed aggregation: partial groups through the peer arenas ------------------------------------------------------
namespace {

__global__ void peer_raise_flags_kernel(unsigned long long* const* flags, uint32_t world, unsigned long long epoch) {
  __threadfence_system();
  if (threadIdx.x < world) st_volatile_u64(flags[threadIdx.x], epoch);
}

struct PartialGroupRecord {  // fixed-size wire format of one partial group
  uint64_t key[kMaxKeyWords];
  uint64_t rows, min_position, max_position;
  hyb_row_id row_min, row_max;
  uint32_t null_mask, pad;
  uint64_t accumulators[HYB_MAX_AGGREGATES];
  uint64_t counts[HYB_MAX_AGGREGATES];
};

void merge_accumulator(int32_t function, bool integral, uint64_t* target, uint64_t* target_count, uint64_t source,
                       uint64_t source_count) {
  const auto as_double = [](uint64_t bits) {
    double value;
    std::memcpy(&value, &bits, sizeof(value));
    return value;
  };
  const auto from_double = [](double value) {
    uint64_t bits;
    std::memcpy(&bits, &value, sizeof(bits));
    return bits;
  };
  switch (function) {
    case HYB_AGG_SUM:
    case HYB_AGG_AVG:  // travels as SUM + COUNT
      if (source_count) {
        if (integral) {
          *target = static_cast<uint64_t>(static_cast<int64_t>(*target) + static_cast<int64_t>(source));
        } else {
          *target = *target_count ? from_double(as_double(*target) + as_double(source)) : source;
        }
      }
      break;
    case HYB_AGG_MIN:
    case HYB_AGG_MAX:
      if (source_count) {
        bool take = *target_count == 0;
        if (!take) {
          if (integral) {
            take = function == HYB_AGG_MIN ? static_cast<int64_t>(source) < static_cast<int64_t>(*target)
                                           : static_cast<int64_t>(source) > static_cast<int64_t>(*target);
          } else {
            take = function == HYB_AGG_MIN ? as_double(source) < as_double(*target) : as_double(source) > as_double(*target);
          }
        }
        if (take) *target = source;
      }
      break;
    default:  // COUNT, COUNT(*): the counts are the values
      break;
  }
  *target_count += source_count;
}

}  // namespace

static int exchange_partial_groups(hyb_context* context, const AggregateExchange& exchange, const Table* table,
                                   const hyb_aggregate_query* query, const std::vector<int32_t>& input_types,
                                   std::vector<HostGroup>* groups, bool* out_needs_partitioning) {
  *out_needs_partitioning = false;
  PeerGroup* group = exchange.group;
  const uint32_t world = group->world, rank = group->rank;
  const uint32_t aggregate_count = query->aggregate_count;
  cudaStream_t stream = context->stream;
  const unsigned long long epoch = peer_next_epoch(group);
  HYB_CUDA(cudaEventRecord(group->events[5], stream));  // local pre-aggregation ended (events[0..4] at the caller)

  // ---- serialise this rank's partial groups (positions and representative rows made global) -----------------------------
  const size_t capacity = (kPeerAggregateBlockBytes - 16) / sizeof(PartialGroupRecord);
  const bool overflow = groups->size() > capacity;  // header only: tells every rank to switch to the partitioned exchange
  std::vector<unsigned char> block(kPeerAggregateBlockBytes, 0);
  const uint64_t header[2] = {groups->size(), aggregate_count};
  std::memcpy(block.data(), header, sizeof(header));
  auto* records = reinterpret_cast<PartialGroupRecord*>(block.data() + 16);
  for (size_t g = 0; g < (overflow ? 0 : groups->size()); ++g) {
    const HostGroup& source = (*groups)[g];
    PartialGroupRecord& record = records[g];
    for (size_t w = 0; w < kMaxKeyWords; ++w) record.key[w] = w < source.key.size() ? source.key[w] : 0;
    record.rows = source.rows;
    record.null_mask = source.null_mask;
    record.row_min = position_to_row_id_host(table, source.min_position);
    record.row_max = position_to_row_id_host(table, source.max_position);
    record.row_min.chunk_id += exchange.chunk_id_base;
    record.row_max.chunk_id += exchange.chunk_id_base;
    record.min_position = source.min_position + exchange.position_base;
    record.max_position = source.max_position + exchange.position_base;
    for (uint32_t a = 0; a < aggregate_count; ++a) {
      record.accumulators[a] = source.accumulators[a];
      record.counts[a] = source.counts[a];
    }
  }
  const size_t used_bytes = 16 + (overflow ? 0 : groups->size()) * sizeof(PartialGroupRecord);

  // ---- store the block into every rank's arena, raise the flags, wait for everybody's ------------------------------------
  DeviceScratch scratch(context);
  void* staged = nullptr;
  HYB_TRY(scratch.alloc(kPeerAggregateBlockBytes, &staged));
  HYB_CUDA(cudaMemcpyAsync(staged, block.data(), used_bytes, cudaMemcpyHostToDevice, stream));
  unsigned long long* host_flags[kPeerMax] = {};
  for (uint32_t peer = 0; peer < world; ++peer) {
    HYB_CUDA(cudaMemcpyAsync(group->control(peer)->aggregate_block[rank], staged, used_bytes, cudaMemcpyDefault, stream));
    host_flags[peer] = &group->control(peer)->aggregate_flag[rank];
  }
  unsigned long long** flags = nullptr;
  HYB_TRY(scratch.alloc_array(kPeerMax, &flags));
  HYB_CUDA(cudaMemcpyAsync(flags, host_flags, sizeof(host_flags), cudaMemcpyHostToDevice, stream));
  peer_raise_flags_kernel<<<1, 32, 0, stream>>>(flags, world, epoch);
  HYB_CUDA(cudaGetLastError());
  HYB_TRY(peer_wait(context, group->control(rank)->aggregate_flag, world, epoch));
  std::vector<unsigned char> all(size_t{world} * kPeerAggregateBlockBytes);
  HYB_CUDA(cudaMemcpyAsync(all.data(), group->control(rank)->aggregate_block, all.size(), cudaMemcpyDeviceToHost, stream));
  HYB_CUDA(cudaEventRecord(group->events[6], stream));
  HYB_CUDA(cudaStreamSynchronize(stream));
  group->stats.nvlink_bytes = used_bytes * (world - 1);

  for (uint32_t source_rank = 0; source_rank < world; ++source_rank) {
    uint64_t source_header[2];
    std::memcpy(source_header, all.data() + size_t{source_rank} * kPeerAggregateBlockBytes, sizeof(source_header));
    if (source_header[0] > capacity) *out_needs_partitioning = true;
  }
  if (*out_needs_partitioning) return HYB_OK;  // `groups` untouched: the caller exchanges them partitioned

  // ---- merge in rank order (every rank computes the same complete result) ---------------------------------------------------
  std::vector<HostGroup> merged;
  for (uint32_t source_rank = 0; source_rank < world; ++source_rank) {
    const unsigned char* base = all.data() + size_t{source_rank} * kPeerAggregateBlockBytes;
    uint64_t source_header[2];
    std::memcpy(source_header, base, sizeof(source_header));
    HYB_CHECK(source_header[0] <= capacity && source_header[1] == aggregate_count, HYB_ERR_INVALID,
              "rank " + std::to_string(source_rank) + " sent a partial-group block of another query");
    const auto* source_records = reinterpret_cast<const PartialGroupRecord*>(base + 16);
    for (uint64_t g = 0; g < source_header[0]; ++g) {
      const PartialGroupRecord& record = source_records[g];
      const size_t key_words = std::max<uint32_t>(query->groupby_count, 1);
      HostGroup* target = nullptr;
      for (auto& candidate : merged) {
        if (candidate.null_mask == record.null_mask && std::equal(candidate.key.begin(), candidate.key.end(), record.key)) {
          target = &candidate;
          break;
        }
      }
      if (!target) {
        merged.emplace_back();
        target = &merged.back();
        target->key.assign(record.key, record.key + key_words);
        target->null_mask = record.null_mask;
        target->accumulators.assign(aggregate_count, 0);
        target->counts.assign(aggregate_count, 0);
        target->has_global_rows = true;
        target->min_position = ~uint64_t{0};
        target->max_position = 0;
      }
      if (record.rows) {
        if (record.min_position < target->min_position || target->rows == 0) {
          target->min_position = record.min_position;
          target->row_min = record.row_min;
        }
        if (record.max_position >= target->max_position || target->rows == 0) {
          target->max_position = record.max_position;
          target->row_max = record.row_max;
        }
      }
      target->rows += record.rows;
      for (uint32_t a = 0; a < aggregate_count; ++a) {
        const int32_t function = query->aggregates[a].function;
        const bool integral = input_types[a] == HYB_TYPE_INT32 || input_types[a] == HYB_TYPE_INT64;
        merge_accumulator(function, integral, &target->accumulators[a], &target->counts[a], record.accumulators[a], record.counts[a]);
      }
    }
  }
  *groups = std::move(merged);
  return HYB_OK;
}

// ---- high-cardinality form: partial groups are partitioned by the hash of their key and every group is merged by ONE rank ----
namespace {

// Row `rank` of every rank's count matrix (side 0) and of its side_bounds: per-destination record counts and
// {min key, max key, rows, groups} of this rank's partial groups; then the count flag.
__global__ void peer_publish_group_counts_kernel(PeerControl* const* controls, uint32_t rank, uint32_t world, unsigned long long epoch,
                                                 const unsigned long long* counts, long long min_key, long long max_key,
                                                 long long rows, long long groups) {
  const uint32_t peer = threadIdx.x / 32, lane = threadIdx.x & 31;
  if (peer < world) {
    PeerControl* control = controls[peer];
    if (lane < world) control->counts[0][rank][lane] = counts[lane];
    if (lane == 0) {
      long long* row = control->side_bounds[rank];
      row[0] = min_key, row[1] = max_key, row[2] = rows, row[3] = groups;
    }
    __threadfence_system();
    __syncwarp();
    if (lane == 0) st_volatile_u64(&control->count_flag[rank], epoch);
  }
}

uint64_t host_mix64(uint64_t x) {
  x ^= x >> 33;
  x *= 0xFF51AFD7ED558CCDull;
  x ^= x >> 33;
  x *= 0xC4CEB9FE1A85EC53ull;
  x ^= x >> 33;
  return x;
}

int upload_controls(hyb_context* context, PeerGroup* group, DeviceScratch& scratch, PeerControl*** out_controls) {
  PeerControl** controls = nullptr;
  HYB_TRY(scratch.alloc_array(kPeerMax, &controls));
  PeerControl* host_controls[kPeerMax] = {};
  for (uint32_t peer = 0; peer < group->world; ++peer) host_controls[peer] = group->control(peer);
  HYB_CUDA(cudaMemcpyAsync(controls, host_controls, sizeof(host_controls), cudaMemcpyHostToDevice, context->stream));
  *out_controls = controls;
  return HYB_OK;
}

}  // namespace

static int exchange_partial_groups_partitioned(hyb_context* context, const AggregateExchange& exchange, const Table* table,
                                               const hyb_aggregate_query* query, const std::vector<int32_t>& input_types,
                                               std::vector<HostGroup>* groups, int* out_immediate) {
  PeerGroup* group = exchange.group;
  const uint32_t world = group->world, rank = group->rank;
  const uint32_t aggregate_count = query->aggregate_count;
  const size_t key_words = std::max<uint32_t>(query->groupby_count, 1);
  cudaStream_t stream = context->stream;
  const unsigned long long epoch = peer_next_epoch(group);
  HYB_CUDA(cudaEventRecord(group->events[5], stream));

  // ---- 1. serialise, destination-major (owner = hash of the key words; the same group lands on the same rank from everywhere).
  //         Wire format, in 64-bit words: key[key_words] | rows, min_position, max_position | row_min, row_max | null_mask |
  //         accumulators[aggregate_count] | counts[aggregate_count]
  const size_t record_words = key_words + 6 + 2 * size_t{aggregate_count};
  const size_t record_bytes = record_words * sizeof(uint64_t);
  std::vector<uint32_t> owner(groups->size());
  std::vector<unsigned long long> counts(kPeerMax, 0);
  long long min_key = std::numeric_limits<long long>::max(), max_key = 0, rows = 0;
  for (size_t g = 0; g < groups->size(); ++g) {
    const HostGroup& source = (*groups)[g];
    uint64_t hash = 0x9E3779B97F4A7C15ull ^ source.null_mask;
    for (size_t w = 0; w < key_words; ++w) hash = host_mix64(hash ^ (w < source.key.size() ? source.key[w] : 0));
    owner[g] = static_cast<uint32_t>(hash % world);
    ++counts[owner[g]];
    rows += static_cast<long long>(source.rows);
    if (!source.null_mask && !source.key.empty()) {
      min_key = std::min<long long>(min_key, static_cast<long long>(source.key[0]));
      max_key = std::max<long long>(max_key, static_cast<long long>(source.key[0]));
    }
  }
  std::vector<size_t> start(world + 1, 0);
  for (uint32_t d = 0; d < world; ++d) start[d + 1] = start[d] + counts[d];
  std::vector<uint64_t> records(std::max<size_t>(groups->size(), 1) * record_words);
  std::vector<size_t> cursor(start.begin(), start.end() - 1);
  const auto pack_row_id = [](hyb_row_id row) { return (static_cast<uint64_t>(row.chunk_id) << 32) | row.chunk_offset; };
  for (size_t g = 0; g < groups->size(); ++g) {
    const HostGroup& source = (*groups)[g];
    uint64_t* record = records.data() + (cursor[owner[g]]++) * record_words;
    for (size_t w = 0; w < key_words; ++w) record[w] = w < source.key.size() ? source.key[w] : 0;
    uint64_t* fields = record + key_words;
    hyb_row_id row_min = position_to_row_id_host(table, source.min_position);
    hyb_row_id row_max = position_to_row_id_host(table, source.max_position);
    row_min.chunk_id += exchange.chunk_id_base;
    row_max.chunk_id += exchange.chunk_id_base;
    fields[0] = source.rows;
    fields[1] = source.min_position + exchange.position_base;
    fields[2] = source.max_position + exchange.position_base;
    fields[3] = pack_row_id(row_min);
    fields[4] = pack_row_id(row_max);
    fields[5] = source.null_mask;
    for (uint32_t a = 0; a < aggregate_count; ++a) {
      fields[6 + a] = source.accumulators[a];
      fields[6 + aggregate_count + a] = source.counts[a];
    }
  }

  // ---- 2. publish the per-destination counts and the key statistics; read everybody's ----------------------------------------
  DeviceScratch scratch(context);
  PeerControl** controls = nullptr;
  HYB_TRY(upload_controls(context, group, scratch, &controls));
  unsigned long long* d_counts = nullptr;
  HYB_TRY(scratch.alloc_array(kPeerMax, &d_counts));
  HYB_CUDA(cudaMemcpyAsync(d_counts, counts.data(), sizeof(unsigned long long) * kPeerMax, cudaMemcpyHostToDevice, stream));
  peer_publish_group_counts_kernel<<<1, 32 * kPeerMax, 0, stream>>>(controls, rank, world, epoch, d_counts, min_key, max_key, rows,
                                                                    static_cast<long long>(groups->size()));
  HYB_CUDA(cudaGetLastError());
  HYB_TRY(peer_wait(context, group->control(rank)->count_flag, world, epoch));
  HYB_CUDA(cudaMemcpyAsync(group->h_counts, group->control(rank)->counts, sizeof(PeerControl::counts), cudaMemcpyDeviceToHost, stream));
  std::vector<long long> h_bounds(kPeerMax * 8);
  HYB_CUDA(cudaMemcpyAsync(h_bounds.data(), group->control(rank)->side_bounds, sizeof(PeerControl::side_bounds), cudaMemcpyDeviceToHost,
                           stream));
  HYB_CUDA(cudaStreamSynchronize(stream));
  const auto count_at = [&](uint32_t source, uint32_t destination) {
    return group->h_counts[(size_t{0} * kPeerMax + source) * kPeerMax + destination];
  };
  const size_t receive_capacity = 4 * group->region_bytes();
  uint64_t incoming = 0;
  for (uint32_t destination = 0; destination < world; ++destination) {
    uint64_t total = 0;
    for (uint32_t source = 0; source < world; ++source) total += count_at(source, destination);
    HYB_CHECK(total * record_bytes <= receive_capacity, HYB_ERR_OOM,
              "receive arena of rank " + std::to_string(destination) + " too small for " + std::to_string(total) +
                  " partial groups of " + std::to_string(record_bytes) + " bytes");
    if (destination == rank) incoming = total;
  }
  // the immediate-key decision of aggregate_hash.cpp:781-804 on the statistics of the WHOLE input
  {
    long long global_min = std::numeric_limits<long long>::max(), global_max = 0, global_rows = 0;
    for (uint32_t r = 0; r < world; ++r) {
      if (h_bounds[r * 8 + 3] == 0) continue;
      global_min = std::min(global_min, h_bounds[r * 8 + 0]);
      global_max = std::max(global_max, h_bounds[r * 8 + 1]);
      global_rows += h_bounds[r * 8 + 2];
    }
    const bool single_int = query->groupby_count == 1 && table->column_types[query->groupby_column_ids[0]] == HYB_TYPE_INT32;
    *out_immediate = single_int && global_max > 0 && global_max >= global_min &&
                             static_cast<double>(global_max - global_min) < static_cast<double>(global_rows) * 1.2
                         ? 1
                         : 0;
  }

  // ---- 3. stage the records on the device and store each destination's run into its arena (NVLink P2P copies) ----------------
  void* staged = nullptr;
  HYB_TRY(scratch.alloc(std::max<size_t>(records.size() * sizeof(uint64_t), 256), &staged));
  if (!groups->empty()) {
    HYB_CUDA(cudaMemcpyAsync(staged, records.data(), groups->size() * record_bytes, cudaMemcpyHostToDevice, stream));
  }
  uint64_t sent_elsewhere = 0;
  unsigned long long* host_flags[kPeerMax] = {};
  for (uint32_t destination = 0; destination < world; ++destination) {
    uint64_t before = 0;
    for (uint32_t source = 0; source < rank; ++source) before += count_at(source, destination);
    if (counts[destination]) {
      char* target = group->region(destination, 0) + before * record_bytes;
      HYB_CUDA(cudaMemcpyAsync(target, static_cast<const char*>(staged) + start[destination] * record_bytes,
                               counts[destination] * record_bytes, cudaMemcpyDefault, stream));
      if (destination != rank) sent_elsewhere += counts[destination];
    }
    host_flags[destination] = &group->control(destination)->done_flag[rank];
  }
  unsigned long long** flags = nullptr;
  HYB_TRY(scratch.alloc_array(kPeerMax, &flags));
  HYB_CUDA(cudaMemcpyAsync(flags, host_flags, sizeof(host_flags), cudaMemcpyHostToDevice, stream));
  peer_raise_flags_kernel<<<1, 32, 0, stream>>>(flags, world, epoch);
  HYB_CUDA(cudaGetLastError());
  HYB_TRY(peer_wait(context, group->control(rank)->done_flag, world, epoch));
  std::vector<uint64_t> received(std::max<uint64_t>(incoming, 1) * record_words);
  if (incoming) {
    HYB_CUDA(cudaMemcpyAsync(received.data(), group->region(rank, 0), incoming * record_bytes, cudaMemcpyDeviceToHost, stream));
  }
  HYB_CUDA(cudaEventRecord(group->events[6], stream));
  HYB_CUDA(cudaStreamSynchronize(stream));
  group->stats.nvlink_bytes = sent_elsewhere * record_bytes;
  group->stats.tuples_sent = sent_elsewhere;
  group->stats.tuples_received = incoming;
  group->stats.aggregate_partitioned = 1;

  // ---- 4. merge what this rank owns (records arrive grouped by source rank, in rank order) ----------------------------------
  const auto unpack_row_id = [](uint64_t packed) {
    return hyb_row_id{static_cast<uint32_t>(packed >> 32), static_cast<uint32_t>(packed)};
  };
  std::vector<HostGroup> merged;
  std::unordered_map<std::string, size_t> index;
  index.reserve(incoming * 2 + 16);
  std::string probe(key_words * sizeof(uint64_t) + sizeof(uint64_t), '\0');
  for (uint64_t g = 0; g < incoming; ++g) {
    const uint64_t* record = received.data() + g * record_words;
    const uint64_t* fields = record + key_words;
    std::memcpy(probe.data(), record, key_words * sizeof(uint64_t));
    std::memcpy(probe.data() + key_words * sizeof(uint64_t), &fields[5], sizeof(uint64_t));
    const auto [iter, inserted] = index.try_emplace(probe, merged.size());
    if (inserted) {
      merged.emplace_back();
      HostGroup& created = merged.back();
      created.key.assign(record, record + key_words);
      created.null_mask = static_cast<uint32_t>(fields[5]);
      created.accumulators.assign(aggregate_count, 0);
      created.counts.assign(aggregate_count, 0);
      created.has_global_rows = true;
      created.min_position = ~uint64_t{0};
      created.max_position = 0;
    }
    HostGroup& target = merged[iter->second];
    if (fields[0]) {
      if (fields[1] < target.min_position || target.rows == 0) {
        target.min_position = fields[1];
        target.row_min = unpack_row_id(fields[3]);
      }
      if (fields[2] >= target.max_position || target.rows == 0) {
        target.max_position = fields[2];
        target.row_max = unpack_row_id(fields[4]);
      }
    }
    target.rows += fields[0];
    for (uint32_t a = 0; a < aggregate_count; ++a) {
      const int32_t function = query->aggregates[a].function;
      const bool integral = input_types[a] == HYB_TYPE_INT32 || input_types[a] == HYB_TYPE_INT64;
      merge_accumulator(function, integral, &target.accumulators[a], &target.counts[a], fields[6 + a], fields[6 + aggregate_count + a]);
    }
  }
  *groups = std::move(merged);
  return HYB_OK;
}

// The argument checks every aggregate entry point makes before it takes the context's lock.
static int check_aggregate_query(const hyb_aggregate_query* query) {
  HYB_CHECK(query->groupby_count <= HYB_MAX_GROUPBY_COLUMNS, HYB_ERR_UNSUPPORTED, "too many group-by columns");
  HYB_CHECK(query->aggregate_count <= HYB_MAX_AGGREGATES, HYB_ERR_UNSUPPORTED, "too many aggregates");
  HYB_CHECK(query->predicate_count <= HYB_MAX_FUSED_PREDICATES, HYB_ERR_UNSUPPORTED, "too many fused predicates");
  HYB_CHECK(query->groupby_count == 0 || query->groupby_column_ids, HYB_ERR_INVALID, "groupby_column_ids is NULL");
  HYB_CHECK(query->aggregate_count == 0 || query->aggregates, HYB_ERR_INVALID, "aggregates is NULL");
  HYB_CHECK(query->predicate_count == 0 || query->predicates, HYB_ERR_INVALID, "predicates is NULL");
  return HYB_OK;
}

extern "C" {

int hyb_aggregate_hash_expression(hyb_context* context, const hyb_aggregate_query* query,
                                  const hyb_expression_scan_predicate* predicate, const hyb_expression_leaf_tests* tests,
                                  hyb_aggregate_result_t* out_result) {
  HYB_CHECK(context && query && predicate && out_result, HYB_ERR_INVALID, "NULL argument");
  *out_result = 0;
  HYB_TRY(check_aggregate_query(query));
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  const Table* table = find_table(context, query->table);
  HYB_CHECK(table, HYB_ERR_NOT_FOUND, "unknown table handle");
  auto tree = std::make_unique<ExpressionTree>();
  HYB_TRY(compile_expression_tree(table, predicate, tests, tree.get()));
  return aggregate_hash_locked(context, query, out_result, nullptr, tree.get());
}

int hyb_aggregate_hash(hyb_context* context, const hyb_aggregate_query* query, hyb_aggregate_result_t* out_result) {
  HYB_CHECK(context && query && out_result, HYB_ERR_INVALID, "NULL argument");
  *out_result = 0;
  HYB_TRY(check_aggregate_query(query));
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  return aggregate_hash_locked(context, query, out_result, nullptr);
}

int hyb_aggregate_hash_distributed(hyb_context* context, hyb_peer_group_t group_handle, const hyb_aggregate_query* query,
                                   uint32_t chunk_id_base, uint64_t position_base, hyb_aggregate_result_t* out_result) {
  HYB_CHECK(context && query && out_result, HYB_ERR_INVALID, "NULL argument");
  *out_result = 0;
  HYB_TRY(check_aggregate_query(query));
  for (uint32_t a = 0; a < query->aggregate_count; ++a) {
    // Partial distinct sets and Welford states do not fit the exchanged partial groups. Every rank sees the same query,
    // so all ranks decline here, before any exchange.
    const int32_t function = query->aggregates[a].function;
    HYB_CHECK(function != HYB_AGG_COUNT_DISTINCT && function != HYB_AGG_STDDEV_SAMP, HYB_ERR_UNSUPPORTED,
              "distributed COUNT(DISTINCT) / STDDEV_SAMP runs on the CPU operator");
  }
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  PeerGroup* group = find_peer_group(context, group_handle);
  HYB_CHECK(group, HYB_ERR_NOT_FOUND, "unknown peer group handle");
  HYB_CHECK(group->connected || group->world == 1, HYB_ERR_INVALID, "peer group is not connected");
  if (const Table* table = find_table(context, query->table)) {
    for (uint32_t a = 0; a < query->aggregate_count; ++a) {
      // Every shard would rank its strings on its own, and ANY names rows of the shard: like COUNT(DISTINCT), all ranks
      // decline before any exchange.
      const auto& def = query->aggregates[a];
      if (def.function == HYB_AGG_COUNT_STAR) continue;  // no argument; its nodes are never read
      HYB_CHECK(def.node_count <= HYB_MAX_EXPR_NODES, HYB_ERR_INVALID, "bad expression length");
      HYB_CHECK(def.function != HYB_AGG_ANY && !has_string_argument(table, def), HYB_ERR_UNSUPPORTED,
                "distributed ANY and aggregates over string columns run on the CPU operator");
    }
  }
  group->stats = hyb_distributed_stats{};
  for (int event = 0; event < 5; ++event) HYB_CUDA(cudaEventRecord(group->events[event], context->stream));
  const AggregateExchange exchange{group, chunk_id_base, position_base};
  return aggregate_hash_locked(context, query, out_result, &exchange);
}

static AggregateResult* find_aggregate_result(hyb_context* context, hyb_aggregate_result_t handle) {
  auto it = context->aggregate_results.find(handle);
  return it == context->aggregate_results.end() ? nullptr : it->second.get();
}

int hyb_aggregate_result_info(hyb_context* context, hyb_aggregate_result_t handle, uint64_t* out_group_count,
                              int32_t* out_used_immediate_keys) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* result = find_aggregate_result(context, handle);
  HYB_CHECK(result, HYB_ERR_NOT_FOUND, "unknown aggregate result handle");
  if (out_group_count) *out_group_count = result->group_count;
  if (out_used_immediate_keys) *out_used_immediate_keys = result->used_immediate_keys;
  return HYB_OK;
}

int hyb_aggregate_result_row_ids(hyb_context* context, hyb_aggregate_result_t handle, hyb_row_id* out_row_ids) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* result = find_aggregate_result(context, handle);
  HYB_CHECK(result, HYB_ERR_NOT_FOUND, "unknown aggregate result handle");
  HYB_CHECK(out_row_ids || result->row_ids.empty(), HYB_ERR_INVALID, "out_row_ids is NULL");
  std::copy(result->row_ids.begin(), result->row_ids.end(), out_row_ids);
  return HYB_OK;
}

int hyb_aggregate_result_values(hyb_context* context, hyb_aggregate_result_t handle, uint32_t aggregate_index,
                                void* out_values, uint8_t* out_nulls, int32_t* out_value_type) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* result = find_aggregate_result(context, handle);
  HYB_CHECK(result, HYB_ERR_NOT_FOUND, "unknown aggregate result handle");
  HYB_CHECK(aggregate_index < result->columns.size(), HYB_ERR_INVALID, "aggregate_index out of range");
  const auto& column = result->columns[aggregate_index];
  HYB_CHECK(!column.is_any, HYB_ERR_INVALID,
            "aggregate " + std::to_string(aggregate_index) +
                " is ANY: its values are the column at the representative RowIDs (hyb_aggregate_result_row_ids)");
  if (out_values && !column.values.empty()) std::memcpy(out_values, column.values.data(), column.values.size());
  if (out_nulls && !column.nulls.empty()) std::memcpy(out_nulls, column.nulls.data(), column.nulls.size());
  if (out_value_type) *out_value_type = column.value_type;
  return HYB_OK;
}

}  // extern "C"

// ---- Sort + Limit over one aggregate column: top-k selection on the device -------------------------------------------------
namespace {

// Sort key of a candidate: the value mapped to an order-preserving uint64 (largest first after the mapping), ties broken by
// the smaller group index (Sort is stable). 0 = "taken / not a candidate".
struct TopKCandidate {
  unsigned long long key;
  uint32_t index;
};

__device__ __forceinline__ bool top_k_before(const TopKCandidate& a, const TopKCandidate& b) {
  return a.key > b.key || (a.key == b.key && a.index < b.index);
}

// Every CTA selects the k best of its slice by k rounds of a block-wide arg-max (k is small: LIMIT 10 / 20 / 100);
// candidates[cta * k + i] = i-th best of the slice. A second launch with one CTA merges the per-CTA candidates.
__global__ void __launch_bounds__(256) top_k_kernel(const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ indexes,
                                                    uint32_t count, uint32_t k, TopKCandidate* __restrict__ candidates) {
  __shared__ TopKCandidate s_best[8];
  __shared__ TopKCandidate s_round;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t per_cta = (count + gridDim.x - 1) / gridDim.x;
  const uint32_t begin = blockIdx.x * per_cta, end = min(count, begin + per_cta);
  TopKCandidate previous{~0ull, 0u};  // everything at or before `previous` in the order has been emitted
  bool first_round = true;
  for (uint32_t round = 0; round < k; ++round) {
    TopKCandidate best{0ull, 0xFFFFFFFFu};
    for (uint32_t i = begin + threadIdx.x; i < end; i += blockDim.x) {
      const TopKCandidate candidate{keys[i], indexes ? indexes[i] : i};
      if (candidate.key == 0) continue;
      const bool emitted = !first_round && !top_k_before(previous, candidate);  // candidate <= previous in the order
      if (!emitted && (best.index == 0xFFFFFFFFu || top_k_before(candidate, best))) best = candidate;
    }
#pragma unroll
    for (int delta = 16; delta > 0; delta >>= 1) {
      TopKCandidate other;
      other.key = __shfl_xor_sync(0xFFFFFFFFu, best.key, delta);
      other.index = __shfl_xor_sync(0xFFFFFFFFu, best.index, delta);
      if (other.index != 0xFFFFFFFFu && (best.index == 0xFFFFFFFFu || top_k_before(other, best))) best = other;
    }
    if (lane == 0) s_best[warp] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
      TopKCandidate winner = s_best[0];
      for (int w = 1; w < 8; ++w) {
        if (s_best[w].index != 0xFFFFFFFFu && (winner.index == 0xFFFFFFFFu || top_k_before(s_best[w], winner))) winner = s_best[w];
      }
      s_round = winner;
      candidates[static_cast<size_t>(blockIdx.x) * k + round] = winner.index == 0xFFFFFFFFu ? TopKCandidate{0ull, 0xFFFFFFFFu} : winner;
    }
    __syncthreads();
    if (s_round.index == 0xFFFFFFFFu) {
      for (uint32_t rest = round + 1 + threadIdx.x; rest < k; rest += blockDim.x) {
        candidates[static_cast<size_t>(blockIdx.x) * k + rest] = TopKCandidate{0ull, 0xFFFFFFFFu};
      }
      return;
    }
    previous = s_round;
    first_round = false;
    __syncthreads();
  }
}

unsigned long long top_k_order_key(const hyb::AggregateColumn& column, uint64_t group, bool descending) {
  // order-preserving uint64 of the value; NULLs get the smallest non-zero key (they sort last either way)
  if (column.nulls[group]) return 1ull;
  unsigned long long ordered = 0;
  switch (column.value_type) {
    case HYB_TYPE_INT32: {
      int32_t v;
      std::memcpy(&v, column.values.data() + group * 4, 4);
      ordered = static_cast<unsigned long long>(static_cast<long long>(v)) ^ 0x8000000000000000ull;
      break;
    }
    case HYB_TYPE_INT64: {
      long long v;
      std::memcpy(&v, column.values.data() + group * 8, 8);
      ordered = static_cast<unsigned long long>(v) ^ 0x8000000000000000ull;
      break;
    }
    default: {
      double v;
      if (column.value_type == HYB_TYPE_FLOAT32) {
        float f;
        std::memcpy(&f, column.values.data() + group * 4, 4);
        v = f;
      } else {
        std::memcpy(&v, column.values.data() + group * 8, 8);
      }
      unsigned long long bits;
      std::memcpy(&bits, &v, 8);
      ordered = (bits >> 63) ? ~bits : (bits | 0x8000000000000000ull);
      break;
    }
  }
  if (!descending) ordered = ~ordered;
  return std::max<unsigned long long>(ordered, 2ull);  // keep clear of the reserved 0 / 1
}

}  // namespace

extern "C" {

int hyb_aggregate_result_top_k(hyb_context* context, hyb_aggregate_result_t handle, uint32_t aggregate_index, uint32_t k,
                               int32_t descending, uint32_t* out_group_indexes, uint32_t* out_count) {
  HYB_CHECK(context && out_group_indexes && out_count, HYB_ERR_INVALID, "NULL argument");
  HYB_CHECK(k >= 1 && k <= 1024, HYB_ERR_UNSUPPORTED, "LIMIT beyond 1024 rows is not a top-k selection: sort on the CPU operator");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* result = find_aggregate_result(context, handle);
  HYB_CHECK(result, HYB_ERR_NOT_FOUND, "unknown aggregate result handle");
  HYB_CHECK(aggregate_index < result->columns.size(), HYB_ERR_INVALID, "aggregate_index out of range");
  HYB_CHECK(!result->columns[aggregate_index].is_any, HYB_ERR_INVALID, "ANY has no values to sort by");
  HYB_CHECK(result->columns[aggregate_index].value_type != HYB_TYPE_STRING, HYB_ERR_UNSUPPORTED,
            "sorting by a string aggregate runs on the CPU operator");
  const uint64_t groups = result->group_count;
  HYB_CHECK(groups < 0xFFFFFFF0ull, HYB_ERR_UNSUPPORTED, "too many groups");
  *out_count = static_cast<uint32_t>(std::min<uint64_t>(k, groups));
  if (groups == 0) return HYB_OK;
  // the result columns live on the host (AggregateResult): stage the order keys, select on the device
  const auto& column = result->columns[aggregate_index];
  std::vector<unsigned long long> keys(groups);
  for (uint64_t g = 0; g < groups; ++g) keys[g] = top_k_order_key(column, g, descending != 0);
  cudaStream_t stream = context->stream;
  DeviceScratch scratch(context);
  unsigned long long* d_keys = nullptr;
  HYB_TRY(scratch.alloc_array(groups, &d_keys));
  HYB_CUDA(cudaMemcpyAsync(d_keys, keys.data(), sizeof(unsigned long long) * groups, cudaMemcpyHostToDevice, stream));
  const uint32_t grid = static_cast<uint32_t>(std::min<uint64_t>((groups + 4095) / 4096, uint64_t{context->sm_count} * 2));
  TopKCandidate* candidates = nullptr;
  HYB_TRY(scratch.alloc_array(size_t{grid} * k + k, &candidates));
  top_k_kernel<<<grid, 256, 0, stream>>>(d_keys, nullptr, static_cast<uint32_t>(groups), k, candidates);
  HYB_CUDA(cudaGetLastError());
  TopKCandidate* winners = candidates;
  if (grid > 1) {
    // merge: the per-CTA candidates as (key, index) arrays for one more selection by a single CTA
    unsigned long long* merge_keys = nullptr;
    uint32_t* merge_indexes = nullptr;
    HYB_TRY(scratch.alloc_array(size_t{grid} * k, &merge_keys));
    HYB_TRY(scratch.alloc_array(size_t{grid} * k, &merge_indexes));
    std::vector<TopKCandidate> host(size_t{grid} * k);
    HYB_CUDA(cudaMemcpyAsync(host.data(), candidates, sizeof(TopKCandidate) * host.size(), cudaMemcpyDeviceToHost, stream));
    HYB_CUDA(cudaStreamSynchronize(stream));
    std::vector<unsigned long long> host_keys(host.size());
    std::vector<uint32_t> host_indexes(host.size());
    for (size_t i = 0; i < host.size(); ++i) {
      host_keys[i] = host[i].index == 0xFFFFFFFFu ? 0ull : host[i].key;
      host_indexes[i] = host[i].index;
    }
    HYB_CUDA(cudaMemcpyAsync(merge_keys, host_keys.data(), sizeof(unsigned long long) * host_keys.size(), cudaMemcpyHostToDevice, stream));
    HYB_CUDA(cudaMemcpyAsync(merge_indexes, host_indexes.data(), sizeof(uint32_t) * host_indexes.size(), cudaMemcpyHostToDevice, stream));
    winners = candidates + size_t{grid} * k;
    top_k_kernel<<<1, 256, 0, stream>>>(merge_keys, merge_indexes, static_cast<uint32_t>(host.size()), k, winners);
    HYB_CUDA(cudaGetLastError());
    std::vector<TopKCandidate> final_candidates(k);
    HYB_CUDA(cudaMemcpyAsync(final_candidates.data(), winners, sizeof(TopKCandidate) * k, cudaMemcpyDeviceToHost, stream));
    HYB_CUDA(cudaStreamSynchronize(stream));
    for (uint32_t i = 0; i < *out_count; ++i) out_group_indexes[i] = final_candidates[i].index;
    return HYB_OK;
  }
  std::vector<TopKCandidate> final_candidates(k);
  HYB_CUDA(cudaMemcpyAsync(final_candidates.data(), winners, sizeof(TopKCandidate) * k, cudaMemcpyDeviceToHost, stream));
  HYB_CUDA(cudaStreamSynchronize(stream));
  for (uint32_t i = 0; i < *out_count; ++i) out_group_indexes[i] = final_candidates[i].index;
  return HYB_OK;
}

int hyb_aggregate_result_free(hyb_context* context, hyb_aggregate_result_t handle) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  std::lock_guard<std::mutex> lock(context->mutex);
  auto it = context->aggregate_results.find(handle);
  HYB_CHECK(it != context->aggregate_results.end(), HYB_ERR_NOT_FOUND, "unknown aggregate result handle");
  context->aggregate_results.erase(it);
  return HYB_OK;
}

}  // extern "C"
