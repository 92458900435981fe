// JoinHash with secondary predicates on the CPU (test infrastructure only, tests/join_predicates_oracle.py).
//
// orc_join_hash_predicates restates JoinHashImpl::_on_execute with `_secondary_predicates` (join_hash.cpp:270-572): the
// CPU oracle's materialize_input / partition_by_radix / build (oracle/oracle.cpp, included below, unchanged), a build of
// every position per key whenever there are secondary predicates (join_hash.cpp:445-457), and probe / probe_semi_anti
// with a MultiPredicateJoinEvaluator (join_hash_steps.hpp:624-792, :794-922), restated line by line. The evaluator
// compares with the real std::equal_to<void>, std::less<void>, ... on the two columns' own C++ types, so C++ applies its
// usual arithmetic conversions itself (int x float in float, anything with a double in double). No -ffast-math.
#include "../../oracle/oracle.cpp"

#include <memory>

namespace {

// AbstractSegmentAccessor<T>::access (storage/segment_accessor.hpp): std::nullopt for NULL.
template <typename T>
std::optional<T> access(const hyb_table_view* table, uint32_t column, const hyb_row_id& row_id) {
  // The reference never evaluates a NULL_ROW_ID: Inner / Semi skip them and Left / Right / AntiNullAsFalse emit them as
  // NULL keys before the evaluator runs (join_hash_steps.hpp:693-697, :719-727, :847-859). Read it as NULL.
  if (row_id_is_null(row_id)) return std::nullopt;
  const auto& segment = segment_at(table, row_id.chunk_id, column);
  if (segment_is_null(segment, row_id.chunk_offset)) return std::nullopt;
  return segment_value<T>(segment, row_id.chunk_offset);
}

// MultiPredicateJoinEvaluator::BaseFieldComparator / FieldComparator (multi_predicate_join_evaluator.hpp:25-61).
class BaseFieldComparator {
 public:
  virtual ~BaseFieldComparator() = default;
  virtual bool compare(const hyb_row_id& left, const hyb_row_id& right) const = 0;
};

template <typename CompareFunctor, typename L, typename R>
class FieldComparator : public BaseFieldComparator {
 public:
  FieldComparator(CompareFunctor compare_functor, int32_t join_mode, const hyb_table_view* left_table, uint32_t left_column,
                  const hyb_table_view* right_table, uint32_t right_column)
      : _compare_functor(compare_functor), _join_mode(join_mode), _left_table(left_table), _left_column(left_column),
        _right_table(right_table), _right_column(right_column) {}

  bool compare(const hyb_row_id& left, const hyb_row_id& right) const override {  // :44-54
    const auto left_value = access<L>(_left_table, _left_column, left);
    const auto right_value = access<R>(_right_table, _right_column, right);
    if (!left_value || !right_value) return _join_mode == HYB_JOIN_ANTI_NULL_AS_TRUE;
    return _compare_functor(*left_value, *right_value);
  }

 private:
  const CompareFunctor _compare_functor;
  const int32_t _join_mode;
  const hyb_table_view* _left_table;
  const uint32_t _left_column;
  const hyb_table_view* _right_table;
  const uint32_t _right_column;
};

// with_comparator (type_comparison.hpp): the std functor of a condition.
template <typename Functor>
void with_comparator(int32_t condition, const Functor& functor) {
  switch (condition) {
    case HYB_PRED_EQUALS:
      return functor(std::equal_to<void>{});
    case HYB_PRED_NOT_EQUALS:
      return functor(std::not_equal_to<void>{});
    case HYB_PRED_LESS_THAN:
      return functor(std::less<void>{});
    case HYB_PRED_LESS_THAN_EQUALS:
      return functor(std::less_equal<void>{});
    case HYB_PRED_GREATER_THAN:
      return functor(std::greater<void>{});
    default:
      return functor(std::greater_equal<void>{});
  }
}

int32_t column_type(const hyb_table_view* table, uint32_t column) {
  return table->chunk_count ? segment_at(table, 0, column).data_type : HYB_TYPE_INT32;
}

// MultiPredicateJoinEvaluator (multi_predicate_join_evaluator.cpp:18-60). `left` is the build table and a predicate's
// first column a build column, as JoinHashImpl constructs it after flipping (join_hash.cpp:158-165).
class MultiPredicateJoinEvaluator {
 public:
  MultiPredicateJoinEvaluator(const hyb_table_view* left, const hyb_table_view* right, int32_t join_mode,
                              const hyb_join_predicate* predicates, uint32_t predicate_count) {
    for (uint32_t index = 0; index < predicate_count; ++index) {
      const auto& predicate = predicates[index];
      with_type(column_type(left, predicate.build_column_id), [&](auto left_type) {
        with_type(column_type(right, predicate.probe_column_id), [&](auto right_type) {
          using L = decltype(left_type);
          using R = decltype(right_type);
          with_comparator(predicate.condition, [&](auto comparator) {
            _comparators.emplace_back(std::make_unique<FieldComparator<decltype(comparator), L, R>>(
                comparator, join_mode, left, predicate.build_column_id, right, predicate.probe_column_id));
          });
        });
      });
    }
  }

  bool satisfies_all_predicates(const hyb_row_id& left_row_id, const hyb_row_id& right_row_id) const {  // :52-60
    for (const auto& comparator : _comparators) {
      if (!comparator->compare(left_row_id, right_row_id)) return false;
    }
    return true;
  }

 private:
  std::vector<std::unique_ptr<BaseFieldComparator>> _comparators;
};

// probe (join_hash_steps.hpp:624-792) with a MultiPredicateJoinEvaluator
template <typename T, typename HashedType, bool keep_null_values>
void probe_with_predicates(const RadixContainer<T>& probe_container,
                           const std::vector<std::unique_ptr<PosHashTable<HashedType>>>& hash_tables, JoinOutput& out,
                           int32_t mode, const MultiPredicateJoinEvaluator& multi_predicate_join_evaluator) {
  const auto slices = make_slices(probe_container, out, true);
  for (const auto& slice : slices) {
    const auto& partition = probe_container[slice.partition];
    const auto& elements = partition.elements;
    RowIDs build_local, probe_local;
    const size_t table_idx = hash_tables.size() > 1 ? slice.partition : 0;
    if (!hash_tables.empty() && hash_tables.at(table_idx)) {
      const auto& hash_table = *hash_tables[table_idx];
      for (size_t offset = slice.begin; offset < slice.end; ++offset) {
        const auto& element = elements[offset];
        if (mode == HYB_JOIN_INNER && row_id_is_null(element.row_id)) continue;  // :693-698
        const auto range = hash_table.find(static_cast<HashedType>(element.value));
        if (range.first != range.second) {
          if constexpr (keep_null_values) {  // :711-719
            if (partition.null_values[offset]) {
              build_local.push_back(NULL_ROW_ID);
              probe_local.push_back(element.row_id);
              continue;
            }
          }
          bool match_found = false;  // :730-748
          for (const hyb_row_id* it = range.first; it != range.second; ++it) {
            if (multi_predicate_join_evaluator.satisfies_all_predicates(*it, element.row_id)) {
              build_local.push_back(*it);
              probe_local.push_back(element.row_id);
              match_found = true;
            }
          }
          if constexpr (keep_null_values) {
            if (!match_found) {
              build_local.push_back(NULL_ROW_ID);
              probe_local.push_back(element.row_id);
            }
          }
        } else {
          if constexpr (keep_null_values) {
            build_local.push_back(NULL_ROW_ID);
            probe_local.push_back(element.row_id);
          }
        }
      }
    } else {
      if constexpr (keep_null_values) {
        for (size_t offset = slice.begin; offset < slice.end; ++offset) {
          build_local.push_back(NULL_ROW_ID);
          probe_local.push_back(elements[offset].row_id);
        }
      }
    }
    out.build_side[slice.output_idx] = std::move(build_local);
    out.probe_side[slice.output_idx] = std::move(probe_local);
  }
}

// probe_semi_anti (join_hash_steps.hpp:794-922) with a MultiPredicateJoinEvaluator: Semi and AntiNullAsFalse
template <typename T, typename HashedType>
void probe_semi_anti_with_predicates(const RadixContainer<T>& probe_container,
                                     const std::vector<std::unique_ptr<PosHashTable<HashedType>>>& hash_tables,
                                     JoinOutput& out, int32_t mode,
                                     const MultiPredicateJoinEvaluator& multi_predicate_join_evaluator) {
  const auto slices = make_slices(probe_container, out, false);
  for (const auto& slice : slices) {
    const auto& partition = probe_container[slice.partition];
    const auto& elements = partition.elements;
    const auto& null_values = partition.null_values;
    RowIDs local;
    const size_t table_idx = hash_tables.size() > 1 ? slice.partition : 0;
    if (!hash_tables.empty() && hash_tables.at(table_idx)) {
      const auto& hash_table = *hash_tables[table_idx];
      for (size_t offset = slice.begin; offset < slice.end; ++offset) {
        const auto& element = elements[offset];
        if (mode == HYB_JOIN_SEMI) {  // :847-852
          if (row_id_is_null(element.row_id)) continue;
        } else if (null_values[offset]) {  // AntiNullAsFalse, :853-859
          local.push_back(element.row_id);
          continue;
        }
        const auto range = hash_table.find(static_cast<HashedType>(element.value));  // :872-876
        const bool any_build_column_value_matches = std::any_of(range.first, range.second, [&](const hyb_row_id& row_id) {
          return multi_predicate_join_evaluator.satisfies_all_predicates(row_id, element.row_id);
        });
        if ((mode == HYB_JOIN_SEMI && any_build_column_value_matches) ||
            (mode == HYB_JOIN_ANTI_NULL_AS_FALSE && !any_build_column_value_matches)) {  // :879-883
          local.push_back(element.row_id);
        }
      }
    } else if (mode == HYB_JOIN_ANTI_NULL_AS_FALSE) {  // :884-891
      for (size_t offset = slice.begin; offset < slice.end; ++offset) local.push_back(elements[offset].row_id);
    }
    out.probe_side[slice.output_idx] = std::move(local);
  }
}

// JoinHashImpl::_on_execute (join_hash.cpp:270-572) with secondary predicates, single-threaded: materialisation, radix
// partitioning, build with every position (:445-457), probe, then the flattening of oracle.cpp's join_hash_impl.
template <typename BuildT, typename ProbeT>
int join_hash_predicates_impl(const hyb_table_view* build_table, uint32_t build_column, const orc_pos_list* build_filter,
                              const hyb_table_view* probe_table, uint32_t probe_column, const orc_pos_list* probe_filter,
                              int32_t mode, size_t radix_bits, const hyb_join_predicate* predicates,
                              uint32_t predicate_count, orc_join_result* result) {
  using HashedType = std::conditional_t<(sizeof(BuildT) < sizeof(ProbeT)), ProbeT, BuildT>;  // join_hash_traits.hpp:25-31
  const bool keep_nulls_probe = mode != HYB_JOIN_INNER && mode != HYB_JOIN_SEMI;
  std::vector<std::vector<size_t>> histograms_build, histograms_probe;
  RadixContainer<BuildT> materialized_build;
  RadixContainer<ProbeT> materialized_probe;
  BloomFilter build_bloom, probe_bloom;
  const auto materialize_build = [&](const BloomFilter* input) {
    materialized_build = materialize_input<BuildT, HashedType, false>(build_table, build_column, build_filter,
                                                                       histograms_build, radix_bits, build_bloom, input, 1);
  };
  const auto materialize_probe = [&](const BloomFilter* input) {
    materialized_probe =
        keep_nulls_probe ? materialize_input<ProbeT, HashedType, true>(probe_table, probe_column, probe_filter,
                                                                       histograms_probe, radix_bits, probe_bloom, input, 1)
                         : materialize_input<ProbeT, HashedType, false>(probe_table, probe_column, probe_filter,
                                                                        histograms_probe, radix_bits, probe_bloom, input, 1);
  };
  if (table_row_count(build_table, build_filter) < table_row_count(probe_table, probe_filter)) {  // :364-381
    materialize_build(nullptr);
    materialize_probe(&build_bloom);
  } else {
    materialize_probe(nullptr);
    materialize_build(&probe_bloom);
  }
  RadixContainer<BuildT> radix_build;
  RadixContainer<ProbeT> radix_probe;
  if (radix_bits > 0) {
    radix_build = partition_by_radix<BuildT, HashedType, false>(materialized_build, histograms_build, radix_bits, 1);
    radix_probe = keep_nulls_probe
                      ? partition_by_radix<ProbeT, HashedType, true>(materialized_probe, histograms_probe, radix_bits, 1)
                      : partition_by_radix<ProbeT, HashedType, false>(materialized_probe, histograms_probe, radix_bits, 1);
  } else {
    radix_build = std::move(materialized_build);
    radix_probe = std::move(materialized_probe);
  }
  // :445-457: secondary predicates need every build row of a key (JoinHashBuildMode::AllPositions), Semi / Anti included
  const auto hash_tables = build<BuildT, HashedType>(radix_build, /*all_positions=*/true, radix_bits, probe_bloom, 1);
  const MultiPredicateJoinEvaluator evaluator(build_table, probe_table, mode, predicates, predicate_count);
  JoinOutput output;
  if (mode == HYB_JOIN_INNER) {
    probe_with_predicates<ProbeT, HashedType, false>(radix_probe, hash_tables, output, mode, evaluator);
  } else if (mode == HYB_JOIN_LEFT || mode == HYB_JOIN_RIGHT) {
    probe_with_predicates<ProbeT, HashedType, true>(radix_probe, hash_tables, output, mode, evaluator);
  } else {
    probe_semi_anti_with_predicates<ProbeT, HashedType>(radix_probe, hash_tables, output, mode, evaluator);
  }

  // Flatten (as join_hash_impl): partition_offsets by radix partition, slice_offsets the pos lists probe() produced.
  // Output chunks are not restated for joins with secondary predicates: output_chunk_offsets = {0, pair_count}.
  const bool semi_or_anti = mode == HYB_JOIN_SEMI || mode == HYB_JOIN_ANTI_NULL_AS_FALSE;
  const size_t list_count = output.probe_side.size();
  uint64_t total = 0;
  for (const auto& list : output.probe_side) total += list.size();
  result->pair_count = total;
  result->radix_bits = static_cast<int32_t>(radix_bits);
  result->partition_count = static_cast<uint32_t>(size_t{1} << radix_bits);
  result->probe_row_ids = static_cast<hyb_row_id*>(std::malloc(sizeof(hyb_row_id) * std::max<uint64_t>(total, 1)));
  result->build_row_ids =
      semi_or_anti ? nullptr : static_cast<hyb_row_id*>(std::malloc(sizeof(hyb_row_id) * std::max<uint64_t>(total, 1)));
  result->slice_count = static_cast<uint32_t>(list_count);
  result->slice_offsets = static_cast<uint64_t*>(std::malloc(sizeof(uint64_t) * (list_count + 1)));
  result->partition_offsets = static_cast<uint64_t*>(std::malloc(sizeof(uint64_t) * (result->partition_count + 1)));
  std::vector<uint64_t> partition_sizes(result->partition_count, 0);
  uint64_t cursor = 0;
  for (size_t list = 0; list < list_count; ++list) {
    result->slice_offsets[list] = cursor;
    const auto& probe_list = output.probe_side[list];
    if (!probe_list.empty()) {
      std::memcpy(result->probe_row_ids + cursor, probe_list.data(), sizeof(hyb_row_id) * probe_list.size());
      if (!semi_or_anti) {
        std::memcpy(result->build_row_ids + cursor, output.build_side[list].data(), sizeof(hyb_row_id) * probe_list.size());
      }
    }
    partition_sizes[radix_bits > 0 ? output.partition_of_list[list] : 0] += probe_list.size();
    cursor += probe_list.size();
  }
  result->slice_offsets[list_count] = cursor;
  uint64_t running = 0;
  for (uint32_t partition = 0; partition < result->partition_count; ++partition) {
    result->partition_offsets[partition] = running;
    running += partition_sizes[partition];
  }
  result->partition_offsets[result->partition_count] = running;
  result->output_chunk_count = 1;
  result->output_chunk_offsets = static_cast<uint64_t*>(std::malloc(sizeof(uint64_t) * 2));
  result->output_chunk_offsets[0] = 0;
  result->output_chunk_offsets[1] = total;
  return HYB_OK;
}

}  // namespace

extern "C" {

// orc_join_hash with secondary predicates `build.<build_column_id> <condition> probe.<probe_column_id>` (the build /
// probe orientation of hyb_join_hash_predicates). Modes: Inner, Left, Right, Semi, AntiNullAsFalse. Free the result with
// orc_join_result_free.
int orc_join_hash_predicates(const hyb_table_view* build_table, uint32_t build_column, const orc_pos_list* build_filter,
                             const hyb_table_view* probe_table, uint32_t probe_column, const orc_pos_list* probe_filter,
                             int32_t mode, int32_t radix_bits, const hyb_join_predicate* predicates,
                             uint32_t predicate_count, orc_join_result* out) {
  ORC_CHECK(build_table && probe_table && out && (predicates || predicate_count == 0), HYB_ERR_INVALID, "NULL argument");
  std::memset(out, 0, sizeof(*out));
  ORC_CHECK(build_column < build_table->column_count && probe_column < probe_table->column_count, HYB_ERR_INVALID,
            "join column out of range");
  // JoinHash::supports (join_hash.cpp:36-44): no AntiNullAsTrue with secondary predicates
  ORC_CHECK(mode == HYB_JOIN_INNER || mode == HYB_JOIN_LEFT || mode == HYB_JOIN_RIGHT || mode == HYB_JOIN_SEMI ||
                mode == HYB_JOIN_ANTI_NULL_AS_FALSE,
            HYB_ERR_UNSUPPORTED, "JoinMode not restated with secondary predicates");
  for (uint32_t index = 0; index < predicate_count; ++index) {
    const auto& predicate = predicates[index];
    ORC_CHECK(predicate.build_column_id < build_table->column_count && predicate.probe_column_id < probe_table->column_count,
              HYB_ERR_INVALID, "predicate column out of range");
    ORC_CHECK(predicate.condition >= HYB_PRED_EQUALS && predicate.condition <= HYB_PRED_GREATER_THAN_EQUALS,
              HYB_ERR_INVALID, "predicate condition");
    const bool build_string = column_type(build_table, predicate.build_column_id) == HYB_TYPE_STRING;
    const bool probe_string = column_type(probe_table, predicate.probe_column_id) == HYB_TYPE_STRING;
    ORC_CHECK(build_string == probe_string, HYB_ERR_INVALID, "Types of columns cannot be compared.");  // :44-46
    ORC_CHECK(!build_string, HYB_ERR_UNSUPPORTED, "string predicates are not restated");
  }
  const int32_t build_type = column_type(build_table, build_column);
  const int32_t probe_type = column_type(probe_table, probe_column);
  const auto integral = [](int32_t t) { return t == HYB_TYPE_INT32 || t == HYB_TYPE_INT64; };
  ORC_CHECK(integral(build_type) && integral(probe_type), HYB_ERR_UNSUPPORTED, "only integer join keys are restated");
  if (radix_bits < 0) {
    radix_bits = orc_calculate_radix_bits(table_row_count(build_table, build_filter), table_row_count(probe_table, probe_filter));
  }
  const size_t bits = static_cast<size_t>(radix_bits);
  const auto run = [&](auto build_key, auto probe_key) {
    return join_hash_predicates_impl<decltype(build_key), decltype(probe_key)>(
        build_table, build_column, build_filter, probe_table, probe_column, probe_filter, mode, bits, predicates,
        predicate_count, out);
  };
  if (build_type == HYB_TYPE_INT32) return probe_type == HYB_TYPE_INT32 ? run(int32_t{}, int32_t{}) : run(int32_t{}, int64_t{});
  return probe_type == HYB_TYPE_INT32 ? run(int64_t{}, int32_t{}) : run(int64_t{}, int64_t{});
}

}  // extern "C"
