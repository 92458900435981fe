/*
 * hyrise_b200.h — C-ABI of the Hopper (H100, sm_90a) execution path for Hyrise's three bandwidth-bound operators.
 *
 * This header is the drop-in boundary. The reference (hyrise/hyrise @ 2f7bedf3) has no FFI for operators; the seam is
 * the C++ virtual `AbstractOperator::_on_execute()` (src/lib/operators/abstract_operator.hpp:231). Each entry point
 * below replaces the body of one reference function and is what a maintainer's shim inside that function would call
 * (see INTEGRATION.md for the shim code):
 *
 *   hyb_table_scan        <-  TableScan::_on_execute                 src/lib/operators/table_scan.cpp:97-240
 *                             ColumnVsValueTableScanImpl             .../table_scan/column_vs_value_table_scan_impl.cpp:43-272
 *                             ColumnBetweenTableScanImpl             .../table_scan/column_between_table_scan_impl.cpp:42-226
 *                             ColumnIsNullTableScanImpl              .../table_scan/column_is_null_table_scan_impl.cpp
 *                             AbstractTableScanImpl::_scan_with_iterators  .../table_scan/abstract_table_scan_impl.hpp:56-242
 *   hyb_join_hash         <-  JoinHash::_on_execute / JoinHashImpl   src/lib/operators/join_hash.cpp:116-572
 *                             materialize_input/partition_by_radix/build/probe/probe_semi_anti
 *                                                                    src/lib/operators/join_hash/join_hash_steps.hpp:274-922
 *   hyb_aggregate_hash    <-  AggregateHash::_on_execute/_aggregate  src/lib/operators/aggregate_hash.cpp:950-1372
 *   hyb_table_* (pool)    <-  new "device column pool": device copies of ValueSegment / DictionarySegment /
 *                             FrameOfReferenceSegment               src/lib/storage/{value_segment.hpp:84-85,
 *                             dictionary_segment.hpp:88-90, frame_of_reference_segment.hpp:49,94-97}
 *
 * Conventions (SURVEY.md §8b):
 *   - plain C: pointers + sizes, no C++/torch types; every function returns hyb_status (0 = OK);
 *     hyb_last_error() returns a thread-local message. No exception crosses this boundary.
 *   - every entry point is thread-safe and re-entrant; inputs are borrowed and immutable for the duration of the call.
 *   - HYB_ERR_UNSUPPORTED means "run the CPU operator" (e.g. IN over a subquery, string join keys); anything else is a
 *     hard failure the shim turns into Fail(hyb_last_error()).
 *   - results stay device-resident behind handles (so the next operator can consume them without a PCIe round trip)
 *     and are copied out on request into caller-owned host memory (pinned via hyb_host_alloc for full PCIe speed).
 */
#ifndef HYRISE_B200_H
#define HYRISE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HYB_ABI_VERSION 1

/* ------------------------------------------------------------------------------------------------------------------
 * Status codes
 * ---------------------------------------------------------------------------------------------------------------- */
typedef enum hyb_status {
  HYB_OK = 0,
  HYB_ERR_INVALID = 1,     /* bad argument (maps to reference Assert/Fail -> std::logic_error, utils/assert.hpp:48-82) */
  HYB_ERR_UNSUPPORTED = 2, /* not on the GPU path: caller runs the CPU operator */
  HYB_ERR_CUDA = 3,        /* CUDA runtime failure; message holds cudaGetErrorString */
  HYB_ERR_OOM = 4,
  HYB_ERR_NOT_FOUND = 5    /* unknown handle */
} hyb_status;

/* ------------------------------------------------------------------------------------------------------------------
 * Core types — restated from src/lib/types.hpp and src/lib/all_type_variant.hpp:34-39
 * ---------------------------------------------------------------------------------------------------------------- */

/* RowID {ChunkID, ChunkOffset}, 8 bytes — types.hpp:97-117. NULL_ROW_ID = {0xFFFFFFFF, 0xFFFFFFFF}. */
typedef struct hyb_row_id {
  uint32_t chunk_id;
  uint32_t chunk_offset;
} hyb_row_id;

#define HYB_INVALID_CHUNK_ID 0xFFFFFFFFu
#define HYB_INVALID_CHUNK_OFFSET 0xFFFFFFFFu
#define HYB_INVALID_VALUE_ID 0xFFFFFFFFu /* types.hpp INVALID_VALUE_ID */
#define HYB_DEFAULT_CHUNK_SIZE 65535u    /* storage/chunk.hpp:52 */
#define HYB_FOR_BLOCK_SIZE 2048u         /* storage/frame_of_reference_segment.hpp:49 */

typedef enum hyb_data_type { /* all_type_variant.hpp:34-39 (Null excluded) */
  HYB_TYPE_INT32 = 0,
  HYB_TYPE_INT64 = 1,
  HYB_TYPE_FLOAT32 = 2,
  HYB_TYPE_FLOAT64 = 3,
  HYB_TYPE_STRING = 4 /* only value-IDs of string dictionaries reach the device */
} hyb_data_type;

typedef enum hyb_encoding { /* storage/encoding_type.hpp; the three the default TPC-H encoding produces */
  HYB_ENC_UNENCODED = 0,    /* ValueSegment<T> */
  HYB_ENC_DICTIONARY = 1,   /* DictionarySegment<T> */
  HYB_ENC_FRAME_OF_REFERENCE = 2 /* FrameOfReferenceSegment<int32_t> */
} hyb_encoding;

typedef enum hyb_vector_type { /* storage/vector_compression/compressed_vector_type.hpp */
  HYB_VEC_NONE = 0,
  HYB_VEC_FIXED_1B = 1, /* FixedWidthIntegerVector<uint8_t>  */
  HYB_VEC_FIXED_2B = 2, /* FixedWidthIntegerVector<uint16_t> */
  HYB_VEC_FIXED_4B = 3, /* FixedWidthIntegerVector<uint32_t> */
  HYB_VEC_BITPACKED = 4 /* BitPackingVector: LSB-first b-bit fields in uint64 words (compact_iterator.hpp:218-252) */
} hyb_vector_type;

/* PredicateCondition — same order/values as types.hpp:160-179 so a shim can static_cast. */
typedef enum hyb_predicate_condition {
  HYB_PRED_EQUALS = 0,
  HYB_PRED_NOT_EQUALS = 1,
  HYB_PRED_LESS_THAN = 2,
  HYB_PRED_LESS_THAN_EQUALS = 3,
  HYB_PRED_GREATER_THAN = 4,
  HYB_PRED_GREATER_THAN_EQUALS = 5,
  HYB_PRED_BETWEEN_INCLUSIVE = 6,
  HYB_PRED_BETWEEN_LOWER_EXCLUSIVE = 7,
  HYB_PRED_BETWEEN_UPPER_EXCLUSIVE = 8,
  HYB_PRED_BETWEEN_EXCLUSIVE = 9,
  HYB_PRED_IN = 10,                   /* hyb_table_scan_in; unsupported in hyb_scan_predicate */
  HYB_PRED_NOT_IN = 11,               /* hyb_table_scan_in; unsupported in hyb_scan_predicate */
  HYB_PRED_LIKE = 12,                 /* STRING dictionary columns: value_id_bounds = match bitmaps */
  HYB_PRED_NOT_LIKE = 13,             /* STRING dictionary columns: value_id_bounds = match bitmaps */
  HYB_PRED_LIKE_INSENSITIVE = 14,     /* STRING dictionary columns: value_id_bounds = match bitmaps */
  HYB_PRED_NOT_LIKE_INSENSITIVE = 15, /* STRING dictionary columns: value_id_bounds = match bitmaps */
  HYB_PRED_IS_NULL = 16,
  HYB_PRED_IS_NOT_NULL = 17
} hyb_predicate_condition;

/* JoinMode — same values as types.hpp:210. */
typedef enum hyb_join_mode {
  HYB_JOIN_INNER = 0,
  HYB_JOIN_LEFT = 1,
  HYB_JOIN_RIGHT = 2,
  HYB_JOIN_FULL_OUTER = 3, /* unsupported (as in JoinHash) */
  HYB_JOIN_CROSS = 4,      /* unsupported */
  HYB_JOIN_SEMI = 5,
  HYB_JOIN_ANTI_NULL_AS_TRUE = 6,
  HYB_JOIN_ANTI_NULL_AS_FALSE = 7
} hyb_join_mode;

/* WindowFunction subset AggregateHash supports on the device (expression/window_function_expression.hpp). */
typedef enum hyb_aggregate_function {
  HYB_AGG_MIN = 0,
  HYB_AGG_MAX = 1,
  HYB_AGG_SUM = 2,
  HYB_AGG_AVG = 3,
  HYB_AGG_COUNT = 4,      /* COUNT(column): non-NULL rows */
  HYB_AGG_COUNT_STAR = 5, /* COUNT(*): INVALID_COLUMN_ID argument in the reference */
  HYB_AGG_COUNT_DISTINCT = 6,     /* over a STRING column: a bare column whose segments carry dictionary_codes */
  HYB_AGG_STDDEV_SAMP = 7,        /* numeric arguments only (a STRING argument is HYB_ERR_INVALID) */
  HYB_AGG_ANY = 8                 /* pseudo aggregate: a single column, any type; no values (hyb_aggregate_result_values
                                     returns HYB_ERR_INVALID): the shim writes the column at the representative RowIDs */
} hyb_aggregate_function;

/* A typed scalar, already losslessly cast to the column type by the shim (utils/lossless_predicate_cast.hpp:20-60). */
typedef union hyb_value {
  int32_t i32;
  int64_t i64;
  float f32;
  double f64;
} hyb_value;

/* ------------------------------------------------------------------------------------------------------------------
 * Host-side segment / table views (borrowed pointers into the reference's pmr_vectors)
 * ---------------------------------------------------------------------------------------------------------------- */

/*
 * One segment of one chunk. Field use per encoding:
 *   UNENCODED          values = row_count x T; nulls optional.                         value_segment.hpp:84-85
 *   DICTIONARY         values = dictionary (dictionary_size x T, sorted, unique; NULL pointer for STRING),
 *                      attribute_vector = row_count value-IDs in vector_type layout,
 *                      NULL is encoded as value-ID == dictionary_size.                 dictionary_segment.hpp:88-90
 *   FRAME_OF_REFERENCE values = block minima (ceil(row_count/2048) x int32),
 *                      attribute_vector = row_count offsets in vector_type layout, nulls optional.
 *                                                                                      frame_of_reference_segment.hpp:94-97
 * nulls: one byte per row (0/1). The reference stores pmr_vector<bool> (bit-packed); the shim expands it once.
 * dictionary_codes (optional, DICTIONARY only): dictionary_size x uint64 chunk-independent group-by codes for this
 *   segment's dictionary entries — required to group by a STRING column (the shim computes them once per dictionary
 *   with the reference's own key scheme, aggregate_hash.cpp:818-925; O(dictionary) host work, not O(rows)).
 */
typedef struct hyb_segment_desc {
  int32_t encoding;    /* hyb_encoding */
  int32_t data_type;   /* hyb_data_type */
  int32_t vector_type; /* hyb_vector_type (DICTIONARY / FRAME_OF_REFERENCE) */
  int32_t bit_width;   /* BITPACKED only: bits per entry (1..32) */
  uint32_t row_count;
  uint32_t dictionary_size;
  const void* values;
  const uint8_t* nulls;
  const void* attribute_vector;
  const uint64_t* dictionary_codes;
} hyb_segment_desc;

/* A table = chunk_count x column_count segments, row-major by chunk: segments[chunk * column_count + column]. */
typedef struct hyb_table_view {
  uint32_t chunk_count;
  uint32_t column_count;
  const hyb_segment_desc* segments;
} hyb_table_view;

/* ------------------------------------------------------------------------------------------------------------------
 * Context and device column pool
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct hyb_context hyb_context; /* one per (process, device); owns streams, scratch and the column pool */
typedef uint64_t hyb_table_t;           /* device-resident table (handle into the pool) */
typedef uint64_t hyb_pos_list_t;        /* device-resident RowIDPosList set (one list per input chunk) */
typedef uint64_t hyb_join_result_t;
typedef uint64_t hyb_aggregate_result_t;

int hyb_abi_version(void);
const char* hyb_last_error(void);

/* device_index: CUDA ordinal (one process per GPU: pass LOCAL_RANK). */
int hyb_context_create(int device_index, hyb_context** out_context);
int hyb_context_destroy(hyb_context* context);
int hyb_device_count(int* out_count);
/* Block until all work queued by this context has finished. */
int hyb_context_synchronize(hyb_context* context);

/* Tuning / test knobs (not needed for correctness). The HYB_* environment variables of the same meaning are read once,
 * when the context is created; this call changes a knob afterwards. name/value pairs:
 *   "join_table"       = "auto" | "hash" | "direct" | "rank"   hash-table kind of hyb_join_hash (parity tests force each)
 *   "join_span"        = "0" | "1"   8192-row span kernels with shared-memory staged, coalesced PosList stores
 *   "join_rank"        = "ballot" | "match"
 *   "scan_bulk"        = "0" | "1"   cp.async.bulk + mbarrier input pipeline of the scan kernel
 *   "aggregate_stream" = "0" | "1"   bulk-staged streaming kernel for low-cardinality group-bys
 * Unknown names / values return HYB_ERR_INVALID. */
int hyb_context_set_option(hyb_context* context, const char* name, const char* value);

/* Pinned host memory for upload sources / result destinations (a pinned MemoryResource in the reference's terms,
 * cf. src/lib/memory/default_memory_resource.cpp:29-35). */
int hyb_host_alloc(size_t bytes, void** out_ptr);
int hyb_host_free(void* ptr);

/* Upload a whole table into the pool (H2D of every buffer the descriptors point to). */
int hyb_table_upload(hyb_context* context, const hyb_table_view* view, hyb_table_t* out_table);
/* Incremental variant: create an empty table, then append chunks (column_count segments each). */
int hyb_table_create(hyb_context* context, uint32_t column_count, hyb_table_t* out_table);
int hyb_table_append_chunk(hyb_context* context, hyb_table_t table, const hyb_segment_desc* segments);
/* Like hyb_table_append_chunk, but every pointer in `segments` already is a DEVICE pointer on this context's GPU
 * (e.g. tuples received through the multi-GPU exchange). Nothing is copied; the buffers are borrowed until the table is
 * dropped and must be 16-byte aligned with 64 readable bytes after their last element. */
int hyb_table_append_chunk_device(hyb_context* context, hyb_table_t table, const hyb_segment_desc* segments);
int hyb_table_drop(hyb_context* context, hyb_table_t table);

/*
 * Loading path: Hyrise's binary table format (BinaryParser::parse, import_export/binary/binary_parser.cpp:40-344 — what
 * hyriseBenchmarkTPCH caches under tpch_cached_tables/) -> host segments in this header's layout. Value / Dictionary /
 * FrameOfReference segments keep the reference's encoding (FixedWidthInteger and BitPacking vectors as stored), RunLength
 * segments are expanded, FixedStringDictionary and unencoded string segments become string dictionaries; every buffer sits
 * in a 256-byte aligned slot of a few large host blocks — pinned (`pinned` != 0 and a CUDA device is usable) so that
 * hyb_table_upload_binary moves the table with one DMA per block. HYB_ERR_NOT_FOUND: no such file; HYB_ERR_INVALID: what
 * the reference reports with Fail() (invalid encoding / vector type, truncated file); HYB_ERR_UNSUPPORTED: LZ4 segments.
 * The parse itself needs no GPU.
 */
typedef struct hyb_binary_table hyb_binary_table;
int hyb_binary_table_open(const char* path, int32_t pinned, hyb_binary_table** out_table);
void hyb_binary_table_close(hyb_binary_table* table);
int hyb_binary_table_info(const hyb_binary_table* table, uint32_t* out_chunk_size, uint32_t* out_chunk_count, uint32_t* out_column_count);
int hyb_binary_table_column(const hyb_binary_table* table, uint32_t column, const char** out_name, int32_t* out_data_type,
                            int32_t* out_nullable);
/* Segment descriptors (chunk-major) pointing into the table's host blocks; valid until hyb_binary_table_close. */
int hyb_binary_table_view(const hyb_binary_table* table, hyb_table_view* out_view);
/* Per chunk: the sorted-by information the file carries ({column id, SortMode} pairs, chunk.hpp). */
int hyb_binary_table_sorted_columns(const hyb_binary_table* table, uint32_t chunk, uint16_t* out_column_ids, uint8_t* out_sort_modes,
                                    uint32_t* out_count);
/* Host-resident dictionary of a string segment: entry i = chars[offsets[i] .. offsets[i + 1]). */
int hyb_binary_table_string_dictionary(const hyb_binary_table* table, uint32_t chunk, uint32_t column, const char** out_chars,
                                       const uint64_t** out_offsets, uint32_t* out_count);
/* hyb_scan_predicate.value_id_bounds for a string column of this table: per chunk DictionarySegment::lower_bound /
 * upper_bound of `value` (and of `value2` for BETWEEN; pass NULL otherwise): chunk_count x (2 | 4) entries. */
int hyb_binary_table_value_id_bounds(const hyb_binary_table* table, uint32_t column, const char* value, uint64_t value_length,
                                     const char* value2, uint64_t value2_length, uint32_t* out_bounds);

/* value_id_bounds of a LIKE predicate on a string column of this table: the per-chunk dictionary match bitmaps
 * (hyb_like_dictionary_matches over every chunk's dictionary, concatenated in chunk order). out_words == NULL: only
 * *inout_word_count is set, to the number of words needed; otherwise *inout_word_count must be at least that. */
int hyb_binary_table_like_bitmaps(const hyb_binary_table* table, uint32_t column, const char* pattern, uint64_t pattern_length,
                                  int32_t condition, uint32_t* out_words, uint32_t* inout_word_count);

/* hyb_column_scan_predicate.right_in_left of two string columns of this table: hyb_dictionary_translate of every chunk's
 * dictionaries, concatenated in chunk order (one word per right dictionary entry). out_words == NULL: only
 * *inout_count is set, to the number of words needed; otherwise *inout_count must be at least that. */
int hyb_binary_table_column_translation(const hyb_binary_table* table, uint32_t left_column, uint32_t right_column,
                                        uint32_t* out_words, uint32_t* inout_count);

/*
 * Arena upload: when the segment buffers of one or more tables live inside a few large host blocks (a pinned
 * MemoryResource arena, cf. src/lib/memory/default_memory_resource.cpp:29-35 and Chunk::migrate, storage/chunk.hpp:119),
 * DMA each block ONCE and let tables point into the device copies instead of issuing one copy per segment buffer
 * (tens of thousands at SF 10). Buffers must be >= 16-byte aligned inside their block and followed by 64 readable bytes.
 * A buffer of the view that is not inside any block is copied individually, as hyb_table_upload does.
 */
typedef struct hyb_host_block {
  const void* base;
  uint64_t bytes;
} hyb_host_block;
typedef uint64_t hyb_block_set_t;
int hyb_blocks_upload(hyb_context* context, const hyb_host_block* blocks, uint32_t block_count,
                      hyb_block_set_t* out_block_set);
int hyb_table_upload_from_blocks(hyb_context* context, const hyb_table_view* view, hyb_block_set_t block_set,
                                 hyb_table_t* out_table);
/* Releases the device copies once no table references them any more. */
int hyb_blocks_free(hyb_context* context, hyb_block_set_t block_set);
/* The host blocks of a parsed binary table (pointer to an array owned by the table) and the one-call upload. */
int hyb_binary_table_blocks(const hyb_binary_table* table, hyb_host_block* out_blocks, uint32_t* out_count);
int hyb_table_upload_binary(hyb_context* context, const hyb_binary_table* table, hyb_table_t* out_table);
int hyb_table_info(hyb_context* context, hyb_table_t table, uint32_t* out_chunk_count, uint32_t* out_column_count,
                   uint64_t* out_row_count, uint64_t* out_device_bytes);

/*
 * Attach the order ranks of a STRING dictionary column (hyb_dictionary_order_ranks over its dictionaries): `count` words,
 * one per dictionary entry, chunk after chunk. AggregateHash needs them for MIN / MAX over the column (HYB_ERR_UNSUPPORTED
 * without), and reads them as the dictionaries of an INT32 dictionary column with the same value-IDs. HYB_ERR_INVALID:
 * not a string dictionary column, `count` != the sum of the dictionary sizes, words not strictly increasing within a
 * chunk, or a word of 2^31 or more. Appending a chunk drops the ranks. Ranks that disagree across chunks (different
 * words for one string) give wrong MIN / MAX results; they cannot be checked without the strings.
 */
int hyb_table_set_string_order(hyb_context* context, hyb_table_t table, uint32_t column, const uint32_t* ranks,
                               uint64_t count);

/* ------------------------------------------------------------------------------------------------------------------
 * TableScan
 * ---------------------------------------------------------------------------------------------------------------- */

/*
 * column <condition> value / column BETWEEN lower AND upper / column IS [NOT] NULL.
 * For STRING dictionary columns the device never sees strings: the shim passes, per chunk, the value-ID bounds the
 * reference computes with DictionarySegment::lower_bound/upper_bound (dictionary_segment.cpp:94-119):
 *   value_id_bounds[2*chunk+0] = lower_bound(lower), value_id_bounds[2*chunk+1] = upper_bound(lower)        (binary)
 *   value_id_bounds[4*chunk+0..3] = lower_bound(lower), upper_bound(lower), lower_bound(upper), upper_bound(upper)
 *                                                                                                           (between)
 * with HYB_INVALID_VALUE_ID for "past the end". For numeric dictionaries leave it NULL: bounds are computed on the
 * device from `lower`/`upper`.
 * LIKE / NOT LIKE / LIKE INSENSITIVE / NOT LIKE INSENSITIVE (STRING columns only, HYB_ERR_INVALID otherwise):
 * value_id_bounds points to the per-chunk dictionary match bitmaps, the ColumnLikeTableScanImpl's dictionary path
 * (column_like_table_scan_impl.cpp:75-140). Chunk c contributes ceil(dictionary_size_c / 32) words, chunks follow one
 * another in chunk order, and entry i of a chunk's dictionary is bit (i & 31) of its word (i >> 5). A bit is the
 * matcher's result, so NOT variants pass the inverted matches (hyb_like_dictionary_matches computes them). Padding bits
 * are ignored, and the NULL value-ID (== dictionary_size) never matches. Chunks whose bitmap has no bit set are skipped,
 * one contiguous run of set bits scans like a value-ID range, any other set is looked up per row.
 */
typedef struct hyb_scan_predicate {
  uint32_t column_id;
  int32_t condition; /* hyb_predicate_condition */
  hyb_value lower;   /* the value for binary conditions; lower bound for BETWEEN */
  hyb_value upper;   /* upper bound for BETWEEN */
  const uint32_t* value_id_bounds;
} hyb_scan_predicate;

/*
 * Predicate normalisation (host only): what TableScan::create_impl does to a literal before a scan implementation sees
 * it (table_scan.cpp:340-366, :399-441) with lossless_predicate_variant_cast (utils/lossless_predicate_cast.hpp:20-66,
 * .cpp:14-73), lossless_cast (lossless_cast.hpp:31-176) and flip_predicate_condition / between_to_conditions /
 * conditions_to_between (types.cpp:51-153). A shim whose optimizer hands it a literal of another type than the column
 * calls these and passes the results on in hyb_scan_predicate; HYB_ERR_UNSUPPORTED = "no lossless form": the reference
 * falls back to the ExpressionEvaluator, i.e. the CPU operator runs.
 *   `float_col < 3.1 (double)`  ->  `float_col <= 3.0999999f`        `int_col = 16.25`  ->  HYB_ERR_UNSUPPORTED
 * value_on_left: the predicate reads `literal <condition> column`; the returned condition is for `column <cond'> value`.
 */
typedef struct hyb_literal {
  int32_t data_type; /* hyb_data_type, numeric */
  hyb_value value;
} hyb_literal;
int hyb_flip_predicate_condition(int32_t condition, int32_t* out_condition);
int hyb_next_float_towards(double value, double towards, float* out_value, int32_t* out_possible);
int hyb_lossless_predicate_cast(int32_t condition, const hyb_literal* literal, int32_t column_type, int32_t value_on_left,
                                int32_t* out_condition, hyb_value* out_value);
int hyb_lossless_between_cast(int32_t condition, const hyb_literal* lower, const hyb_literal* upper, int32_t column_type,
                              int32_t* out_condition, hyb_value* out_lower, hyb_value* out_upper);

/*
 * LikeMatcher (expression/evaluation/like_matcher.{hpp,cpp}) over one string dictionary (host only, no GPU): entry i =
 * chars[offsets[i] .. offsets[i + 1]); chars may be NULL when every entry is the empty string. out_words receives ceil(count / 32) words, bit (i & 31) of word (i >> 5) set iff
 * entry i satisfies `pattern` under `condition` (one of the four LIKE conditions; NOT variants invert), padding bits
 * cleared; out_match_count (optional) the number of set bits. `_` is one character and `%` any run; there is no escape
 * character. Patterns of the forms abc%, %abc, %abc% and %a%b%... are matched directly; any other becomes the
 * reference's anchored ECMAScript regular expression, whose `_` and `%` do not match '\n' or '\r'. INSENSITIVE lowers
 * A-Z of pattern and entries (std::tolower in the C locale). HYB_ERR_INVALID: not a LIKE condition, or a pattern that
 * is no valid regular expression (an unbalanced `[`), which the reference rejects as well.
 */
int hyb_like_dictionary_matches(const char* pattern, uint64_t pattern_length, int32_t condition, const char* chars,
                                const uint64_t* offsets, uint32_t count, uint32_t* out_words, uint32_t* out_match_count);

/*
 * Scan `table` and produce, per input chunk, the ascending list of matching RowIDs — what
 * AbstractTableScanImpl::scan_chunk returns for every chunk (table_scan.cpp:131). `input_filter` (0 = none) restricts
 * the scan to the positions of a previous scan's result on the same table (reference-table input with single-chunk
 * pos lists, abstract_dereferenced_column_table_scan_impl.cpp:38-46); the output then holds the referenced RowIDs
 * (table_scan.cpp:150-197).
 */
int hyb_table_scan(hyb_context* context, hyb_table_t table, const hyb_scan_predicate* predicate,
                   hyb_pos_list_t input_filter, hyb_pos_list_t* out_pos_list);

/*
 * <left column> <condition> <right column>: ColumnVsColumnTableScanImpl (column_vs_column_table_scan_impl.cpp) with the
 * two-iterator loop of AbstractTableScanImpl::_scan_with_iterators (abstract_table_scan_impl.hpp:56-84). condition is one
 * of HYB_PRED_EQUALS .. HYB_PRED_GREATER_THAN_EQUALS. A row matches iff neither side is NULL and `left <op> right` holds
 * in the operands' common type (the usual arithmetic conversions of std::less<void> and friends):
 *   int32/int64 x int32/int64 -> int64;  int x float -> float (the integer rounded to nearest first);  int32 x double,
 *   float x double -> double;  int64 x double -> double (the int64 rounded);  float x float -> float.
 * NaN is unequal to everything (so `!=` holds for it); -0.0 equals +0.0. STRING x STRING compares the bytes as
 * std::string::compare does; STRING x numeric is HYB_ERR_INVALID, as is any condition outside the six (the LIKE
 * conditions: HYB_ERR_UNSUPPORTED) or a column id out of range. Both ids may name the same column.
 * STRING pairs never bring strings to the device: right_in_left holds, for every chunk in chunk order, one word per entry
 * j of the RIGHT segment's dictionary: 2 * lower_bound(left dictionary of that chunk, right[j]) + (found ? 1 : 0). Left
 * value-ID i is compared as 2 * i + 1, so the two keys order exactly like the strings. Dictionaries must hold fewer than
 * 2^31 entries (HYB_ERR_UNSUPPORTED otherwise). hyb_dictionary_translate builds one chunk's words,
 * hyb_binary_table_column_translation all of a parsed binary table's. Numeric pairs pass right_in_left = NULL.
 * The output and `input_filter` behave exactly as for hyb_table_scan.
 */
typedef struct hyb_column_scan_predicate {
  uint32_t left_column_id;
  int32_t condition;              /* HYB_PRED_EQUALS .. HYB_PRED_GREATER_THAN_EQUALS */
  uint32_t right_column_id;
  uint32_t reserved;              /* 0 */
  const uint32_t* right_in_left;  /* STRING pairs only (see above); NULL for numeric pairs */
} hyb_column_scan_predicate;
int hyb_table_scan_columns(hyb_context* context, hyb_table_t table, const hyb_column_scan_predicate* predicate,
                           hyb_pos_list_t input_filter, hyb_pos_list_t* out_pos_list);

/*
 * right_in_left of one chunk (host only, no GPU): both dictionaries sorted and unique, entry i = chars[offsets[i] ..
 * offsets[i + 1]) (chars may be NULL when every entry is empty). out_words receives right_count words,
 * out_words[j] = 2 * lower_bound(left, right[j]) + (right[j] is in left ? 1 : 0), by bytewise comparison (unsigned
 * chars; a proper prefix sorts first). One merge of the two dictionaries. HYB_ERR_UNSUPPORTED: a dictionary of 2^31
 * entries or more.
 */
int hyb_dictionary_translate(const char* left_chars, const uint64_t* left_offsets, uint32_t left_count,
                             const char* right_chars, const uint64_t* right_offsets, uint32_t right_count,
                             uint32_t* out_words);

/*
 * Order ranks of a string column (host only, no GPU): every entry of `dictionary_count` sorted dictionaries (entry i of
 * dictionary d = chars[d][offsets[d][i] .. offsets[d][i + 1]), the layout of hyb_dictionary_translate; chars[d] may be
 * NULL when every entry is empty) gets its dense rank among the distinct strings of all of them, by bytewise comparison
 * (unsigned chars; a proper prefix sorts first). Equal strings share a rank. out_ranks receives the sum of counts[] words,
 * dictionary after dictionary; out_distinct_count (optional) the number of distinct strings. One k-way merge.
 * HYB_ERR_INVALID: a dictionary that is not strictly increasing; HYB_ERR_UNSUPPORTED: 2^31 or more distinct strings.
 */
int hyb_dictionary_order_ranks(uint32_t dictionary_count, const char* const* chars, const uint64_t* const* offsets,
                               const uint32_t* counts, uint32_t* out_ranks, uint32_t* out_distinct_count);

/* hyb_dictionary_order_ranks over every chunk's dictionary of a string column of a parsed binary table, in chunk order.
 * out_ranks == NULL: only *inout_count is set, to the number of words needed; otherwise *inout_count must be at least
 * that. */
int hyb_binary_table_string_order_ranks(const hyb_binary_table* table, uint32_t column, uint32_t* out_ranks,
                                        uint32_t* inout_count);

/*
 * <column> [NOT] IN (<literal>, ...): ExpressionEvaluator::_evaluate_in_expression (expression_evaluator.cpp:404-511) on a
 * list of literals, the predicate the ExpressionEvaluatorTableScanImpl fallback scans. A row is selected iff the result is
 * non-zero and not NULL:
 *   1. Only type-compatible elements count: on a STRING column the string elements (NULL elements are dropped, their type
 *      is Null); on a numeric column the numeric and the NULL elements (string elements are dropped).
 *   2. No compatible element (the empty list included): IN selects no row, NOT IN selects every row, NULL rows and the
 *      NULL_ROW_IDs of an outer join's PosList included (the result is an unnullable literal TRUE).
 *   3. Otherwise a NULL value never matches; IN matches iff the value equals some non-NULL element; NOT IN iff it equals
 *      no element and the compatible list holds no NULL (numeric `a NOT IN (1, NULL)` selects nothing).
 *   4. Equality is std::equal_to in std::common_type_t<column type, element type>, as for hyb_table_scan_columns: int x int
 *      in int64, int x float in float (the integer rounded to nearest), anything x double in double (an int64 rounded);
 *      NaN equals nothing, -0.0 equals +0.0. So `float_col IN (0.05)` matches no row, `int64_col IN (2^53 as double)`
 *      matches 2^53 and 2^53 + 1.
 * The library applies rules 1-3. A STRING column ignores `elements` and `has_null_element` and takes per-chunk dictionary
 * bitmaps in the layout of the LIKE conditions of hyb_scan_predicate (hyb_in_dictionary_matches, inverted for NOT IN);
 * dictionary_matches == NULL means "the list has no string element". A numeric column takes its numeric elements (any
 * numeric type, any order, duplicates allowed) and needs dictionary_matches == NULL; a caller leaves its string elements
 * out (the struct cannot express them, and rule 1 drops them). HYB_ERR_INVALID: a condition other than HYB_PRED_IN /
 * HYB_PRED_NOT_IN, a column id out of range, a non-numeric hyb_literal, or bitmaps on a numeric column. The output and
 * `input_filter` behave exactly as for hyb_table_scan. HYB_PRED_IN / NOT_IN inside a hyb_scan_predicate (scans and fused
 * aggregate predicates) stay HYB_ERR_UNSUPPORTED: an aggregate consumes this call's PosList through its `filter`.
 */
typedef struct hyb_in_predicate {
  uint32_t column_id;
  int32_t condition;                  /* HYB_PRED_IN | HYB_PRED_NOT_IN */
  uint32_t element_count;             /* numeric literals in `elements` */
  uint32_t has_null_element;          /* the list holds a NULL literal */
  const hyb_literal* elements;        /* numeric elements: any numeric type, any order, duplicates allowed */
  const uint32_t* dictionary_matches; /* STRING columns: per-chunk bitmaps; NULL = the list has no string element */
} hyb_in_predicate;
int hyb_table_scan_in(hyb_context* context, hyb_table_t table, const hyb_in_predicate* predicate,
                      hyb_pos_list_t input_filter, hyb_pos_list_t* out_pos_list);

/*
 * Membership of every entry of one string dictionary in a list of strings (host only, no GPU): bytewise equality, as
 * std::string's operator==. Elements and dictionary use the layout of hyb_dictionary_translate (chars may be NULL when
 * every entry is empty); the elements may come in any order and repeat. out_words receives ceil(dictionary_count / 32)
 * words, bit (i & 31) of word (i >> 5) set iff entry i is in the list (HYB_PRED_IN) or is not (HYB_PRED_NOT_IN, inverted
 * as the NOT LIKE variants are), padding bits cleared; out_match_count (optional) the number of set bits. The caller
 * passes hyb_in_predicate.dictionary_matches = NULL instead when the list has no string element (rule 2 above).
 */
int hyb_in_dictionary_matches(int32_t condition, const char* element_chars, const uint64_t* element_offsets,
                              uint32_t element_count, const char* dictionary_chars, const uint64_t* dictionary_offsets,
                              uint32_t dictionary_count, uint32_t* out_words, uint32_t* out_match_count);

/* hyb_in_predicate.dictionary_matches for a string column of a parsed binary table: hyb_in_dictionary_matches over every
 * chunk's dictionary, concatenated in chunk order. out_words == NULL: only *inout_word_count is set, to the number of
 * words needed; otherwise *inout_word_count must be at least that. */
int hyb_binary_table_in_bitmaps(const hyb_binary_table* table, uint32_t column, int32_t condition, const char* element_chars,
                                const uint64_t* element_offsets, uint32_t element_count, uint32_t* out_words,
                                uint32_t* inout_word_count);

/*
 * The numeric list of an IN predicate as the values of `column_type` it matches under rule 4 (host only, no GPU): sorted,
 * disjoint closed intervals [lo, hi] in the column's type, out_bounds[2 * i] = lo and out_bounds[2 * i + 1] = hi (the
 * member of hyb_value that column_type names). NaN elements vanish, -0.0 and +0.0 form one interval (stored as +0.0), an
 * element that no value of the column type equals (0.05 against a float column, 2^40 against int32) vanishes, and a double
 * or float element against an integer column can cover several integers. Intervals that touch are merged. On entry
 * *inout_interval_count is the capacity of out_bounds in intervals (count <= capacity suffices); on return it is the
 * number of intervals. out_bounds == NULL: only the count is returned. HYB_ERR_INVALID: a non-numeric column or element.
 */
int hyb_in_list_normalize(int32_t column_type, const hyb_literal* elements, uint32_t count, hyb_value* out_bounds,
                          uint32_t* inout_interval_count);

/* Total matches and per-chunk boundaries: out_chunk_offsets has chunk_count + 1 entries; chunk c's RowIDs are
 * [out_chunk_offsets[c], out_chunk_offsets[c+1]) of the flat list. Either pointer may be NULL. */
int hyb_pos_list_info(hyb_context* context, hyb_pos_list_t pos_list, uint64_t* out_total, uint32_t* out_chunk_count);
int hyb_pos_list_chunk_offsets(hyb_context* context, hyb_pos_list_t pos_list, uint64_t* out_chunk_offsets);
/* Copy RowIDs [begin, begin+count) of the flat list to host memory. */
int hyb_pos_list_copy(hyb_context* context, hyb_pos_list_t pos_list, uint64_t begin, uint64_t count,
                      hyb_row_id* out_row_ids);
int hyb_pos_list_free(hyb_context* context, hyb_pos_list_t pos_list);

/* ------------------------------------------------------------------------------------------------------------------
 * JoinHash (equi-join on one int32/int64 key column per side)
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct hyb_join_side {
  hyb_table_t table;
  uint32_t column_id;
  hyb_pos_list_t filter; /* 0 = all rows; else join only these positions (reference-table input) */
} hyb_join_side;

/*
 * build/probe sides are chosen by the caller exactly as JoinHash::_on_execute does (join_hash.cpp:139-155).
 * radix_bits: the reference's partition count (calculate_radix_bits, join_hash.cpp:70-114; pass -1 to have it computed
 * from the input sizes). It only fixes the ORDER and SLICING of the output: pairs are emitted grouped by
 * hash(key) & (2^radix_bits - 1) (std::hash<int> = identity), inside a partition in probe-row order, for one probe row
 * in build-row order — identical to probe() over radix-partitioned inputs (join_hash_steps.hpp:624-792).
 * Semi/Anti modes emit probe RowIDs only (probe_semi_anti, :794-922).
 */
int hyb_join_hash(hyb_context* context, const hyb_join_side* build, const hyb_join_side* probe, int32_t mode,
                  int32_t radix_bits, hyb_join_result_t* out_result);

/*
 * Secondary join predicates: `build.key = probe.key AND build.<build_column_id> <condition> probe.<probe_column_id> AND
 * ...` (JoinHash's OperatorJoinPredicates after the primary one, join_hash_steps.hpp:690-748, :844-883; the comparison
 * of MultiPredicateJoinEvaluator, multi_predicate_join_evaluator.cpp). A predicate reads `build value <condition> probe
 * value`; a caller that swaps the inputs flips each predicate's columns and condition (join_hash.cpp:158-165,
 * hyb_flip_predicate_condition).
 *   - condition: =, !=, <, <=, >, >=. A candidate (a build row with the probe row's key) passes when every predicate holds.
 *   - Columns: int32, int64, float or double, in any pairing, compared in C++'s common type as hyb_table_scan_columns
 *     compares (int x int in int64, int x float in float, anything with a double in double). NaN fails every condition
 *     but !=; -0.0 equals +0.0. A NULL on either side makes the predicate false; a NULL_ROW_ID of a side's filter reads
 *     as NULL in every column.
 *   - Inner: the pairs whose key matches and that pass, in hyb_join_hash's order (partition, probe row, build row).
 *   - Left / Right (the probe side is preserved): the passing pairs; a probe row with key matches but no passing
 *     candidate emits one (NULL_ROW_ID, probe) row where its pairs would have been; NULL keys and rows without a key
 *     match emit (NULL_ROW_ID, probe) as in hyb_join_hash.
 *   - Semi: the probe row once if some candidate passes. AntiNullAsFalse: the probe row if no candidate passes (rows
 *     without a key match and NULL keys included). AntiNullAsTrue: HYB_ERR_UNSUPPORTED.
 * predicate_count == 0 is hyb_join_hash: the same result and hyb_join_path. Otherwise the path carries
 * HYB_JOIN_PATH_SECONDARY and hyb_join_result_output_chunks returns HYB_ERR_UNSUPPORTED for the result (the reference
 * cuts its slices by probe elements, not by emitted rows). Errors: HYB_ERR_UNSUPPORTED for a string x string pair, more
 * than HYB_MAX_JOIN_PREDICATES predicates, AntiNullAsTrue, or a side whose RowIDs stand for another table's (the received
 * tuples of a radix exchange); HYB_ERR_INVALID for a string x numeric pair ("Types of columns cannot be compared"), a
 * column out of range, a condition other than the six above, or a non-zero `reserved`.
 */
#define HYB_MAX_JOIN_PREDICATES 4
typedef struct hyb_join_predicate {
  uint32_t build_column_id;
  uint32_t probe_column_id;
  int32_t condition; /* HYB_PRED_EQUALS .. HYB_PRED_GREATER_THAN_EQUALS */
  uint32_t reserved; /* must be 0 */
} hyb_join_predicate;
int hyb_join_hash_predicates(hyb_context* context, const hyb_join_side* build, const hyb_join_side* probe, int32_t mode,
                             int32_t radix_bits, const hyb_join_predicate* predicates, uint32_t predicate_count,
                             hyb_join_result_t* out_result);

/* out_pair_count: number of emitted rows; out_partition_count: 2^radix_bits. */
int hyb_join_result_info(hyb_context* context, hyb_join_result_t result, uint64_t* out_pair_count,
                         uint32_t* out_partition_count, int32_t* out_radix_bits);
/* partition_count + 1 offsets into the flat pair list (output of partition p = [off[p], off[p+1])). */
int hyb_join_result_partition_offsets(hyb_context* context, hyb_join_result_t result, uint64_t* out_offsets);
/* Copy pairs [begin, begin+count). out_build_row_ids may be NULL (always for Semi/Anti). */
int hyb_join_result_copy(hyb_context* context, hyb_join_result_t result, uint64_t begin, uint64_t count,
                         hyb_row_id* out_build_row_ids, hyb_row_id* out_probe_row_ids);
int hyb_join_result_free(hyb_context* context, hyb_join_result_t result);

/*
 * Composing operators on the device (SURVEY.md 8f-3): one side of a join result as a PosList on that side's table — the
 * reference table a following operator of the plan consumes (join_output_writing.cpp:95-200: output ReferenceSegments always
 * point at the ORIGINAL data table, which is what the RowIDs of a result already do). side: 0 = build, 1 = probe. The list
 * is in result order (not table order: `hyb_pos_list_info` reports one chunk), may hold NULL_ROW_ID for outer joins, and is
 * accepted as `filter` / `input_filter` by hyb_table_scan, hyb_join_hash and hyb_aggregate_hash like a scan's PosList:
 * scans keep the input order (abstract_dereferenced_column_table_scan_impl.cpp:49-86: matches are positions of the input
 * list, mapped back to the referenced RowIDs by table_scan.cpp:150-197), NULL rows never match / never join.
 */
int hyb_join_result_pos_list(hyb_context* context, hyb_join_result_t result, int32_t side, hyb_pos_list_t* out_pos_list);

/*
 * The chunks write_output_chunks would cut the result into (join_output_writing.cpp:205-340): the PosLists probe() emits —
 * one per non-empty radix partition, cut every PROBE_SIZE_PER_CHUNK = 131 070 probe elements of the partition
 * (join_hash_steps.hpp:47, :655) — merged while they hold fewer than MIN_SIZE = 1000 rows and the merge stays below
 * MAX_SIZE = 4000 (:255-296). out_offsets receives *inout_count + 1 offsets into the flat pair list; call with
 * out_offsets = NULL to get the count. (Slices are cut over the emitted rows of a partition: without secondary
 * predicates and Bloom-filter false positives that is the reference's element count for PK-FK joins; see DESIGN.md.)
 */
int hyb_join_result_output_chunks(hyb_context* context, hyb_join_result_t result, uint64_t* out_offsets, uint32_t* inout_count);

/*
 * Multi-GPU radix exchange, step 1 (materialize_input, join_hash_steps.hpp:274-420, without the Bloom filter): write one
 * join side as {key, RowID} tuples into caller-provided DEVICE buffers of hyb_join_side_positions() elements each:
 * out_keys[i] = key as int64, out_row_ids[i] = chunk_id + chunk_id_base | chunk_offset << 32, in row order. Rows with a
 * NULL key get out_row_ids[i] = -1 (Inner/Semi joins drop them before the exchange). The host layer partitions the
 * tuples by hash(key) & (world - 1), exchanges them with one all-to-all (NCCL) and joins what it received with
 * hyb_table_append_chunk_device + hyb_join_hash.
 */
int hyb_join_side_positions(hyb_context* context, const hyb_join_side* side, uint64_t* out_positions);
int hyb_join_materialize(hyb_context* context, const hyb_join_side* side, uint32_t chunk_id_base, void* out_keys_device,
                         void* out_row_ids_device);

/*
 * Multi-GPU radix exchange, sender side in one step (materialize_input + partition_by_radix, join_hash_steps.hpp:274-420
 * and :422-560, with the RANK that owns a radix partition as the partition): writes the side's non-NULL {key, RowID}
 * tuples into caller-provided DEVICE buffers of hyb_join_side_positions() elements each, grouped by
 * key & (partition_count - 1) and in row order inside a group (a stable split, so that the receiving rank sees the rows
 * of every source rank in their original order). out_keys[i] = key as int64, out_row_ids[i] = {chunk_id + chunk_id_base,
 * chunk_offset}. out_partition_offsets (HOST, partition_count + 1 entries): group p occupies [offsets[p], offsets[p + 1]).
 * The host layer sends group p to rank p with one all-to-all (NCCL) and joins what it received with
 * hyb_table_append_chunk_device + hyb_join_hash. partition_count: power of two <= 256.
 */
int hyb_join_partition(hyb_context* context, const hyb_join_side* side, uint32_t partition_count, uint32_t chunk_id_base,
                       void* out_keys_device, void* out_row_ids_device, uint64_t* out_partition_offsets);

/*
 * The same split fused with the exchange: ONE ranked-write kernel stores every group straight into the memory of the rank
 * that owns it (NVLink peer-to-peer stores through CUDA IPC mappings) — no send buffer, no NCCL payload transfer.
 * Between the count pass and the write pass the library calls `exchange(user, counts, dest_keys, dest_row_ids)` with this
 * rank's tuple count per destination rank; the host layer all-gathers the counts (the only collective of the exchange,
 * world_size^2 integers) and answers with, for every destination rank d, the DEVICE addresses (valid in THIS process:
 * hyb_exchange_arena_open) where this rank's group d starts inside rank d's receive arena. The call returns after this
 * rank's stores have completed; a barrier across ranks then makes every arena complete. world_size: power of two <= 16.
 */
#define HYB_IPC_HANDLE_BYTES 64
typedef int (*hyb_exchange_fn)(void* user, const uint64_t* counts, void** dest_keys, void** dest_row_ids);
int hyb_join_partition_push(hyb_context* context, const hyb_join_side* side, uint32_t world_size, uint32_t chunk_id_base,
                            hyb_exchange_fn exchange, void* user);
/* Receive arenas: plain device memory of this rank exported to / imported from the other ranks of the node. */
int hyb_exchange_arena_create(hyb_context* context, uint64_t bytes, void** out_device_ptr, void* out_ipc_handle);
int hyb_exchange_arena_open(hyb_context* context, const void* ipc_handle, void** out_peer_ptr);
int hyb_exchange_arena_close(hyb_context* context, void* peer_ptr);
int hyb_exchange_arena_destroy(hyb_context* context, void* device_ptr);

/*
 * Peer groups: the multi-GPU operators without host orchestration. One process per GPU; every rank creates its group
 * (allocating its exchange arena: a control block plus four regions of tuple_capacity tuples), the host layer
 * all-gathers the IPC handles once (the only use of torch.distributed / NCCL besides verification), every rank connects.
 * After that a distributed operator is ONE C-ABI call per rank: counts, statistics and partial groups travel through the
 * arenas with NVLink peer stores issued by the library's kernels, ranks order themselves with epoch flags polled on the
 * device, and the only host round trip is the one that reads the world x world count matrix. Every rank must make the
 * same distributed calls in the same order. world: power of two <= 16.
 */
typedef uint64_t hyb_peer_group_t;
int hyb_peer_group_create(hyb_context* context, uint32_t rank, uint32_t world, uint64_t tuple_capacity, void* out_ipc_handle,
                          hyb_peer_group_t* out_group);
/* all_ipc_handles: world x HYB_IPC_HANDLE_BYTES, in rank order (the own entry is ignored). */
int hyb_peer_group_connect(hyb_context* context, hyb_peer_group_t group, const void* all_ipc_handles);
int hyb_peer_group_destroy(hyb_context* context, hyb_peer_group_t group);

/*
 * Inner JoinHash over ranks (SURVEY.md 8e). The ranks first exchange the [min, max] of their build and probe keys through
 * the control blocks. Co-located shards (no rank's probe range touches another rank's build range) are joined locally and
 * the RowIDs are globalised by adding build_chunk_base / probe_chunk_base to the chunk ids: every rank then holds its slice
 * of EVERY radix partition, and partition p of the global result is the concatenation of the ranks' slices in rank order
 * (hyb_distributed_stats.colocated == 1). Otherwise both sides are split by the rank that owns the radix partition
 * (key & (world - 1), the reference's hash(key) & mask with the identity hash) and pushed straight into the owners' arenas
 * by the fused split + NVLink store kernel; every rank joins what it received and emits the GLOBAL RowIDs that travelled
 * with the keys: a rank ends up with the partitions p = rank (mod world) of the reference-ordered result, in the
 * reference's order (colocated == 0). HYB_JOIN_COLOCATED=0 / option "join_colocated" forces the exchange.
 */
int hyb_join_hash_distributed(hyb_context* context, hyb_peer_group_t group, const hyb_join_side* build,
                              const hyb_join_side* probe, uint32_t build_chunk_base, uint32_t probe_chunk_base,
                              int32_t radix_bits, hyb_join_result_t* out_result);

/*
 * AggregateHash over ranks: every rank pre-aggregates its shard (AVG travels as SUM and COUNT). The ranks agree on the form:
 * low cardinality (every rank's partial groups fit one 32 KB block): the blocks are stored into every peer's arena and
 * merged by all ranks in rank order — every rank returns the complete, bit-identical result; high cardinality (Q3 / Q18
 * shapes): the partial groups are partitioned by the hash of their key, pushed into the owners' tuple regions over NVLink
 * and merged by the owner — a rank returns the groups it owns (hyb_distributed_stats.aggregate_partitioned == 1).
 * Representative RowIDs refer to the global table (chunk ids shifted by chunk_id_base); position_base = number of rows of
 * the global table before this rank's shard (first-appearance order across ranks).
 * COUNT(DISTINCT) and STDDEV_SAMP return HYB_ERR_UNSUPPORTED before any exchange (their partial states do not merge
 * through the blocks); so do ANY and any aggregate over a string column (each shard would rank its own strings). Every
 * rank sees the same query, so all ranks decline together.
 */
int hyb_aggregate_hash_distributed(hyb_context* context, hyb_peer_group_t group, const struct hyb_aggregate_query* query,
                                   uint32_t chunk_id_base, uint64_t position_base, hyb_aggregate_result_t* out_result);

/* Phases of the last distributed call on this rank (CUDA-event times on the context stream). */
typedef struct hyb_distributed_stats {
  float split_count_ms;      /* per-destination counts of both sides + publishing them to the peers */
  float count_wait_ms;       /* waiting for every peer's counts (device-side flag wait) incl. the host read of the matrix */
  float push_ms;             /* fused split + NVLink stores of both sides */
  float done_wait_ms;        /* waiting for every peer's stores */
  float local_ms;            /* local join (or pre-aggregation) */
  float finish_ms;           /* RowID translation / merge */
  uint64_t tuples_sent;      /* to other ranks */
  uint64_t tuples_received;  /* from all ranks, own included */
  uint64_t nvlink_bytes;     /* bytes this rank stored into peer memory */
  uint32_t colocated;        /* join: 1 = the ranks' key ranges did not overlap across ranks, every rank joined its own shards
                                (result layout: every rank holds its slice of EVERY partition, global order = rank order
                                inside a partition); 0 = radix exchange (a partition lives on rank partition % world) */
  uint32_t aggregate_partitioned; /* aggregate: 1 = high-cardinality form — the partial groups were partitioned by the hash of
                                     their key and this rank's result holds the groups it owns (every group on exactly one
                                     rank, in the reference's order among the rank's groups; the global order is the merge
                                     of the ranks' results by representative RowID / key); 0 = every rank holds the complete
                                     result */
} hyb_distributed_stats;
int hyb_peer_group_stats(hyb_context* context, hyb_peer_group_t group, hyb_distributed_stats* out_stats);

/* ------------------------------------------------------------------------------------------------------------------
 * AggregateHash (with optionally fused scan predicates and Projection arithmetic)
 * ---------------------------------------------------------------------------------------------------------------- */

/* Arithmetic expression over columns in reverse Polish notation, evaluated with the reference's type rules
 * (expression/expression_utils.cpp:172-205: float∘float→float, int∘float→float, int∘int→int ...). A plain column is
 * the one-op program {HYB_EXPR_COLUMN}. */
typedef enum hyb_expr_op {
  HYB_EXPR_COLUMN = 0,   /* push column `column_id` */
  HYB_EXPR_LITERAL = 1,  /* push literal (type in literal_type, value in literal) */
  HYB_EXPR_ADD = 2,
  HYB_EXPR_SUB = 3,
  HYB_EXPR_MUL = 4,
  HYB_EXPR_DIV = 5,
  HYB_EXPR_MOD = 6,  /* ModuloEvaluator (expression_functors.hpp:152-186); hyb_table_scan_expression only */
  HYB_EXPR_NULL = 7  /* push a NULL literal (null_()); hyb_table_scan_expression only */
} hyb_expr_op;

typedef struct hyb_expr_node {
  int32_t op;           /* hyb_expr_op */
  uint32_t column_id;   /* COLUMN */
  int32_t literal_type; /* LITERAL: hyb_data_type */
  hyb_value literal;    /* LITERAL */
} hyb_expr_node;

#define HYB_MAX_EXPR_NODES 16
#define HYB_MAX_GROUPBY_COLUMNS 8
#define HYB_MAX_AGGREGATES 16
#define HYB_MAX_FUSED_PREDICATES 8

/*
 * Numeric predicates of the ExpressionEvaluatorTableScanImpl fallback (table_scan.cpp:312-452): comparisons, BETWEEN and
 * IS [NOT] NULL over arithmetic operands, combined with AND / OR, as ExpressionEvaluator::evaluate_expression_to_pos_list
 * computes them (expression_evaluator.cpp:1129-1262). The operand programs are RPN lists of hyb_expr_node (COLUMN,
 * LITERAL, NULL, ADD, SUB, MUL, DIV, MOD; at most HYB_MAX_EXPR_NODES nodes each). The rules:
 *   Node types   A node's type is expression_common_type of its arguments (expression_utils.cpp:172-205): int32 only
 *                with int32, int64 with ints, float32 with int32 / float32, float64 otherwise (int64 x float32 included).
 *                A NULL takes its sibling's type; NULL with NULL stays NULL (ArithmeticsLiterals evaluates
 *                `NULL - NULL` to NULL).
 *   + - *        Computed in std::common_type of the two argument types, then cast to the node type
 *                (expression_functors.hpp:136-145; int64 x float32 is computed in float and stored as double). Integer
 *                overflow wraps in two's complement; the reference leaves it undefined.
 *   /            Both arguments cast to the node type first; integer division truncates toward zero. NULL if the
 *                divisor is 0 (-0.0 included) (DivisionEvaluator, expression_functors.hpp:188-218).
 *   %            Integral % in std::common_type when both arguments are integers; otherwise std::fmod in float when
 *                both are float32 and in double else (std::fmod's promotion of an integer argument), cast to the node
 *                type. NULL if the divisor is 0 (expression_functors.hpp:152-186).
 *   Undefined    INT_MIN / -1 and INT_MIN % -1 (either width) trap in the reference. Here x / -1 is 0 - x in two's
 *                complement (so INT_MIN) and x % -1 is 0.
 *   NULL         NULL in, NULL out, for every arithmetic node.
 *   Comparisons  In std::common_type of the two sides' types, as hyb_table_scan_columns. NaN is unequal to everything,
 *                -0.0 equals +0.0, and a NULL side never matches.
 *   BETWEEN      As rewrite_between_expression (expression_evaluator.cpp:95): `value >(=) lower AND value <(=) upper`,
 *                each comparison in its own common type; _evaluate_between_expression is an equivalent special case.
 *   IS [NOT] NULL  of the operand's value.
 *   AND / OR     Intersection and union of the children's selections (expression_evaluator.cpp:1250-1262). There is
 *                no NOT on this path.
 * `terms` is a postfix list of leaves and AND / OR nodes: a leaf pushes its selection, AND / OR pop two and push one,
 * and exactly one selection remains. A leaf's operands: = .. >=: {left, right}; the four BETWEEN conditions: {value,
 * lower, upper}; IS [NOT] NULL: {operand}; unused operands have node_count 0.
 * A NULL_ROW_ID of an outer join's PosList reads as NULL in every column: it is selected iff the predicate holds with
 * every column NULL (`a + 1 IS NULL` does, a comparison never does). A predicate that reads no column selects every row
 * or none.
 * HYB_ERR_UNSUPPORTED: a STRING column or literal, an IN / NOT IN or LIKE leaf condition (hyb_table_scan_in and the LIKE
 * conditions of hyb_table_scan take those, and hyb_table_scan_expression_tests takes them as leaves of a tree), more than HYB_MAX_EXPRESSION_LEAVES leaves, more than
 * HYB_MAX_EXPRESSION_COLUMNS distinct columns, or an operand of more than HYB_MAX_EXPR_NODES nodes. HYB_ERR_INVALID: a
 * malformed term list or program (stack underflow, values left over, an unknown op or condition, a column id out of
 * range). The output and `input_filter` behave exactly as for hyb_table_scan.
 */
#define HYB_MAX_EXPRESSION_LEAVES 8
#define HYB_MAX_EXPRESSION_COLUMNS 8
typedef enum hyb_expression_term_kind {
  HYB_TERM_LEAF = 0,
  HYB_TERM_AND = 1,
  HYB_TERM_OR = 2,
  HYB_TERM_SCAN = 3, /* leaf: the next entry of tests->scans, as hyb_table_scan takes it (hyb_table_scan_expression_tests) */
  HYB_TERM_IN = 4    /* leaf: the next entry of tests->ins, as hyb_table_scan_in takes it (hyb_table_scan_expression_tests) */
} hyb_expression_term_kind;
typedef struct hyb_expression_term {
  int32_t kind;                /* hyb_expression_term_kind */
  int32_t condition;           /* LEAF: = .. >=, the four BETWEEN conditions, IS NULL, IS NOT NULL */
  uint32_t node_counts[3];     /* LEAF: nodes of each operand program */
  uint32_t reserved;           /* 0 */
  hyb_expr_node operands[3][HYB_MAX_EXPR_NODES];
} hyb_expression_term;
typedef struct hyb_expression_scan_predicate {
  uint32_t term_count;
  uint32_t reserved;                 /* 0 */
  const hyb_expression_term* terms;  /* postfix */
} hyb_expression_scan_predicate;
int hyb_table_scan_expression(hyb_context* context, hyb_table_t table, const hyb_expression_scan_predicate* predicate,
                              hyb_pos_list_t input_filter, hyb_pos_list_t* out_pos_list);

/*
 * hyb_table_scan_expression whose AND / OR tree may also hold column-test leaves: the single-column scans the reference's
 * ExpressionEvaluator runs for In and Like leaves and for string comparisons (expression_evaluator.cpp:1225-1245: a leaf
 * selects the rows whose result is non-zero and not NULL; AND / OR intersect and unite, :1249-1264).
 *   HYB_TERM_SCAN  the next entry of tests->scans (postfix order), as hyb_table_scan takes it: every condition on every
 *                  column type, string comparisons and BETWEEN through value_id_bounds, the four LIKE variants through
 *                  the dictionary match bitmaps. A numeric literal must already have the column's type: the caller
 *                  produces it with hyb_lossless_predicate_cast / hyb_lossless_between_cast and, when there is no lossless
 *                  form, writes the comparison as an operand leaf instead, which compares in the common type.
 *   HYB_TERM_IN    the next entry of tests->ins, as hyb_table_scan_in takes it (rules 1-4 there).
 * Each leaf selects exactly the rows the standalone call selects. Its `condition`, `node_counts` and `reserved` are 0.
 * Operand leaves (HYB_TERM_LEAF) and column-test leaves mix freely. A NULL_ROW_ID of an outer join's PosList reads as NULL
 * in every column: a HYB_TERM_SCAN leaf holds for it only under IS NULL, a HYB_TERM_IN leaf only for a NOT IN whose list
 * has no compatible element (rule 2 of hyb_table_scan_in), an operand leaf as in hyb_table_scan_expression.
 * hyb_operator_stats::path: 1 = column-test leaves only, 2 = both kinds (hyb_table_scan_expression reports 0).
 * HYB_ERR_INVALID: scan_count / in_count that differ from the number of HYB_TERM_SCAN / HYB_TERM_IN terms, non-zero
 * `condition` / `node_counts` / `reserved` on such a term, an IN / NOT IN condition in a scans entry, whatever
 * hyb_table_scan_expression rejects as malformed, and whatever hyb_table_scan / hyb_table_scan_in reject as invalid (LIKE
 * on a numeric column, bitmaps on a numeric IN column, ...). HYB_ERR_UNSUPPORTED: more than HYB_MAX_EXPRESSION_TESTS
 * column-test leaves, more than HYB_MAX_EXPRESSION_DEPTH selections on the postfix stack at one time, and everything
 * hyb_table_scan_expression does not support in an operand leaf (string operands among them). The old entry point keeps
 * rejecting kinds 3 and 4 with HYB_ERR_INVALID. The output and `input_filter` behave exactly as for hyb_table_scan.
 */
#define HYB_MAX_EXPRESSION_TESTS 16 /* column-test leaves, in addition to HYB_MAX_EXPRESSION_LEAVES operand leaves */
#define HYB_MAX_EXPRESSION_DEPTH 8  /* selections on the postfix stack at any time */
typedef struct hyb_expression_leaf_tests {
  uint32_t scan_count;             /* == number of HYB_TERM_SCAN terms; the k-th such term (postfix order) is scans[k] */
  uint32_t in_count;               /* == number of HYB_TERM_IN terms */
  const hyb_scan_predicate* scans;
  const hyb_in_predicate* ins;
} hyb_expression_leaf_tests;
int hyb_table_scan_expression_tests(hyb_context* context, hyb_table_t table, const hyb_expression_scan_predicate* predicate,
                                    const hyb_expression_leaf_tests* tests, hyb_pos_list_t input_filter,
                                    hyb_pos_list_t* out_pos_list);

typedef struct hyb_aggregate_def {
  int32_t function; /* hyb_aggregate_function */
  uint32_t node_count; /* 0 for COUNT(*) */
  hyb_expr_node nodes[HYB_MAX_EXPR_NODES];
} hyb_aggregate_def;

typedef struct hyb_aggregate_query {
  hyb_table_t table;
  hyb_pos_list_t filter;           /* 0 = all rows; else aggregate only these positions */
  uint32_t predicate_count;        /* fused conjunctive ColumnVsValue/Between/IsNull predicates (may be 0) */
  const hyb_scan_predicate* predicates;
  uint32_t groupby_count;
  const uint32_t* groupby_column_ids;
  uint32_t aggregate_count;
  const hyb_aggregate_def* aggregates;
} hyb_aggregate_query;

/*
 * Groups are reported in the order AggregateHash emits them: first appearance in row order, or — when the reference's
 * "immediate key" shortcut applies (single int32 group-by column with a dense key range, aggregate_hash.cpp:781-804)
 * — ascending key order with the NULL group first. Representative RowIDs mirror aggregate_hash.cpp:367,394.
 */
int hyb_aggregate_hash(hyb_context* context, const hyb_aggregate_query* query, hyb_aggregate_result_t* out_result);

/*
 * hyb_aggregate_hash whose WHERE clause also holds an ExpressionEvaluator tree: the AND / OR trees of
 * hyb_table_scan_expression_tests (operand leaves, string comparisons, LIKE, [NOT] IN), fused into the aggregate's row
 * loop instead of a scan that writes a PosList the aggregate then reads back. A row is aggregated iff
 *   - it is in query->filter (or the query has no filter),
 *   - it passes every query->predicates entry, and
 *   - the tree selects it, exactly as hyb_table_scan_expression_tests selects it for the same `predicate`, `tests` and
 *     input_filter = query->filter.
 * The result is that of the scan followed by hyb_aggregate_hash with the scan's PosList as `filter`: the same groups in
 * the same order, the same representative RowIDs, counts and integer sums; float SUM / AVG / STDDEV_SAMP to rounding
 * (the summation order may differ).
 * `tests` may be NULL when the tree has no HYB_TERM_SCAN / HYB_TERM_IN leaves: the tree is then checked by
 * hyb_table_scan_expression's rules, as hyb_table_scan_expression_tests does for such a tree.
 * Errors: whatever hyb_table_scan_expression_tests rejects for the tree, with the same code (the leaf, column and depth
 * limits included), and whatever hyb_aggregate_hash rejects for the query; a `filter` that may hold NULL_ROW_IDs stays
 * HYB_ERR_UNSUPPORTED.
 * hyb_operator_stats::path is the hyb_aggregate_path that ran: a tree takes the register-tile or the general kernel, never
 * the streaming kernels. algorithmic_bytes counts every column once, whichever of the tree, the predicates, the group-by
 * and the aggregates reads it, plus the uploaded leaf tests, bitmaps, intervals and programs.
 */
int hyb_aggregate_hash_expression(hyb_context* context, const hyb_aggregate_query* query,
                                  const hyb_expression_scan_predicate* predicate, const hyb_expression_leaf_tests* tests,
                                  hyb_aggregate_result_t* out_result);

int hyb_aggregate_result_info(hyb_context* context, hyb_aggregate_result_t result, uint64_t* out_group_count,
                              int32_t* out_used_immediate_keys);
/* One representative RowID per group (what write_groupby_output turns into ReferenceSegments, :421-537). */
int hyb_aggregate_result_row_ids(hyb_context* context, hyb_aggregate_result_t result, hyb_row_id* out_row_ids);
/*
 * Values of aggregate `aggregate_index` for all groups. Result type follows WindowFunctionTraits
 * (aggregate/window_function_traits.hpp:14-77): COUNT* -> int64; SUM(int) -> int64; SUM(float/double) -> double;
 * AVG -> double; MIN/MAX -> the column type; COUNT(DISTINCT) -> int64, never NULL (NULLs are ignored, -0.0 and +0.0
 * are one value, every NaN row is a new value); STDDEV_SAMP -> double, NULL for fewer than 2 non-NULL values.
 * `out_values` receives group_count elements of that type (8 bytes for int64/double, 4 for int32/float); out_value_type
 * tells which. out_nulls (optional) gets 1 where the reference writes NULL (aggregate_count == 0).
 *
 * Over a STRING column, as a bare column only (a string expression: HYB_ERR_UNSUPPORTED):
 *   COUNT -> int64, the non-NULL rows (value-ID != dictionary size); takes the general kernel.
 *   MIN / MAX -> out_value_type HYB_TYPE_STRING: one hyb_dictionary_position per group, the entry of the table's
 *     dictionaries holding the smallest / largest string (bytewise, as char_traits<char>::compare), NULL when the group
 *     has no non-NULL value. Needs hyb_table_set_string_order on the column; runs on the general kernel.
 * ANY -> HYB_ERR_INVALID here: its values are the column at hyb_aggregate_result_row_ids. ANY never changes the kernel
 * or the groups of the other aggregates; an all-ANY query returns what the query without aggregates returns.
 *
 * COUNT(DISTINCT) over a STRING column is accepted as a bare column whose DICTIONARY segments all carry
 * dictionary_codes (equal codes <=> equal strings); otherwise, and for a string expression, HYB_ERR_UNSUPPORTED.
 * STDDEV_SAMP uses the corrected two-pass method (a second sweep over the same rows), not Welford's sequential update:
 * results agree with the reference to rounding, and a group of equal int32 / float values gives exactly 0.0 while it
 * holds fewer than 2^22 / 2^29 rows.
 */
typedef struct hyb_dictionary_position { /* a string MIN / MAX: entry value_id of chunk chunk_id's dictionary */
  uint32_t chunk_id;
  uint32_t value_id;
} hyb_dictionary_position;
int hyb_aggregate_result_values(hyb_context* context, hyb_aggregate_result_t result, uint32_t aggregate_index,
                                void* out_values, uint8_t* out_nulls, int32_t* out_value_type);
int hyb_aggregate_result_free(hyb_context* context, hyb_aggregate_result_t result);

/*
 * Sort + Limit over an aggregate's output (operators/sort.cpp, operators/limit.cpp — `ORDER BY <aggregate> DESC LIMIT k`,
 * the tail of TPC-H Q3 / Q10 / Q18): the k groups with the largest (descending != 0) or smallest values of aggregate
 * `aggregate_index`, ties in group order (Sort is stable). The values are sorted on the device (top-k selection kernel);
 * out_group_indexes receives min(k, group_count) indexes into the result's groups. NULL values sort last.
 */
int hyb_aggregate_result_top_k(hyb_context* context, hyb_aggregate_result_t result, uint32_t aggregate_index, uint32_t k,
                               int32_t descending, uint32_t* out_group_indexes, uint32_t* out_count);

/* ------------------------------------------------------------------------------------------------------------------
 * Sort (operators/sort.cpp:287-516)
 * ---------------------------------------------------------------------------------------------------------------- */

/*
 * ORDER BY over up to HYB_MAX_SORT_COLUMNS columns. SortColumnDefinition{column, AscendingNullsFirst |
 * DescendingNullsFirst} (sort.cpp:294-296; the SQL translator maps ASC / DESC to these two, sql_translator.cpp:125-126).
 * The result is the reference's: one stable sort per definition, from the last to the first (:318-332, :422-432), each
 * putting the column's NULL rows in front of the non-NULL rows in their current order, DESC included (:435-443). So it is
 * one stable lexicographic sort whose key per column is (is-not-NULL, value):
 *   - values compare with std::less / std::greater in the column's type; ties keep the input order;
 *   - strings compare bytewise (char_traits<char>) through the ranks of hyb_table_set_string_order;
 *   - -0.0 and +0.0 tie; every NaN is one value larger than +inf (the reference's order of NaN rows is unspecified), so
 *     NaN rows come last among the non-NULL rows in ASC and first in DESC;
 *   - a NULL_ROW_ID entry of the input (one side of an outer join) is NULL in every column, as a ReferenceSegment reads it.
 */
#define HYB_MAX_SORT_COLUMNS 8
typedef struct hyb_sort_column {
  uint32_t column_id;
  int32_t descending; /* 0: AscendingNullsFirst, else DescendingNullsFirst */
} hyb_sort_column;

/*
 * Sort of a table (input_filter = 0: every row, chunk by chunk, row by row) or of a PosList on it (its order is the input
 * order, :456-501). out_pos_list: the input's RowIDs in sorted order as one chunk in result order (like
 * hyb_join_result_pos_list); it may hold NULL_ROW_ID when the input may, and every operator accepts it as a filter.
 * Every type and encoding of the pool; STRING dictionary columns need hyb_table_set_string_order.
 * HYB_ERR_UNSUPPORTED: a string column without ranks, more than HYB_MAX_SORT_COLUMNS columns, 2^32 or more rows.
 * HYB_ERR_INVALID: no columns, a column out of range, a filter on another table, an unknown handle.
 * hyb_operator_stats: kernel_launches, input_rows = output_rows, algorithmic_bytes = what the passes that ran moved
 * (key gather, digit histograms, every count + scatter pass, the RowID write); path = the number of scatter passes.
 */
int hyb_sort(hyb_context* context, hyb_table_t table, hyb_pos_list_t input_filter, const hyb_sort_column* columns,
             uint32_t column_count, hyb_pos_list_t* out_pos_list);

/*
 * The same sort over an aggregate result's groups (the Sort after an AggregateHash). A key is aggregate `index` (its
 * values as hyb_aggregate_result_values reports them, NULL where out_nulls is 1) or column `index` of the aggregated table
 * read at the group's representative RowID (what write_groupby_output's ReferenceSegments show, aggregate_hash.cpp:421-537).
 * out_group_indexes receives all group_count indexes in sorted order; LIMIT k is its first k entries. A result without
 * groups returns HYB_OK and writes nothing.
 * HYB_ERR_UNSUPPORTED: a string or ANY aggregate key (sort by the column instead), a string column without ranks, more
 * than HYB_MAX_SORT_COLUMNS keys, 2^32 or more groups. HYB_ERR_INVALID: no keys, an index out of range, an unknown kind,
 * an unknown result, a column key after the aggregated table was dropped.
 * Unlike hyb_aggregate_result_top_k (NULLs last), NULL values sort first, as the reference's Sort puts them.
 */
#define HYB_SORT_KEY_AGGREGATE 0
#define HYB_SORT_KEY_COLUMN 1
typedef struct hyb_aggregate_sort_key {
  int32_t kind; /* HYB_SORT_KEY_AGGREGATE | HYB_SORT_KEY_COLUMN */
  uint32_t index;
  int32_t descending;
} hyb_aggregate_sort_key;
int hyb_aggregate_result_sort(hyb_context* context, hyb_aggregate_result_t result, const hyb_aggregate_sort_key* keys,
                              uint32_t key_count, uint32_t* out_group_indexes);

/*
 * An aggregate result as an ordinary table of the pool: the reference's AggregateHash output (aggregate values in a
 * materialised Data table, aggregate_hash.cpp:1301-1324; GROUP BY columns through the representative rows, :421-537), so a
 * HAVING is hyb_table_scan (or any other scan) over it, an IN subquery a semi join onto it, and a view's aggregate, join
 * or sort takes it like any stored table.
 *   - Row g of the table is group g of the result, in the result's group order, at RowID {g / chunk_size, g % chunk_size};
 *     every chunk but the last holds chunk_size rows. A result without groups gives a table without chunks whose column
 *     types are set, so every operator over it returns its empty result.
 *   - Column c is columns[c]: kind HYB_SORT_KEY_AGGREGATE = aggregate `index` of the result, exactly what
 *     hyb_aggregate_result_values reports (its type, bit-identical values including NaN payloads and -0.0, its NULLs);
 *     kind HYB_SORT_KEY_COLUMN = the aggregated table's numeric column `index`, any encoding, decoded at the group's
 *     representative RowID (what write_groupby_output's ReferenceSegments show): NULL where that row is NULL (the NULL
 *     group) or the RowID is NULL_ROW_ID (the synthesised row of an empty input without GROUP BY). ANY is taken this way.
 *   - Every segment is an UNENCODED value segment in table-owned device memory. An aggregate column carries a NULL vector
 *     when one of its groups is NULL, a COLUMN column always does.
 *   - The table owns its buffers (hyb_table_drop frees them) and depends on neither the result nor the aggregated table:
 *     either may be freed or dropped first. The result stays host-resident; its values are uploaded once per call.
 * HYB_ERR_UNSUPPORTED: a string MIN / MAX, a STRING column (rows from different source chunks share no dictionary),
 * 2^32 - 1 or more groups. HYB_ERR_INVALID: NULL pointers, no columns, chunk_size 0, an unknown result, an unknown kind,
 * an index out of range, ANY as an aggregate column (take it through HYB_SORT_KEY_COLUMN), a COLUMN column after the
 * aggregated table was dropped or with a representative RowID outside it (a distributed result's global RowIDs).
 * hyb_operator_stats: input_rows = output_rows = group_count; kernel_launches = 1 when a COLUMN column and a group exist
 * (aggregate_table_gather_kernel, all COLUMN columns in one launch), else 0; algorithmic_bytes = bytes uploaded
 * (aggregate values and NULL bytes, the representative RowIDs when gathered) + source column bytes gathered (element size
 * per group and COLUMN column) + bytes the gather writes (element size + 1 NULL byte per group and COLUMN column);
 * path = 0.
 */
typedef struct hyb_aggregate_output_column {
  int32_t kind; /* HYB_SORT_KEY_AGGREGATE | HYB_SORT_KEY_COLUMN, the vocabulary of hyb_aggregate_sort_key */
  uint32_t index;
} hyb_aggregate_output_column;
int hyb_aggregate_result_table(hyb_context* context, hyb_aggregate_result_t result,
                               const hyb_aggregate_output_column* columns, uint32_t column_count, uint32_t chunk_size,
                               hyb_table_t* out_table);

/* ------------------------------------------------------------------------------------------------------------------
 * Instrumentation (fills the reference's performance_data, operators/operator_performance_data.hpp:46-97)
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct hyb_operator_stats {
  float device_ms;            /* CUDA-event time of the operator's kernels on the context stream */
  float dominant_kernel_ms;   /* the bandwidth-bound kernel alone (scan / probe / aggregate kernel) */
  uint32_t kernel_launches;   /* kernels launched by the last operator call */
  uint32_t path;              /* hyb_aggregate_path of an AggregateHash call, hyb_join_path of a JoinHash call; 0 after
                                 a scan */
  uint64_t algorithmic_bytes; /* compulsory traffic of the dominant kernel (SURVEY.md §8d) */
  uint64_t input_rows;
  uint64_t output_rows;
} hyb_operator_stats;

/* The kernel whose groups an AggregateHash call returned (hyb_operator_stats::path). Attempts that overflow fall back in
 * this order, so the code names the last kernel launched before the result was materialised. */
typedef enum hyb_aggregate_path {
  HYB_AGG_PATH_NONE = 0,            /* not an aggregate */
  HYB_AGG_PATH_STREAM_STATIC = 1,   /* aggregate_stream_static_kernel: a row loop compiled for the plan's shape */
  HYB_AGG_PATH_STREAM_GENERIC = 2,  /* aggregate_stream_kernel: the layout-generic row loop */
  HYB_AGG_PATH_TILE_G4 = 3,         /* aggregate_fast_kernel with 4 group slots (1 slot when there is no group-by) */
  HYB_AGG_PATH_TILE_G8 = 4,         /* aggregate_fast_kernel with 8 group slots */
  HYB_AGG_PATH_GENERAL = 5,         /* aggregate_general_kernel on its first group table */
  HYB_AGG_PATH_GENERAL_REGROWN = 6, /* aggregate_general_kernel after at least one larger group table or larger
                                       COUNT(DISTINCT) set */
} hyb_aggregate_path;

/* The table and kernels of a JoinHash call (hyb_operator_stats::path): one TABLE code | one PROBE code | RERUN.
 * Combinations that cannot occur: a rank table is built only from strictly increasing (so unique) keys and never reruns,
 * and the tile kernels' lean loop reads direct tables only (rank | TILE_LEAN); hash tables never take the span kernels or
 * the lean loop (the lean loop and the span kernels index a direct or rank table); Semi / Anti joins rerun only with
 * secondary predicates and never take the span kernels (both serve Inner joins only); TABLE_HASH needs int32 keys on both sides, TABLE_HASH_WIDE
 * an int64 key on either side; DIRECT_SHIFTED takes the span kernels or the lean loop only for int64 probe keys. */
typedef enum hyb_join_path {
  HYB_JOIN_PATH_TABLE_RANK = 1,            /* rank table: presence bits + smallest position per 32 key values */
  HYB_JOIN_PATH_TABLE_DIRECT = 2,          /* direct table indexed by key - min */
  HYB_JOIN_PATH_TABLE_DIRECT_SHIFTED = 3,  /* direct table indexed by (key - min) >> shift, shift > 0 (the build keys
                                              agree in their `shift` low bits) */
  HYB_JOIN_PATH_TABLE_HASH = 4,            /* open-addressing table, 32-bit key compare */
  HYB_JOIN_PATH_TABLE_HASH_WIDE = 5,       /* open-addressing table, low 32 bits in the slot, full int64 key verified */
  HYB_JOIN_PATH_TABLE_MASK = 0xF,
  HYB_JOIN_PATH_PROBE_NONE = 0x00,         /* no probe rows: no probe kernel ran */
  HYB_JOIN_PATH_PROBE_SPAN = 0x10,         /* join_span_count_kernel + join_span_write_kernel */
  HYB_JOIN_PATH_PROBE_TILE_LEAN = 0x20,    /* tile kernels with the lean direct-table loop enabled for eligible tiles */
  HYB_JOIN_PATH_PROBE_TILE = 0x30,         /* tile kernels, generic loop only */
  HYB_JOIN_PATH_PROBE_MASK = 0xF0,
  HYB_JOIN_PATH_RERUN = 0x100,             /* duplicate build keys: the per-key position lists were built and the probe
                                              ran again on the tile kernels' generic loop; the PROBE code names the first
                                              probe */
  HYB_JOIN_PATH_SECONDARY = 0x200,         /* hyb_join_hash_predicates with predicates: the tile kernels' generic loop
                                              evaluated them per candidate (PROBE_TILE); a duplicated build key reruns,
                                              Semi / Anti joins included */
} hyb_join_path;

/* Stats of the last operator call made on this context by the calling thread. */
int hyb_last_operator_stats(hyb_context* context, hyb_operator_stats* out_stats);

/* Multi-GPU support: raw device pointers of result buffers so the host layer can hand them to NCCL
 * (torch.distributed) for the radix exchange. Pointers stay valid until the result is freed. */
int hyb_pos_list_device_ptr(hyb_context* context, hyb_pos_list_t pos_list, void** out_device_row_ids);
int hyb_join_result_device_ptrs(hyb_context* context, hyb_join_result_t result, void** out_build_row_ids,
                                void** out_probe_row_ids);
/* The context's CUDA stream (cudaStream_t as void*), so torch can order its collectives after our kernels. */
int hyb_context_stream(hyb_context* context, void** out_stream);

#ifdef __cplusplus
}
#endif

#endif /* HYRISE_B200_H */
