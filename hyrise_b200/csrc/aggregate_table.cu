// An aggregate result as an ordinary table of the device pool (hyb_aggregate_result_table): the reference's AggregateHash
// writes its aggregates into a materialised Data table (aggregate_hash.cpp:1301-1324) and its GROUP BY columns as
// ReferenceSegments on the representative rows (:421-537), so a HAVING is a TableScan over that output and an IN subquery
// a semi join on it. Here every column is an unencoded value segment the table owns:
//   - an AGGREGATE column is the result's host values and NULL bytes, uploaded once into the chunk slices;
//   - a COLUMN column is gathered by one kernel for all COLUMN outputs: the aggregated table's column decoded at each
//     group's representative RowID (decode1 of column_pair.cuh), NULL where the row is NULL or the RowID is NULL_ROW_ID.
// Row g sits at {g / chunk_size, g % chunk_size}. Every chunk slice starts on a 256-byte boundary and has at least 64
// readable bytes after its last element, as hyb_table_append_chunk_device asks of segment buffers.
#include <algorithm>
#include <vector>

#include "column_pair.cuh"
#include "device_utils.cuh"
#include "internal.hpp"

namespace hyb {
namespace {

constexpr uint32_t kGatherThreads = 256;

// One COLUMN output: the source column's descriptors and the destination's chunk slices, `stride` bytes apart.
struct GatherColumn {
  const DevSegment* segments;
  char* values;
  uint8_t* nulls;
  uint64_t value_stride;
  uint64_t null_stride;
  int32_t data_type;
  uint32_t pad;
};

template <typename Conv, typename Out>
__device__ __forceinline__ bool gather_value(const DevSegment& segment, uint32_t row, Out* out) {
  typename Conv::T value{};
  const bool is_null = decode1<Conv>(segment, row, value);
  *out = is_null ? Out{} : static_cast<Out>(value);
  return is_null;
}

__global__ void __launch_bounds__(kGatherThreads) aggregate_table_gather_kernel(const hyb_row_id* __restrict__ row_ids,
                                                                                uint32_t group_count, uint32_t chunk_size,
                                                                                const GatherColumn* __restrict__ columns,
                                                                                uint32_t column_count) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < group_count; g += stride) {  // 32-bit: no division call
    const hyb_row_id row = row_ids[g];
    const uint32_t chunk = g / chunk_size;
    const uint32_t offset = g - chunk * chunk_size;
    for (uint32_t c = 0; c < column_count; ++c) {
      const GatherColumn column = columns[c];
      char* slice = column.values + chunk * column.value_stride;
      bool is_null = true;
      switch (column.data_type) {
        case HYB_TYPE_INT32: {
          int32_t* out = reinterpret_cast<int32_t*>(slice) + offset;
          if (row.chunk_id == HYB_INVALID_CHUNK_ID) *out = 0;
          else is_null = gather_value<AsInt64>(column.segments[row.chunk_id], row.chunk_offset, out);
          break;
        }
        case HYB_TYPE_INT64: {
          long long* out = reinterpret_cast<long long*>(slice) + offset;
          if (row.chunk_id == HYB_INVALID_CHUNK_ID) *out = 0;
          else is_null = gather_value<AsInt64>(column.segments[row.chunk_id], row.chunk_offset, out);
          break;
        }
        case HYB_TYPE_FLOAT32: {
          float* out = reinterpret_cast<float*>(slice) + offset;
          if (row.chunk_id == HYB_INVALID_CHUNK_ID) *out = 0.0f;
          else is_null = gather_value<AsFloat>(column.segments[row.chunk_id], row.chunk_offset, out);
          break;
        }
        default: {
          double* out = reinterpret_cast<double*>(slice) + offset;
          if (row.chunk_id == HYB_INVALID_CHUNK_ID) *out = 0.0;
          else is_null = gather_value<AsDouble>(column.segments[row.chunk_id], row.chunk_offset, out);
          break;
        }
      }
      column.nulls[chunk * column.null_stride + offset] = is_null ? 1 : 0;
    }
  }
}

uint64_t slice_stride(uint32_t chunk_size, size_t element_bytes) {
  const uint64_t bytes = uint64_t{chunk_size} * element_bytes + Arena::kTailPad;
  return (bytes + Arena::kAlign - 1) / Arena::kAlign * Arena::kAlign;
}

// Host bytes (group_count elements of `element_bytes`) into the chunk slices of `device`: one strided copy for the full
// chunks, one copy for the last one.
int upload_slices(hyb_context* context, char* device, uint64_t stride, const uint8_t* host, size_t element_bytes,
                  uint64_t group_count, uint32_t chunk_size) {
  const uint64_t full_chunks = group_count / chunk_size;
  const size_t slice_bytes = size_t{chunk_size} * element_bytes;
  if (full_chunks) {
    HYB_CUDA(cudaMemcpy2DAsync(device, stride, host, slice_bytes, slice_bytes, full_chunks, cudaMemcpyHostToDevice,
                               context->stream));
  }
  const uint64_t tail = group_count - full_chunks * chunk_size;
  if (tail) {
    HYB_CUDA(cudaMemcpyAsync(device + full_chunks * stride, host + full_chunks * slice_bytes, tail * element_bytes,
                             cudaMemcpyHostToDevice, context->stream));
  }
  return HYB_OK;
}

// Where one output column's chunk slices live.
struct OutputColumn {
  int32_t data_type = 0;
  char* values = nullptr;
  uint8_t* nulls = nullptr;  // nullptr: the column holds no NULL
  uint64_t value_stride = 0, null_stride = 0;
};

int check_columns(hyb_context* context, const AggregateResult& result, const hyb_aggregate_output_column* columns,
                  uint32_t column_count, Table** out_source, std::vector<int32_t>* out_types) {
  Table* source = nullptr;
  for (uint32_t c = 0; c < column_count; ++c) {
    const auto& column = columns[c];
    const std::string where = "output column " + std::to_string(c);
    if (column.kind == HYB_SORT_KEY_AGGREGATE) {
      HYB_CHECK(column.index < result.columns.size(), HYB_ERR_INVALID, where + ": aggregate index out of range");
      const auto& aggregate = result.columns[column.index];
      HYB_CHECK(!aggregate.is_any, HYB_ERR_INVALID,
                where + ": ANY has no values; take its column through HYB_SORT_KEY_COLUMN");
      HYB_CHECK(aggregate.value_type != HYB_TYPE_STRING, HYB_ERR_UNSUPPORTED,
                where + ": a string MIN / MAX stays with the CPU operator");
      out_types->push_back(aggregate.value_type);
    } else {
      HYB_CHECK(column.kind == HYB_SORT_KEY_COLUMN, HYB_ERR_INVALID, where + ": unknown kind");
      if (!source) {
        source = find_table(context, result.table);
        HYB_CHECK(source, HYB_ERR_INVALID, "the aggregated table has been dropped");
      }
      HYB_CHECK(column.index < source->column_count, HYB_ERR_INVALID, where + ": column index out of range");
      const int32_t type = source->column_types[column.index];
      HYB_CHECK(type != HYB_TYPE_STRING, HYB_ERR_UNSUPPORTED,
                where + ": a string column has no shared dictionary across source chunks");
      HYB_CHECK(data_type_size(type) != 0, HYB_ERR_INVALID,
                where + ": the column has no type (the aggregated table was uploaded without chunks)");
      out_types->push_back(type);
    }
  }
  if (source) {  // representative RowIDs must point into the table (a distributed result's may not)
    for (const hyb_row_id& row : result.row_ids) {
      if (row.chunk_id == HYB_INVALID_CHUNK_ID) continue;
      HYB_CHECK(row.chunk_id < source->chunk_count() && row.chunk_offset < source->chunk_rows[row.chunk_id],
                HYB_ERR_INVALID, "a representative RowID lies outside the aggregated table");
    }
  }
  *out_source = source;
  return HYB_OK;
}

}  // namespace
}  // namespace hyb

using namespace hyb;

extern "C" {

int hyb_aggregate_result_table(hyb_context* context, hyb_aggregate_result_t handle,
                               const hyb_aggregate_output_column* columns, uint32_t column_count, uint32_t chunk_size,
                               hyb_table_t* out_table) {
  HYB_CHECK(context && columns && out_table, HYB_ERR_INVALID, "NULL argument");
  *out_table = 0;
  HYB_CHECK(column_count > 0, HYB_ERR_INVALID, "a table needs at least one column");
  HYB_CHECK(chunk_size > 0, HYB_ERR_INVALID, "chunk_size is 0");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  const auto found = context->aggregate_results.find(handle);
  HYB_CHECK(found != context->aggregate_results.end(), HYB_ERR_INVALID, "unknown aggregate result handle");
  const AggregateResult& result = *found->second;
  Table* source = nullptr;
  std::vector<int32_t> types;
  HYB_TRY(check_columns(context, result, columns, column_count, &source, &types));
  const uint64_t groups = result.group_count;
  HYB_CHECK(groups < 0xFFFFFFFFull, HYB_ERR_UNSUPPORTED, "a table of 2^32 - 1 or more groups stays with the CPU operator");
  const uint64_t chunk_count = (groups + chunk_size - 1) / chunk_size;
  if (source) HYB_TRY(sync_table_descriptors(context, source));

  timing_begin(context);
  auto table = std::make_unique<Table>();
  table->owner = context;
  table->arena.owner = context;
  table->column_count = column_count;
  table->column_types = types;
  table->chunk_row_start.push_back(0);
  uint64_t upload_bytes = 0, gather_bytes = 0, written_bytes = 0;
  std::vector<OutputColumn> outputs(column_count);
  std::vector<GatherColumn> gathers;
  for (uint32_t c = 0; c < column_count && groups; ++c) {
    OutputColumn& output = outputs[c];
    output.data_type = types[c];
    const size_t element = data_type_size(types[c]);
    output.value_stride = slice_stride(chunk_size, element);
    output.null_stride = slice_stride(chunk_size, 1);
    output.values = static_cast<char*>(table->arena.alloc(output.value_stride * chunk_count));
    HYB_CHECK(output.values, HYB_ERR_OOM, "device column pool: out of memory for an aggregate table column");
    bool has_nulls = true;
    if (columns[c].kind == HYB_SORT_KEY_AGGREGATE) {
      const AggregateColumn& aggregate = result.columns[columns[c].index];
      has_nulls = std::find(aggregate.nulls.begin(), aggregate.nulls.end(), uint8_t{1}) != aggregate.nulls.end();
      HYB_TRY(upload_slices(context, output.values, output.value_stride, aggregate.values.data(), element, groups, chunk_size));
      upload_bytes += groups * element;
    }
    if (has_nulls) {  // COLUMN outputs always carry one: the gather writes it
      output.nulls = static_cast<uint8_t*>(table->arena.alloc(output.null_stride * chunk_count));
      HYB_CHECK(output.nulls, HYB_ERR_OOM, "device column pool: out of memory for an aggregate table NULL vector");
    }
    if (columns[c].kind == HYB_SORT_KEY_AGGREGATE) {
      if (has_nulls) {
        HYB_TRY(upload_slices(context, reinterpret_cast<char*>(output.nulls), output.null_stride,
                              result.columns[columns[c].index].nulls.data(), 1, groups, chunk_size));
        upload_bytes += groups;
      }
    } else {
      gathers.push_back(GatherColumn{source->d_segments + size_t{columns[c].index} * source->chunk_count(), output.values,
                                     output.nulls, output.value_stride, output.null_stride, types[c], 0});
      gather_bytes += groups * element;
      written_bytes += groups * (element + 1);
    }
  }

  uint32_t launches = 0;
  timing_kernel_begin(context);
  if (!gathers.empty()) {
    DeviceScratch scratch(context);
    hyb_row_id* row_ids = nullptr;
    GatherColumn* d_gathers = nullptr;
    HYB_TRY(scratch.alloc_array(groups, &row_ids));
    HYB_TRY(scratch.alloc_array(gathers.size(), &d_gathers));
    HYB_CUDA(cudaMemcpyAsync(row_ids, result.row_ids.data(), sizeof(hyb_row_id) * groups, cudaMemcpyHostToDevice,
                             context->stream));
    HYB_CUDA(cudaMemcpyAsync(d_gathers, gathers.data(), sizeof(GatherColumn) * gathers.size(), cudaMemcpyHostToDevice,
                             context->stream));
    upload_bytes += sizeof(hyb_row_id) * groups + sizeof(GatherColumn) * gathers.size();
    const uint32_t grid = static_cast<uint32_t>(std::max<uint64_t>(
        1, std::min<uint64_t>((groups + kGatherThreads - 1) / kGatherThreads, uint64_t{static_cast<uint32_t>(context->sm_count)} * 8)));
    aggregate_table_gather_kernel<<<grid, kGatherThreads, 0, context->stream>>>(row_ids, static_cast<uint32_t>(groups),
                                                                                 chunk_size, d_gathers,
                                                                                 static_cast<uint32_t>(gathers.size()));
    HYB_CUDA(cudaGetLastError());
    launches = 1;
    // the scratch returns to the cache when this scope ends; later work on the stream is ordered after the kernel
  }
  timing_kernel_end(context);

  // Segment descriptors, chunk row counts and starts as append_chunk_locked sets them for unencoded segments.
  for (uint64_t chunk = 0; chunk < chunk_count; ++chunk) {
    const uint32_t rows = static_cast<uint32_t>(std::min<uint64_t>(chunk_size, groups - chunk * chunk_size));
    for (uint32_t c = 0; c < column_count; ++c) {
      const OutputColumn& output = outputs[c];
      DevSegment segment{};
      segment.values = output.values + chunk * output.value_stride;
      segment.nulls = output.nulls ? output.nulls + chunk * output.null_stride : nullptr;
      segment.row_count = rows;
      segment.encoding = HYB_ENC_UNENCODED;
      segment.data_type = static_cast<uint8_t>(output.data_type);
      segment.vector_type = HYB_VEC_NONE;
      segment.pad = output.nulls ? kSegmentMayContainNulls : 0u;
      table->segments.push_back(segment);
    }
    table->chunk_rows.push_back(rows);
    table->chunk_row_start.push_back(table->chunk_row_start.back() + rows);
    table->max_chunk_rows = std::max(table->max_chunk_rows, rows);
  }
  table->dirty = true;
  HYB_CUDA(cudaStreamSynchronize(context->stream));  // the result's host buffers are borrowed for the duration of the call
  timing_end(context, launches, upload_bytes + gather_bytes + written_bytes, groups, groups);

  const auto table_handle = context->next_handle++;
  context->tables.emplace(table_handle, std::move(table));
  *out_table = table_handle;
  return HYB_OK;
}

}  // extern "C"
