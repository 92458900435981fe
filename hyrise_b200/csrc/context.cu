// Context, device column pool (arena + segment upload), handle registry, timing. Host-side only; no kernels here.
//
// The pool is the "new src/lib/storage device column pool" of the north star: device copies of the buffers behind
// ValueSegment (value_segment.hpp:84-85), DictionarySegment (dictionary_segment.hpp:88-90) and
// FrameOfReferenceSegment (frame_of_reference_segment.hpp:94-97), addressed by (table, chunk, column).
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "device_utils.cuh"
#include "internal.hpp"

namespace hyb {

static thread_local std::string g_last_error;

void set_error(const std::string& message) { g_last_error = message; }

int fail(int status, const std::string& message) {
  g_last_error = message;
  return status;
}

static void cache_release_free_blocks(hyb_context* context);

// cudaMalloc outside the block cache (table slabs, exchange arenas): on out-of-memory the context's idle cache blocks — up to
// 64 GiB after a big join — go back to the driver and the allocation is tried once more.
cudaError_t device_malloc_retry(hyb_context* context, void** out, size_t bytes) {
  cudaError_t error = cudaMalloc(out, bytes);
  if (error == cudaErrorMemoryAllocation && context) {
    cudaGetLastError();
    cache_release_free_blocks(context);
    error = cudaMalloc(out, bytes);
  }
  if (error != cudaSuccess) cudaGetLastError();
  return error;
}

// ---------------------------------------------------------------------------------------------------------------------
// Arena
// ---------------------------------------------------------------------------------------------------------------------
void* Arena::alloc(size_t bytes) {
  const size_t need = ((bytes + kTailPad + kAlign - 1) / kAlign) * kAlign;
  if (_slabs.empty() || _slabs.back().offset + need > _slabs.back().size) {
    // Slabs grow geometrically (64 MB .. 1 GB) so SF100 tables need tens, not thousands, of cudaMalloc calls.
    size_t slab_size = std::max<size_t>(need, std::min<size_t>(size_t{1} << 30, std::max<size_t>(size_t{64} << 20,
                                                                                                   _reserved / 2)));
    slab_size = ((slab_size + kAlign - 1) / kAlign) * kAlign;
    char* base = nullptr;
    if (device_malloc_retry(owner, reinterpret_cast<void**>(&base), slab_size) != cudaSuccess) return nullptr;
    _slabs.push_back({base, slab_size, 0});
    _reserved += slab_size;
  }
  auto& slab = _slabs.back();
  void* ptr = slab.base + slab.offset;
  slab.offset += need;
  _used += need;
  return ptr;
}

void Arena::release() {
  for (auto& slab : _slabs) cudaFree(slab.base);
  _slabs.clear();
  _reserved = _used = 0;
}

BlockSet::~BlockSet() {
  for (auto& block : blocks) device_free(owner, block.device_base);
}

const void* BlockSet::translate(const void* host, size_t bytes) const {
  const char* pointer = static_cast<const char*>(host);
  for (const auto& block : blocks) {
    if (pointer >= block.host_base && pointer + bytes <= block.host_base + block.bytes) {
      return block.device_base + (pointer - block.host_base);
    }
  }
  return nullptr;
}

// Descriptor arrays / tile maps: cached device blocks when the table knows its context (every table created through the
// C-ABI does), driver allocations otherwise.
static cudaError_t table_alloc(hyb_context* owner, size_t bytes, void** out) {
  if (owner) return device_alloc(owner, bytes, out) == HYB_OK ? cudaSuccess : cudaErrorMemoryAllocation;
  return cudaMalloc(out, bytes);
}

static void table_free(hyb_context* owner, void* ptr) {
  if (!ptr) return;
  if (owner) {
    device_free(owner, ptr);
  } else {
    cudaFree(ptr);
  }
}

Table::~Table() {
  table_free(owner, d_segments);
  table_free(owner, d_chunk_row_start);
  for (auto& entry : d_tile_maps) table_free(owner, entry.second.first);
}

Table::StringColumnView::~StringColumnView() {
  device_free(owner, d_segments);
  device_free(owner, d_words);
  device_free(owner, d_first_entry);
}

PosList::~PosList() {
  device_free(owner, d_row_ids);
  device_free(owner, d_chunk_end);
}

JoinResult::~JoinResult() {
  device_free(owner, d_build);
  device_free(owner, d_probe);
  device_free(owner, d_partition_offsets);
}

Table* find_table(hyb_context* context, hyb_table_t handle) {
  auto it = context->tables.find(handle);
  return it == context->tables.end() ? nullptr : it->second.get();
}

PosList* find_pos_list(hyb_context* context, hyb_pos_list_t handle) {
  auto it = context->pos_lists.find(handle);
  return it == context->pos_lists.end() ? nullptr : it->second.get();
}

int pos_list_total(hyb_context* context, const PosList* list, uint64_t* out_rows) {
  HYB_CUDA(cudaStreamSynchronize(context->stream));
  HYB_CUDA(cudaMemcpy(out_rows, list->d_chunk_end + list->chunk_count, sizeof(uint64_t), cudaMemcpyDeviceToHost));
  // a scan over a table without rows launches no tile: its total stays at the "unset" fill
  if (*out_rows == ~uint64_t{0}) *out_rows = 0;
  return HYB_OK;
}

static size_t cache_rounded_size(size_t bytes) {
  if (bytes <= 512) return 512;
  if (bytes >= (size_t{1} << 20)) return (bytes + (size_t{1} << 20) - 1) & ~((size_t{1} << 20) - 1);  // 1 MiB steps
  size_t size = 512;
  while (size < bytes) size <<= 1;
  return size;
}

static void cache_release_free_blocks(hyb_context* context) {
  auto& cache = context->cache;
  if (cache.free_blocks.empty()) return;
  cudaStreamSynchronize(context->stream);  // queued kernels may still use blocks that were returned after launch
  for (auto& entry : cache.free_blocks) {
    cudaFree(entry.second);
    cache.block_size.erase(entry.second);
  }
  cache.free_blocks.clear();
  cache.free_bytes = 0;
}

int device_alloc(hyb_context* context, size_t bytes, void** out) {
  *out = nullptr;
  auto& cache = context->cache;
  const size_t size = cache_rounded_size(bytes);
  // best fit, wasting at most 1/8 of the block (large blocks are kept for large requests)
  const auto it = cache.free_blocks.lower_bound(size);
  if (it != cache.free_blocks.end() && it->first <= size + std::max<size_t>(size / 8, size_t{1} << 20)) {
    *out = it->second;
    cache.free_bytes -= it->first;
    cache.free_blocks.erase(it);
    return HYB_OK;
  }
  void* block = nullptr;
  cudaError_t error = cudaMalloc(&block, size);
  if (error == cudaErrorMemoryAllocation) {
    cudaGetLastError();
    cache_release_free_blocks(context);
    error = cudaMalloc(&block, size);
  }
  HYB_CUDA(error);
  cache.block_size.emplace(block, size);
  *out = block;
  return HYB_OK;
}

void device_free(hyb_context* context, void* ptr) {
  if (!ptr || !context) return;
  auto& cache = context->cache;
  const auto it = cache.block_size.find(ptr);
  if (it == cache.block_size.end()) return;  // not ours (adopted caller buffer)
  cache.free_blocks.emplace(it->second, ptr);
  cache.free_bytes += it->second;
  // Bound what an idle context holds on to: beyond 64 GiB of unused blocks, give everything back to the driver.
  if (cache.free_bytes > (size_t{64} << 30)) cache_release_free_blocks(context);
}

void device_cache_destroy(hyb_context* context) {
  cudaStreamSynchronize(context->stream);
  for (auto& entry : context->cache.block_size) cudaFree(entry.first);
  context->cache.block_size.clear();
  context->cache.free_blocks.clear();
  context->cache.free_bytes = 0;
}

int sync_table_descriptors(hyb_context* context, Table* table) {
  if (!table->dirty) return HYB_OK;
  const uint32_t chunk_count = table->chunk_count();
  if (table->fixed_single_chunk_capacity && table->d_segments) {
    // only the row count changed: patch the descriptor (stream-ordered; the sources are members that outlive the copies'
    // staging) and keep the tile maps
    HYB_CUDA(cudaMemcpyAsync(table->d_segments, table->segments.data(), sizeof(DevSegment), cudaMemcpyHostToDevice, context->stream));
    HYB_CUDA(cudaMemcpyAsync(table->d_chunk_row_start, table->chunk_row_start.data(), 2 * sizeof(uint64_t), cudaMemcpyHostToDevice,
                             context->stream));
    table->dirty = false;
    return HYB_OK;
  }
  if (table->d_chunk_capacity < chunk_count || !table->d_segments) {
    // Descriptor arrays are read by kernels already queued on the stream: wait before replacing them.
    HYB_CUDA(cudaStreamSynchronize(context->stream));
    table_free(table->owner, table->d_segments);
    table_free(table->owner, table->d_chunk_row_start);
    table->d_segments = nullptr;
    table->d_chunk_row_start = nullptr;
    table->d_chunk_capacity = std::max<uint32_t>(chunk_count, 16);
    HYB_CUDA(table_alloc(table->owner, sizeof(DevSegment) * size_t{table->d_chunk_capacity} * table->column_count,
                         reinterpret_cast<void**>(&table->d_segments)));
    HYB_CUDA(table_alloc(table->owner, sizeof(uint64_t) * (size_t{table->d_chunk_capacity} + 1),
                         reinterpret_cast<void**>(&table->d_chunk_row_start)));
  }
  // Column-major staging so that one column's descriptors are contiguous for the kernels.
  std::vector<DevSegment> staged(size_t{chunk_count} * table->column_count);
  for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
    for (uint32_t column = 0; column < table->column_count; ++column) {
      staged[size_t{column} * chunk_count + chunk] = table->segments[size_t{chunk} * table->column_count + column];
    }
  }
  if (!staged.empty()) {
    HYB_CUDA(cudaMemcpyAsync(table->d_segments, staged.data(), staged.size() * sizeof(DevSegment),
                             cudaMemcpyHostToDevice, context->stream));
  }
  HYB_CUDA(cudaMemcpyAsync(table->d_chunk_row_start, table->chunk_row_start.data(),
                           table->chunk_row_start.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, context->stream));
  // `staged` is pageable, so the copies above have completed with respect to the host buffer on return.
  HYB_CUDA(cudaStreamSynchronize(context->stream));
  for (auto& entry : table->d_tile_maps) table_free(table->owner, entry.second.first);
  table->d_tile_maps.clear();
  table->key_bounds.clear();
  table->plan_memo.clear();
  table->string_views.clear();
  table->dirty = false;
  return HYB_OK;
}

int get_tile_map(hyb_context* context, Table* table, uint32_t tile_rows, const uint2** out_device,
                 uint32_t* out_tile_count) {
  auto it = table->d_tile_maps.find(tile_rows);
  if (it != table->d_tile_maps.end() && table->fixed_single_chunk_capacity) {
    *out_device = it->second.first;
    *out_tile_count = (table->chunk_rows[0] + tile_rows - 1) / tile_rows;  // the map covers the whole capacity
    return HYB_OK;
  }
  if (it == table->d_tile_maps.end()) {
    // One entry per tile: {chunk, first row | last-tile-of-chunk flag in bit 31}. Tiles never straddle chunks.
    std::vector<uint2> map;
    const uint32_t chunk_count = table->chunk_count();
    for (uint32_t chunk = 0; chunk < chunk_count; ++chunk) {
      const uint32_t rows = table->fixed_single_chunk_capacity ? table->fixed_single_chunk_capacity : table->chunk_rows[chunk];
      for (uint32_t row0 = 0; row0 < rows; row0 += tile_rows) {
        const bool last = row0 + tile_rows >= rows;
        map.push_back(make_uint2(chunk, row0 | (last ? 0x80000000u : 0u)));
      }
    }
    uint2* device = nullptr;
    HYB_CUDA(table_alloc(table->owner, sizeof(uint2) * std::max<size_t>(map.size(), 1), reinterpret_cast<void**>(&device)));
    if (!map.empty()) {
      // stream-ordered behind whatever used the cached block before; `map` is pageable: staged before the call returns
      HYB_CUDA(cudaMemcpyAsync(device, map.data(), sizeof(uint2) * map.size(), cudaMemcpyHostToDevice, context->stream));
    }
    it = table->d_tile_maps.emplace(tile_rows, std::make_pair(device, static_cast<uint32_t>(map.size()))).first;
  }
  *out_device = it->second.first;
  *out_tile_count = table->fixed_single_chunk_capacity ? (table->chunk_rows[0] + tile_rows - 1) / tile_rows : it->second.second;
  return HYB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Timing: CUDA events on the context stream (the stream every kernel of this library is launched on).
// ---------------------------------------------------------------------------------------------------------------------
static void ensure_events(hyb_context* context) {
  auto& timing = context->timing;
  if (!timing.op_begin) {
    cudaEventCreate(&timing.op_begin);
    cudaEventCreate(&timing.op_end);
    for (int span = 0; span < OperatorTiming::kMaxKernelSpans; ++span) {
      cudaEventCreate(&timing.kernel_begin[span]);
      cudaEventCreate(&timing.kernel_end[span]);
    }
    cudaEventCreate(&timing.count_ready);
    cudaHostAlloc(&timing.h_output_count, sizeof(uint64_t), cudaHostAllocPortable);
    *timing.h_output_count = 0;
  }
}

void timing_begin(hyb_context* context) {
  ensure_events(context);
  context->timing.valid = false;
  context->timing.kernel_spans = 0;
  cudaEventRecord(context->timing.op_begin, context->stream);
}

void timing_kernel_begin(hyb_context* context) {
  auto& timing = context->timing;
  if (timing.kernel_spans < OperatorTiming::kMaxKernelSpans) {
    cudaEventRecord(timing.kernel_begin[timing.kernel_spans], context->stream);
  }
}

void timing_kernel_end(hyb_context* context) {
  auto& timing = context->timing;
  if (timing.kernel_spans < OperatorTiming::kMaxKernelSpans) {
    cudaEventRecord(timing.kernel_end[timing.kernel_spans], context->stream);
    ++timing.kernel_spans;
  }
}

void timing_end(hyb_context* context, uint32_t launches, uint64_t algorithmic_bytes, uint64_t input_rows,
                uint64_t output_rows) {
  auto& timing = context->timing;
  cudaEventRecord(timing.op_end, context->stream);
  timing.stats = hyb_operator_stats{};
  timing.stats.kernel_launches = launches;
  timing.stats.algorithmic_bytes = algorithmic_bytes;
  timing.stats.input_rows = input_rows;
  timing.stats.output_rows = output_rows;
  timing.d_output_count = nullptr;
  timing.output_bytes_each = 0;
  timing.valid = true;
}

// Operators whose output size is data dependent call this right after timing_end.
void timing_output_count(hyb_context* context, const uint64_t* d_count, uint32_t bytes_each) {
  auto& timing = context->timing;
  timing.d_output_count = d_count;
  timing.output_bytes_each = bytes_each;
  cudaMemcpyAsync(timing.h_output_count, d_count, sizeof(uint64_t), cudaMemcpyDeviceToHost, context->stream);
  cudaEventRecord(timing.count_ready, context->stream);
}

// One CTA per dictionary segment: does any row carry the NULL value-ID (== dictionary size)? Lets kernels skip NULL
// handling for segments without NULLs (the reference knows this from the column definition, `_column_is_nullable`).
__global__ void probe_null_value_ids_kernel(const DevSegment* __restrict__ segments, uint32_t count,
                                            uint32_t* __restrict__ flags) {
  const uint32_t index = blockIdx.x;
  if (index >= count) return;
  const DevSegment segment = segments[index];
  bool found = false;
  for (uint32_t row = threadIdx.x; row < segment.row_count; row += blockDim.x) {
    found = found || load_code1(segment.av, segment.vector_type, segment.bit_width, row) >= segment.dict_size;
  }
  if (__syncthreads_or(found) && threadIdx.x == 0) flags[index] = 1;
}

// Fills DevSegment::pad for the segments [first_segment, end) of the host copy (call with the stream idle or ordered).
int probe_null_flags(hyb_context* context, Table* table, size_t first_segment) {
  std::vector<size_t> dictionary_segments;
  for (size_t index = first_segment; index < table->segments.size(); ++index) {
    auto& segment = table->segments[index];
    segment.pad = 0;
    if (segment.encoding == HYB_ENC_DICTIONARY) {
      if (segment.row_count) dictionary_segments.push_back(index);
    } else if (segment.nulls) {
      segment.pad = kSegmentMayContainNulls;
    }
  }
  if (dictionary_segments.empty()) return HYB_OK;
  std::vector<DevSegment> staged;
  staged.reserve(dictionary_segments.size());
  for (const size_t index : dictionary_segments) staged.push_back(table->segments[index]);
  void* d_segments = nullptr;
  void* d_flags = nullptr;
  HYB_TRY(device_alloc(context, sizeof(DevSegment) * staged.size(), &d_segments));
  HYB_TRY(device_alloc(context, sizeof(uint32_t) * staged.size(), &d_flags));
  HYB_CUDA(cudaMemcpyAsync(d_segments, staged.data(), sizeof(DevSegment) * staged.size(), cudaMemcpyHostToDevice, context->stream));
  HYB_CUDA(cudaMemsetAsync(d_flags, 0, sizeof(uint32_t) * staged.size(), context->stream));
  probe_null_value_ids_kernel<<<static_cast<uint32_t>(staged.size()), 256, 0, context->stream>>>(
      static_cast<const DevSegment*>(d_segments), static_cast<uint32_t>(staged.size()), static_cast<uint32_t*>(d_flags));
  HYB_CUDA(cudaGetLastError());
  std::vector<uint32_t> flags(staged.size());
  HYB_CUDA(cudaMemcpyAsync(flags.data(), d_flags, sizeof(uint32_t) * flags.size(), cudaMemcpyDeviceToHost, context->stream));
  HYB_CUDA(cudaStreamSynchronize(context->stream));
  device_free(context, d_segments);
  device_free(context, d_flags);
  for (size_t i = 0; i < dictionary_segments.size(); ++i) {
    if (flags[i]) table->segments[dictionary_segments[i]].pad = kSegmentMayContainNulls;
  }
  return HYB_OK;
}

}  // namespace hyb

using namespace hyb;

// ---------------------------------------------------------------------------------------------------------------------
// C-ABI: context
// ---------------------------------------------------------------------------------------------------------------------
extern "C" {

int hyb_abi_version(void) { return HYB_ABI_VERSION; }

const char* hyb_last_error(void) { return g_last_error.c_str(); }

int hyb_device_count(int* out_count) {
  HYB_CHECK(out_count, HYB_ERR_INVALID, "out_count is NULL");
  int count = 0;
  cudaError_t error = cudaGetDeviceCount(&count);
  if (error != cudaSuccess) {
    cudaGetLastError();
    *out_count = 0;
    return fail(HYB_ERR_CUDA, std::string("cudaGetDeviceCount: ") + cudaGetErrorString(error));
  }
  *out_count = count;
  return HYB_OK;
}

static bool apply_option(hyb::ContextOptions& options, const std::string& name, const std::string& value) {
  const auto as_flag = [&](bool* out) {
    if (value == "0" || value == "1") {
      *out = value == "1";
      return true;
    }
    return false;
  };
  if (name == "join_table") {
    if (value == "auto") options.join_table = hyb::ContextOptions::kAuto;
    else if (value == "hash") options.join_table = hyb::ContextOptions::kHash;
    else if (value == "direct") options.join_table = hyb::ContextOptions::kDirect;
    else if (value == "rank") options.join_table = hyb::ContextOptions::kRank;
    else return false;
    return true;
  }
  if (name == "join_rank") {
    if (value != "ballot" && value != "match") return false;
    options.join_ballot_rank = value == "ballot";
    return true;
  }
  if (name == "join_span") return as_flag(&options.join_span);
  if (name == "join_colocated") return as_flag(&options.join_colocated);
  if (name == "scan_bulk") return as_flag(&options.scan_bulk);
  if (name == "scan_two_pass") return as_flag(&options.scan_two_pass);
  if (name == "aggregate_stream") return as_flag(&options.aggregate_stream);
  if (name == "aggregate_static_shapes") return as_flag(&options.aggregate_static_shapes);
  if (name == "trace") return as_flag(&options.trace);
  if (name == "aggregate_stages") {
    if (value.size() != 1 || value[0] < '2' || value[0] > '8') return false;
    options.aggregate_stages = static_cast<uint32_t>(value[0] - '0');
    return true;
  }
  return false;
}

int hyb_context_set_option(hyb_context* context, const char* name, const char* value) {
  HYB_CHECK(context && name && value, HYB_ERR_INVALID, "NULL argument");
  std::lock_guard<std::mutex> lock(context->mutex);
  HYB_CHECK(apply_option(context->options, name, value), HYB_ERR_INVALID,
            std::string("unknown option ") + name + " = " + value);
  return HYB_OK;
}

int hyb_context_create(int device_index, hyb_context** out_context) {
  HYB_CHECK(out_context, HYB_ERR_INVALID, "out_context is NULL");
  *out_context = nullptr;
  int count = 0;
  HYB_CUDA(cudaGetDeviceCount(&count));
  HYB_CHECK(device_index >= 0 && device_index < count, HYB_ERR_INVALID,
            "device_index " + std::to_string(device_index) + " out of range (" + std::to_string(count) + " devices)");
  DeviceGuard guard(device_index);
  cudaDeviceProp prop{};
  HYB_CUDA(cudaGetDeviceProperties(&prop, device_index));
  // architecture-specific sm_90a code loads on compute capability 9.0 and nothing else
  HYB_CHECK(prop.major == 9 && prop.minor == 0, HYB_ERR_UNSUPPORTED,
            std::string("libhyrise_b200 is built for sm_90a (H100) only; device is ") + prop.name + " (sm_" +
                std::to_string(prop.major) + std::to_string(prop.minor) + ")");
  auto context = std::make_unique<hyb_context>();
  context->device = device_index;
  context->sm_count = prop.multiProcessorCount;
  // The environment is consulted here and nowhere else (operator calls never touch getenv).
  const std::pair<const char*, const char*> knobs[] = {
      {"HYB_JOIN_TABLE", "join_table"}, {"HYB_JOIN_SPAN", "join_span"},     {"HYB_JOIN_RANK", "join_rank"},
      {"HYB_SCAN_BULK", "scan_bulk"},   {"HYB_AGG_STREAM", "aggregate_stream"},
      {"HYB_AGG_SHAPES", "aggregate_static_shapes"}, {"HYB_TRACE", "trace"}, {"HYB_AGG_STAGES", "aggregate_stages"},
      {"HYB_JOIN_COLOCATED", "join_colocated"}, {"HYB_SCAN_TWO_PASS", "scan_two_pass"}};
  for (const auto& knob : knobs) {
    const char* text = std::getenv(knob.first);
    if (text && !apply_option(context->options, knob.second, text)) {
      return fail(HYB_ERR_INVALID, std::string("bad value for ") + knob.first + ": " + text);
    }
  }
  HYB_CUDA(cudaStreamCreateWithFlags(&context->stream, cudaStreamNonBlocking));
  *out_context = context.release();
  return HYB_OK;
}

int hyb_context_destroy(hyb_context* context) {
  if (!context) return HYB_OK;
  {
    DeviceGuard guard(context->device);
    cudaStreamSynchronize(context->stream);
    context->peer_groups.clear();
    context->pos_lists.clear();
    context->join_results.clear();
    context->aggregate_results.clear();
    context->tables.clear();
    context->block_sets.clear();
    device_cache_destroy(context);
    if (context->timing.op_begin) {
      cudaEventDestroy(context->timing.op_begin);
      cudaEventDestroy(context->timing.op_end);
      for (int span = 0; span < OperatorTiming::kMaxKernelSpans; ++span) {
        cudaEventDestroy(context->timing.kernel_begin[span]);
        cudaEventDestroy(context->timing.kernel_end[span]);
      }
      cudaEventDestroy(context->timing.count_ready);
      cudaFreeHost(context->timing.h_output_count);
    }
    cudaStreamSynchronize(context->stream);
    cudaStreamDestroy(context->stream);
  }
  delete context;
  return HYB_OK;
}

int hyb_context_synchronize(hyb_context* context) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  DeviceGuard guard(context->device);
  HYB_CUDA(cudaStreamSynchronize(context->stream));
  return HYB_OK;
}

int hyb_context_stream(hyb_context* context, void** out_stream) {
  HYB_CHECK(context && out_stream, HYB_ERR_INVALID, "NULL argument");
  *out_stream = static_cast<void*>(context->stream);
  return HYB_OK;
}

int hyb_host_alloc(size_t bytes, void** out_ptr) {
  HYB_CHECK(out_ptr, HYB_ERR_INVALID, "out_ptr is NULL");
  *out_ptr = nullptr;
  HYB_CUDA(cudaHostAlloc(out_ptr, bytes == 0 ? 16 : bytes, cudaHostAllocPortable));
  return HYB_OK;
}

int hyb_host_free(void* ptr) {
  if (ptr) HYB_CUDA(cudaFreeHost(ptr));
  return HYB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// C-ABI: device column pool
// ---------------------------------------------------------------------------------------------------------------------
static int validate_segment(const hyb_segment_desc& desc, uint32_t chunk, uint32_t column) {
  const std::string where = " (chunk " + std::to_string(chunk) + ", column " + std::to_string(column) + ")";
  HYB_CHECK(desc.data_type >= HYB_TYPE_INT32 && desc.data_type <= HYB_TYPE_STRING, HYB_ERR_INVALID,
            "unknown data_type" + where);
  switch (desc.encoding) {
    case HYB_ENC_UNENCODED:
      HYB_CHECK(desc.data_type != HYB_TYPE_STRING, HYB_ERR_UNSUPPORTED,
                "unencoded string segments stay on the CPU" + where);
      HYB_CHECK(desc.values || desc.row_count == 0, HYB_ERR_INVALID, "ValueSegment without values" + where);
      break;
    case HYB_ENC_DICTIONARY:
      HYB_CHECK(desc.attribute_vector || desc.row_count == 0, HYB_ERR_INVALID,
                "DictionarySegment without attribute vector" + where);
      HYB_CHECK(desc.data_type == HYB_TYPE_STRING || desc.values || desc.dictionary_size == 0, HYB_ERR_INVALID,
                "numeric DictionarySegment without dictionary" + where);
      HYB_CHECK(desc.vector_type >= HYB_VEC_FIXED_1B && desc.vector_type <= HYB_VEC_BITPACKED, HYB_ERR_INVALID,
                "bad vector_type" + where);
      break;
    case HYB_ENC_FRAME_OF_REFERENCE:
      HYB_CHECK(desc.data_type == HYB_TYPE_INT32, HYB_ERR_INVALID, "FrameOfReference is int32 only" + where);
      HYB_CHECK((desc.values && desc.attribute_vector) || desc.row_count == 0, HYB_ERR_INVALID,
                "FrameOfReferenceSegment without minima/offsets" + where);
      HYB_CHECK(desc.vector_type >= HYB_VEC_FIXED_1B && desc.vector_type <= HYB_VEC_BITPACKED, HYB_ERR_INVALID,
                "bad vector_type" + where);
      break;
    default:
      return fail(HYB_ERR_UNSUPPORTED, "encoding " + std::to_string(desc.encoding) + " is not on the GPU path" + where);
  }
  if (desc.vector_type == HYB_VEC_BITPACKED) {
    HYB_CHECK(desc.bit_width >= 1 && desc.bit_width <= 32, HYB_ERR_INVALID, "bit_width out of range" + where);
  }
  return HYB_OK;
}

static int upload_buffer(hyb_context* context, Table* table, const void* host, size_t bytes, const void** out_device) {
  *out_device = nullptr;
  if (host == nullptr) return HYB_OK;
  if (table->adopting_device_buffers) {
    *out_device = host;  // hyb_table_append_chunk_device: already a device pointer, borrowed
    return HYB_OK;
  }
  if (table->block_set) {
    // arena upload: the buffer already is on the device inside its block's copy
    const void* resident = table->block_set->translate(host, bytes);
    if (resident) {
      *out_device = resident;
      return HYB_OK;
    }
  }
  void* device = table->arena.alloc(bytes);
  HYB_CHECK(device, HYB_ERR_OOM, "device column pool: out of memory allocating " + std::to_string(bytes) + " bytes");
  if (bytes) HYB_CUDA(cudaMemcpyAsync(device, host, bytes, cudaMemcpyHostToDevice, context->stream));
  *out_device = device;
  return HYB_OK;
}

static int append_chunk_locked(hyb_context* context, Table* table, const hyb_segment_desc* segments) {
  const uint32_t chunk = table->chunk_count();
  const uint32_t rows = table->column_count ? segments[0].row_count : 0;
  std::vector<DevSegment> staged(table->column_count);
  for (uint32_t column = 0; column < table->column_count; ++column) {
    const auto& desc = segments[column];
    HYB_TRY(validate_segment(desc, chunk, column));
    HYB_CHECK(desc.row_count == rows, HYB_ERR_INVALID, "segments of one chunk must have equal row counts");
    if (chunk == 0) {
      table->column_types[column] = desc.data_type;
    } else {
      HYB_CHECK(table->column_types[column] == desc.data_type, HYB_ERR_INVALID,
                "column " + std::to_string(column) + " changes data type between chunks");
    }
    DevSegment dev{};
    dev.row_count = rows;
    dev.dict_size = desc.dictionary_size;
    dev.encoding = static_cast<uint8_t>(desc.encoding);
    dev.data_type = static_cast<uint8_t>(desc.data_type);
    dev.vector_type = static_cast<uint8_t>(desc.encoding == HYB_ENC_UNENCODED ? HYB_VEC_NONE : desc.vector_type);
    dev.bit_width = static_cast<uint8_t>(desc.vector_type == HYB_VEC_BITPACKED ? desc.bit_width : 0);
    const size_t element = data_type_size(desc.data_type);
    switch (desc.encoding) {
      case HYB_ENC_UNENCODED:
        HYB_TRY(upload_buffer(context, table, desc.values, element * rows, &dev.values));
        break;
      case HYB_ENC_DICTIONARY:
        if (desc.data_type != HYB_TYPE_STRING) {
          HYB_TRY(upload_buffer(context, table, desc.values, element * desc.dictionary_size, &dev.values));
        }
        HYB_TRY(upload_buffer(context, table, desc.attribute_vector, vector_bytes(desc.vector_type, desc.bit_width, rows),
                              &dev.av));
        if (desc.dictionary_codes) {
          const void* codes = nullptr;
          HYB_TRY(upload_buffer(context, table, desc.dictionary_codes, sizeof(uint64_t) * desc.dictionary_size, &codes));
          dev.dict_codes = static_cast<const uint64_t*>(codes);
        }
        break;
      case HYB_ENC_FRAME_OF_REFERENCE: {
        const size_t blocks = (size_t{rows} + HYB_FOR_BLOCK_SIZE - 1) / HYB_FOR_BLOCK_SIZE;
        HYB_TRY(upload_buffer(context, table, desc.values, sizeof(int32_t) * blocks, &dev.values));
        HYB_TRY(upload_buffer(context, table, desc.attribute_vector, vector_bytes(desc.vector_type, desc.bit_width, rows),
                              &dev.av));
        break;
      }
    }
    if (desc.nulls && desc.encoding != HYB_ENC_DICTIONARY) {
      const void* nulls = nullptr;
      HYB_TRY(upload_buffer(context, table, desc.nulls, rows, &nulls));
      dev.nulls = static_cast<const uint8_t*>(nulls);
    }
    staged[column] = dev;
  }
  table->segments.insert(table->segments.end(), staged.begin(), staged.end());
  if (chunk > 0 && table->chunk_rows.back() != table->chunk_rows.front()) table->uniform_chunks = false;
  if (chunk > 0 && rows > table->chunk_rows.front()) table->uniform_chunks = false;
  table->chunk_rows.push_back(rows);
  table->chunk_row_start.push_back(table->chunk_row_start.back() + rows);
  table->max_chunk_rows = std::max(table->max_chunk_rows, rows);
  table->dirty = true;
  return HYB_OK;
}

int hyb_table_create(hyb_context* context, uint32_t column_count, hyb_table_t* out_table) {
  HYB_CHECK(context && out_table, HYB_ERR_INVALID, "NULL argument");
  HYB_CHECK(column_count > 0, HYB_ERR_INVALID, "a table needs at least one column");
  std::lock_guard<std::mutex> lock(context->mutex);
  auto table = std::make_unique<Table>();
  table->arena.owner = context;
  table->owner = context;
  table->column_count = column_count;
  table->column_types.assign(column_count, -1);
  table->chunk_row_start.push_back(0);
  const auto handle = context->next_handle++;
  context->tables.emplace(handle, std::move(table));
  *out_table = handle;
  return HYB_OK;
}

int hyb_table_append_chunk(hyb_context* context, hyb_table_t handle, const hyb_segment_desc* segments) {
  HYB_CHECK(context && segments, HYB_ERR_INVALID, "NULL argument");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* table = find_table(context, handle);
  HYB_CHECK(table, HYB_ERR_NOT_FOUND, "unknown table handle");
  const size_t first_segment = table->segments.size();
  HYB_TRY(append_chunk_locked(context, table, segments));
  // The source buffers are borrowed only for the duration of the call (probe_null_flags synchronises the stream).
  HYB_TRY(probe_null_flags(context, table, first_segment));
  HYB_CUDA(cudaStreamSynchronize(context->stream));
  return HYB_OK;
}

int hyb_table_append_chunk_device(hyb_context* context, hyb_table_t handle, const hyb_segment_desc* segments) {
  HYB_CHECK(context && segments, HYB_ERR_INVALID, "NULL argument");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* table = find_table(context, handle);
  HYB_CHECK(table, HYB_ERR_NOT_FOUND, "unknown table handle");
  const size_t first_segment = table->segments.size();
  table->adopting_device_buffers = true;
  const int status = append_chunk_locked(context, table, segments);
  table->adopting_device_buffers = false;
  HYB_TRY(status);
  HYB_TRY(probe_null_flags(context, table, first_segment));
  return HYB_OK;
}

int hyb_table_upload(hyb_context* context, const hyb_table_view* view, hyb_table_t* out_table) {
  HYB_CHECK(context && view && out_table, HYB_ERR_INVALID, "NULL argument");
  HYB_CHECK(view->column_count > 0, HYB_ERR_INVALID, "a table needs at least one column");
  HYB_CHECK(view->segments || view->chunk_count == 0, HYB_ERR_INVALID, "view->segments is NULL");
  HYB_TRY(hyb_table_create(context, view->column_count, out_table));
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* table = find_table(context, *out_table);
  int status = HYB_OK;
  for (uint32_t chunk = 0; chunk < view->chunk_count && status == HYB_OK; ++chunk) {
    status = append_chunk_locked(context, table, view->segments + size_t{chunk} * view->column_count);
  }
  if (status == HYB_OK) status = probe_null_flags(context, table, 0);
  if (status == HYB_OK) {
    cudaError_t error = cudaStreamSynchronize(context->stream);
    if (error != cudaSuccess) status = fail(HYB_ERR_CUDA, std::string("upload: ") + cudaGetErrorString(error));
  }
  if (status != HYB_OK) {
    cudaStreamSynchronize(context->stream);
    context->tables.erase(*out_table);
    *out_table = 0;
  }
  return status;
}

int hyb_blocks_upload(hyb_context* context, const hyb_host_block* blocks, uint32_t block_count,
                      hyb_block_set_t* out_block_set) {
  HYB_CHECK(context && out_block_set && (blocks || block_count == 0), HYB_ERR_INVALID, "NULL argument");
  *out_block_set = 0;
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto set = std::make_shared<BlockSet>();
  set->owner = context;
  for (uint32_t index = 0; index < block_count; ++index) {
    HYB_CHECK(blocks[index].base, HYB_ERR_INVALID, "block base is NULL");
    void* device = nullptr;
    HYB_TRY(device_alloc(context, blocks[index].bytes + Arena::kTailPad, &device));
    set->blocks.push_back({static_cast<const char*>(blocks[index].base), blocks[index].bytes, static_cast<char*>(device)});
    HYB_CUDA(cudaMemcpyAsync(device, blocks[index].base, blocks[index].bytes, cudaMemcpyHostToDevice, context->stream));
  }
  HYB_CUDA(cudaStreamSynchronize(context->stream));  // the blocks are borrowed for the duration of the call
  const auto handle = context->next_handle++;
  context->block_sets.emplace(handle, std::move(set));
  *out_block_set = handle;
  return HYB_OK;
}

int hyb_blocks_free(hyb_context* context, hyb_block_set_t handle) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto it = context->block_sets.find(handle);
  HYB_CHECK(it != context->block_sets.end(), HYB_ERR_NOT_FOUND, "unknown block set handle");
  HYB_CUDA(cudaStreamSynchronize(context->stream));
  context->block_sets.erase(it);  // tables created from it keep the device memory alive until they are dropped
  return HYB_OK;
}

int hyb_table_upload_from_blocks(hyb_context* context, const hyb_table_view* view, hyb_block_set_t block_set,
                                 hyb_table_t* out_table) {
  HYB_CHECK(context && view && out_table, HYB_ERR_INVALID, "NULL argument");
  HYB_CHECK(view->column_count > 0, HYB_ERR_INVALID, "a table needs at least one column");
  HYB_CHECK(view->segments || view->chunk_count == 0, HYB_ERR_INVALID, "view->segments is NULL");
  HYB_TRY(hyb_table_create(context, view->column_count, out_table));
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto set = context->block_sets.find(block_set);
  if (set == context->block_sets.end()) {
    context->tables.erase(*out_table);
    *out_table = 0;
    return fail(HYB_ERR_NOT_FOUND, "unknown block set handle");
  }
  auto* table = find_table(context, *out_table);
  table->block_set = set->second;
  int status = HYB_OK;
  for (uint32_t chunk = 0; chunk < view->chunk_count && status == HYB_OK; ++chunk) {
    status = append_chunk_locked(context, table, view->segments + size_t{chunk} * view->column_count);
  }
  if (status == HYB_OK) status = probe_null_flags(context, table, 0);
  if (status == HYB_OK) {
    cudaError_t error = cudaStreamSynchronize(context->stream);
    if (error != cudaSuccess) status = fail(HYB_ERR_CUDA, std::string("upload: ") + cudaGetErrorString(error));
  }
  if (status != HYB_OK) {
    cudaStreamSynchronize(context->stream);
    context->tables.erase(*out_table);
    *out_table = 0;
  }
  return status;
}

int hyb_table_drop(hyb_context* context, hyb_table_t handle) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto it = context->tables.find(handle);
  HYB_CHECK(it != context->tables.end(), HYB_ERR_NOT_FOUND, "unknown table handle");
  HYB_CUDA(cudaStreamSynchronize(context->stream));
  context->tables.erase(it);
  return HYB_OK;
}

int hyb_table_info(hyb_context* context, hyb_table_t handle, uint32_t* out_chunk_count, uint32_t* out_column_count,
                   uint64_t* out_row_count, uint64_t* out_device_bytes) {
  HYB_CHECK(context, HYB_ERR_INVALID, "context is NULL");
  std::lock_guard<std::mutex> lock(context->mutex);
  auto* table = find_table(context, handle);
  HYB_CHECK(table, HYB_ERR_NOT_FOUND, "unknown table handle");
  if (out_chunk_count) *out_chunk_count = table->chunk_count();
  if (out_column_count) *out_column_count = table->column_count;
  if (out_row_count) *out_row_count = table->row_count();
  if (out_device_bytes) *out_device_bytes = table->arena.bytes_used();
  return HYB_OK;
}

int hyb_last_operator_stats(hyb_context* context, hyb_operator_stats* out_stats) {
  HYB_CHECK(context && out_stats, HYB_ERR_INVALID, "NULL argument");
  DeviceGuard guard(context->device);
  std::lock_guard<std::mutex> lock(context->mutex);
  auto& timing = context->timing;
  HYB_CHECK(timing.valid, HYB_ERR_INVALID, "no operator has run on this context yet");
  HYB_CUDA(cudaEventSynchronize(timing.op_end));
  float op_ms = 0.f, kernel_ms = 0.f;
  HYB_CUDA(cudaEventElapsedTime(&op_ms, timing.op_begin, timing.op_end));
  for (int span = 0; span < timing.kernel_spans; ++span) {
    float span_ms = 0.f;
    HYB_CUDA(cudaEventElapsedTime(&span_ms, timing.kernel_begin[span], timing.kernel_end[span]));
    kernel_ms += span_ms;
  }
  timing.stats.device_ms = op_ms;
  timing.stats.dominant_kernel_ms = kernel_ms;
  if (timing.d_output_count) {
    HYB_CUDA(cudaEventSynchronize(timing.count_ready));
    uint64_t count = *timing.h_output_count;
    if (count == ~uint64_t{0}) count = 0;
    timing.stats.output_rows = count;
    timing.stats.algorithmic_bytes += count * timing.output_bytes_each;
    timing.d_output_count = nullptr;
  }
  *out_stats = timing.stats;
  return HYB_OK;
}

}  // extern "C"
