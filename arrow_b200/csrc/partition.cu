// partition.cu -- destination ids for the one exchange step of the multi-GPU hash-aggregate
// and SortIndices (SURVEY.md section 8e; the reference has no distributed path, its per-thread
// analogue is GroupByNode::Merge, acero/groupby_aggregate_node.cc:255-298).
//
//   b2_hash_partition  : id[i] = hash64(key[i]) % n_parts   (null keys -> partition 0); the same
//                        hash64 the Grouper table uses, so one owner sees every duplicate of a key.
//   b2_range_partition : id[i] = #splitters whose ordered key is <= ordered_key(value[i])
//                        (upper bound), in the same total order SortIndices uses (sign-flipped
//                        ints, IEEE total order with -0 == +0, NaN last, bitwise NOT for
//                        Descending); null rows get id = n_splitters + 1 (they do not move).
// Both are streaming HBM-bound passes: read W B/row, write 4 B/row.
#include <type_traits>
#include <vector>

#include "bitmap.h"
#include "hash_table.cuh"

namespace b2 {

__global__ void __launch_bounds__(kBlock) hash_partition_kernel(const void* keys, int width, BitmapReader valid, int64_t n,
                                                                uint32_t n_parts, uint32_t* out) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    uint32_t p = 0;
    if (valid.bit(i)) p = static_cast<uint32_t>(hash64(load_key_bits(keys, width, i)) % n_parts);
    out[i] = p;
  }
}

template <typename T>
__device__ __forceinline__ uint64_t total_order_key(T v, bool descending) {
  uint64_t k;
  if constexpr (std::is_floating_point<T>::value) {
    if (v != v) return ~0ull;  // NaNs after every value in either order (they are "null-like")
    double d = static_cast<double>(v);
    if (d == 0.0) d = 0.0;
    uint64_t b = static_cast<uint64_t>(__double_as_longlong(d));
    k = (b >> 63) ? ~b : (b | 0x8000000000000000ull);
    if (descending) k = ~k;
    return k;
  } else if constexpr (std::is_signed<T>::value) {
    k = static_cast<uint64_t>(static_cast<int64_t>(v)) ^ 0x8000000000000000ull;
  } else {
    k = static_cast<uint64_t>(v);
  }
  return descending ? ~k : k;
}

template <typename T>
__global__ void __launch_bounds__(kBlock) range_partition_kernel(const T* __restrict__ values, BitmapReader valid, int64_t n,
                                                                 const T* __restrict__ splitters, int n_split, bool descending,
                                                                 uint32_t* __restrict__ out) {
  __shared__ uint64_t s_split[64];
  if (threadIdx.x < n_split) s_split[threadIdx.x] = total_order_key<T>(splitters[threadIdx.x], descending);
  __syncthreads();
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    uint32_t p = static_cast<uint32_t>(n_split) + 1;
    if (valid.bit(i)) {
      const uint64_t k = total_order_key<T>(values[i], descending);
      p = 0;
      for (int j = 0; j < n_split; ++j) p += (s_split[j] <= k) ? 1u : 0u;
    }
    out[i] = p;
  }
}

// ---- range split: the sender side of the distributed SortIndices in two streaming passes -------------------------------
// Stable (P+1)-way split of (value, row number) pairs by range id: bin = #splitters <= value in SortIndices' total order,
// null rows in bin P.  Replaces range ids + sort_indices(ids) + two takes + an offset add (five passes over the shard) by
// count -> scan -> scatter; the row numbers leave as uint32 (row_base + i), ready to be the payload of b2_sort_payload.
constexpr int kSplitTile = 2048;
constexpr int kSplitMaxBins = 32;  // P + 1 <= 32 (one bin per lane)

template <typename T>
__device__ __forceinline__ uint32_t range_bin(const T* __restrict__ values, const BitmapReader& valid, int64_t i, const uint64_t* s_split,
                                              int n_split, bool descending) {
  if (!valid.bit(i)) return static_cast<uint32_t>(n_split) + 1;
  const uint64_t k = total_order_key<T>(values[i], descending);
  uint32_t p = 0;
  for (int j = 0; j < n_split; ++j) p += (s_split[j] <= k) ? 1u : 0u;
  return p;
}

// tile_counts[bin * n_tiles + tile] = rows of the tile that fall in `bin` (bin-major: one scan gives absolute positions)
template <typename T>
__global__ void __launch_bounds__(kBlock) range_split_count_kernel(const T* __restrict__ values, BitmapReader valid, int64_t n,
                                                                   const T* __restrict__ splitters, int n_split, bool descending,
                                                                   int64_t n_tiles, int64_t* __restrict__ tile_counts) {
  __shared__ uint64_t s_split[64];
  __shared__ uint32_t s_cnt[kSplitMaxBins];
  if (threadIdx.x < n_split) s_split[threadIdx.x] = total_order_key<T>(splitters[threadIdx.x], descending);
  if (threadIdx.x < kSplitMaxBins) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  const int64_t tile = blockIdx.x;
  const unsigned lane = lane_id();
  uint32_t mine = 0;  // lane b counts bin b
  for (int r = threadIdx.x; r < kSplitTile; r += kBlock) {
    const int64_t i = tile * kSplitTile + r;
    const uint32_t b = i < n ? range_bin<T>(values, valid, i, s_split, n_split, descending) : 0xffffffffu;
    for (int q = 0; q <= n_split + 1; ++q) {
      const unsigned m = __ballot_sync(0xffffffffu, b == (uint32_t)q);
      if ((int)lane == q) mine += __popc(m);
    }
  }
  if ((int)lane <= n_split + 1 && mine) atomicAdd(&s_cnt[lane], mine);
  __syncthreads();
  if ((int)threadIdx.x <= n_split + 1) tile_counts[(int64_t)threadIdx.x * n_tiles + tile] = s_cnt[threadIdx.x];
}

template <typename T>
__global__ void __launch_bounds__(kBlock) range_split_scatter_kernel(const T* __restrict__ values, BitmapReader valid, int64_t n,
                                                                     const T* __restrict__ splitters, int n_split, bool descending,
                                                                     int64_t n_tiles, const int64_t* __restrict__ tile_offsets,
                                                                     uint32_t row_base, T* __restrict__ out_values,
                                                                     uint32_t* __restrict__ out_rows) {
  __shared__ uint64_t s_split[64];
  __shared__ uint32_t s_warp[kWarpsPerBlock][kSplitMaxBins];  // rows of each warp per bin, then exclusive over warps
  if (threadIdx.x < n_split) s_split[threadIdx.x] = total_order_key<T>(splitters[threadIdx.x], descending);
  __syncthreads();
  const int64_t tile = blockIdx.x;
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  constexpr int kRowsPerWarp = kSplitTile / kWarpsPerBlock;  // 256 consecutive rows per warp: rank order = row order
  const int64_t w0 = tile * kSplitTile + (int64_t)warp * kRowsPerWarp;
  const int bins = n_split + 2;
  // pass A: this warp's rows per bin
  uint32_t mine = 0;
  uint32_t b_of[kRowsPerWarp / 32];
#pragma unroll
  for (int it = 0; it < kRowsPerWarp / 32; ++it) {
    const int64_t i = w0 + it * 32 + lane;
    b_of[it] = i < n ? range_bin<T>(values, valid, i, s_split, n_split, descending) : 0xffffffffu;
    for (int q = 0; q < bins; ++q) {
      const unsigned m = __ballot_sync(0xffffffffu, b_of[it] == (uint32_t)q);
      if ((int)lane == q) mine += __popc(m);
    }
  }
  if ((int)lane < kSplitMaxBins) s_warp[warp][lane] = mine;
  __syncthreads();
  if (threadIdx.x < kSplitMaxBins) {  // exclusive over the warps, per bin
    uint32_t run = 0;
    for (int w = 0; w < kWarpsPerBlock; ++w) {
      const uint32_t c = s_warp[w][threadIdx.x];
      s_warp[w][threadIdx.x] = run;
      run += c;
    }
  }
  __syncthreads();
  // pass B: positions.  lane q keeps the running count of bin q inside this warp
  uint32_t running = 0;
#pragma unroll
  for (int it = 0; it < kRowsPerWarp / 32; ++it) {
    const int64_t i = w0 + it * 32 + lane;
    const uint32_t b = b_of[it];
    uint32_t rank = 0, before = 0;
    for (int q = 0; q < bins; ++q) {
      const unsigned m = __ballot_sync(0xffffffffu, b == (uint32_t)q);
      const uint32_t run_q = __shfl_sync(0xffffffffu, running, q);
      if (b == (uint32_t)q) {
        rank = __popc(m & lanemask_lt());
        before = run_q;
      }
      if ((int)lane == q) running += __popc(m);
    }
    if (i < n) {
      const int64_t pos = tile_offsets[(int64_t)b * n_tiles + tile] + s_warp[warp][b] + before + rank;
      out_values[pos] = values[i];
      out_rows[pos] = row_base + static_cast<uint32_t>(i);
    }
  }
}

// counts[b] = #rows with ids[i] == b for b < n_bins (rows with larger ids are counted in `out_of_range`)
__global__ void __launch_bounds__(kBlock) bincount_kernel(const uint32_t* __restrict__ ids, int64_t n, uint32_t n_bins,
                                                          unsigned long long* counts) {
  extern __shared__ uint32_t s_hist[];  // n_bins + 1
  for (uint32_t i = threadIdx.x; i <= n_bins; i += kBlock) s_hist[i] = 0;
  __syncthreads();
  // a block never adds more than 2^31 rows to one bin: its share of the rows is bounded by the grid size
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const uint32_t b = __ldcs(ids + i);
    atomicAdd(&s_hist[b < n_bins ? b : n_bins], 1u);
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i <= n_bins; i += kBlock)
    if (s_hist[i]) atomicAdd(&counts[i], (unsigned long long)s_hist[i]);
}

}  // namespace b2

using namespace b2;

template <typename T>
static int run_range_split(B2Context* ctx, const B2Array* values, const B2Array* splitters, int order, uint32_t row_base, void* out_values,
                           uint32_t* out_rows, int64_t* out_counts, cudaStream_t s) {
  const int64_t n = values->length;
  const int n_split = (int)splitters->length;
  const int bins = n_split + 2;
  const int64_t n_tiles = (n + kSplitTile - 1) / kSplitTile;
  Temp counts(ctx, s), offsets(ctx, s);
  B2_RETURN_NOT_OK(counts.alloc(sizeof(int64_t) * (size_t)(bins * n_tiles)));
  B2_RETURN_NOT_OK(offsets.alloc(sizeof(int64_t) * (size_t)(bins * n_tiles)));
  BitmapReader valid(values->null_count == 0 ? nullptr : values->validity, values->offset, n);
  const T* v = static_cast<const T*>(values->data) + values->offset;
  const T* sp = static_cast<const T*>(splitters->data) + splitters->offset;
  range_split_count_kernel<T><<<(unsigned)n_tiles, kBlock, 0, s>>>(v, valid, n, sp, n_split, order == 1, n_tiles, counts.as<int64_t>());
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(launch_exclusive_scan_i64(counts.as<int64_t>(), (int64_t)bins * n_tiles, offsets.as<int64_t>(), nullptr, s));
  range_split_scatter_kernel<T><<<(unsigned)n_tiles, kBlock, 0, s>>>(v, valid, n, sp, n_split, order == 1, n_tiles, offsets.as<int64_t>(),
                                                                       row_base, static_cast<T*>(out_values), out_rows);
  B2_LAUNCHED();
  // bin sizes = differences of the bins' first offsets
  std::vector<int64_t> first(bins);
  for (int b = 0; b < bins; ++b)
    B2_CUDA(cudaMemcpyAsync(&first[b], offsets.as<int64_t>() + (int64_t)b * n_tiles, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  B2_CUDA(cudaStreamSynchronize(s));
  for (int b = 0; b < bins; ++b) out_counts[b] = (b + 1 < bins ? first[b + 1] : n) - first[b];
  return B2_OK;
}

extern "C" int b2_range_split(B2Context* ctx, const B2Array* values, const B2Array* splitters, int order, uint64_t row_base,
                              B2Array* out_values, B2Array* out_rows, int64_t* out_counts, void* stream) {
  if (!ctx || !values || !splitters || !out_values || !out_rows || !out_counts) return set_error(B2_INVALID, "b2_range_split: null argument");
  if (values->type != splitters->type) return set_error(B2_TYPE_ERROR, "splitters must have the values' type");
  if (splitters->length > kSplitMaxBins - 2) return set_error(B2_INVALID, "at most %d splitters", kSplitMaxBins - 2);
  if (splitters->null_count > 0) return set_error(B2_INVALID, "splitters must not contain nulls");
  if (!type_is_numeric(values->type)) return set_error(B2_NOT_IMPLEMENTED, "b2_range_split: type id %d", values->type);
  const int64_t n = values->length;
  if (row_base + (uint64_t)n >= (1ull << 32)) return set_error(B2_NOT_IMPLEMENTED, "b2_range_split: row numbers must fit 32 bits");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int w = type_width(values->type);
  Temp ov(ctx, s), orows(ctx, s);
  B2_RETURN_NOT_OK(ov.alloc((size_t)n * w));
  B2_RETURN_NOT_OK(orows.alloc(sizeof(uint32_t) * (size_t)n));
  for (int b = 0; b < (int)splitters->length + 2; ++b) out_counts[b] = 0;
  if (n > 0) {
    const uint32_t rb = (uint32_t)row_base;
    B2_RETURN_NOT_OK(visit_type(NumericTypes{}, values->type, [&](auto tag) {
      return run_range_split<decltype(tag)>(ctx, values, splitters, order, rb, ov.ptr, orows.as<uint32_t>(), out_counts, s);
    }));
  }
  fill_out(out_values, values->type, n, 0, nullptr, ov.release());
  fill_out(out_rows, B2_UINT32, n, 0, nullptr, orows.release());
  return B2_OK;
}

extern "C" int b2_bincount(B2Context* ctx, const B2Array* ids, int n_bins, int64_t* out_counts, void* stream) {
  if (!ctx || !ids || !out_counts) return set_error(B2_INVALID, "b2_bincount: null argument");
  if (ids->type != B2_UINT32) return set_error(B2_TYPE_ERROR, "b2_bincount: ids must be uint32 (type id %d)", ids->type);
  if (n_bins < 1 || n_bins > 8192) return set_error(B2_INVALID, "b2_bincount: n_bins must be in [1, 8192]");
  if (ids->null_count > 0) return set_error(B2_INVALID, "b2_bincount: ids must not contain nulls");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = ids->length;
  for (int i = 0; i < n_bins; ++i) out_counts[i] = 0;
  if (n == 0) return B2_OK;
  Temp counts(ctx, s);
  const size_t bytes = sizeof(unsigned long long) * (size_t)(n_bins + 1);
  B2_RETURN_NOT_OK(counts.alloc(bytes));
  B2_CUDA(cudaMemsetAsync(counts.ptr, 0, bytes, s));
  bincount_kernel<<<grid_for(n, kBlock * 16, kSMs * 8), kBlock, sizeof(uint32_t) * (n_bins + 1), s>>>(
      static_cast<const uint32_t*>(ids->data) + ids->offset, n, (uint32_t)n_bins, counts.as<unsigned long long>());
  B2_LAUNCHED();
  std::vector<unsigned long long> host(n_bins + 1);
  B2_CUDA(cudaMemcpyAsync(host.data(), counts.ptr, bytes, cudaMemcpyDeviceToHost, s));
  B2_CUDA(cudaStreamSynchronize(s));
  if (host[n_bins] != 0)
    return set_error(B2_INDEX_ERROR, "b2_bincount: %llu ids are >= n_bins (%d)", host[n_bins], n_bins);
  for (int i = 0; i < n_bins; ++i) out_counts[i] = (int64_t)host[i];
  return B2_OK;
}

extern "C" int b2_hash_partition(B2Context* ctx, const B2Array* keys, int n_parts, B2Array* out_ids, void* stream) {
  if (!ctx || !keys || !out_ids) return set_error(B2_INVALID, "b2_hash_partition: null argument");
  if (n_parts < 1) return set_error(B2_INVALID, "n_parts must be >= 1");
  const int w = type_width(keys->type);
  if (w == 0) return set_error(B2_NOT_IMPLEMENTED, "b2_hash_partition: key type id %d", keys->type);
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = keys->length;
  Temp ids(ctx, s);
  B2_RETURN_NOT_OK(ids.alloc(sizeof(uint32_t) * (size_t)n));
  if (n > 0) {
    BitmapReader valid(keys->null_count == 0 ? nullptr : keys->validity, keys->offset, n);
    hash_partition_kernel<<<grid_for(n, kBlock * 4, kSMs * 16), kBlock, 0, s>>>(
        static_cast<const char*>(keys->data) + keys->offset * w, w, valid, n, (uint32_t)n_parts, ids.as<uint32_t>());
    B2_LAUNCHED();
  }
  fill_out(out_ids, B2_UINT32, n, 0, nullptr, ids.release());
  return B2_OK;
}

template <typename T>
static int run_range(const B2Array* values, const B2Array* splitters, int order, uint32_t* out, cudaStream_t s) {
  const int64_t n = values->length;
  BitmapReader valid(values->null_count == 0 ? nullptr : values->validity, values->offset, n);
  range_partition_kernel<T><<<grid_for(n, kBlock * 4, kSMs * 16), kBlock, 0, s>>>(
      static_cast<const T*>(values->data) + values->offset, valid, n,
      static_cast<const T*>(splitters->data) + splitters->offset, (int)splitters->length, order == 1, out);
  B2_LAUNCHED();
  return B2_OK;
}

extern "C" int b2_range_partition(B2Context* ctx, const B2Array* values, const B2Array* splitters, int order,
                                  B2Array* out_ids, void* stream) {
  if (!ctx || !values || !splitters || !out_ids) return set_error(B2_INVALID, "b2_range_partition: null argument");
  if (values->type != splitters->type) return set_error(B2_TYPE_ERROR, "splitters must have the values' type");
  if (splitters->length > 63) return set_error(B2_INVALID, "at most 63 splitters");
  if (splitters->null_count > 0) return set_error(B2_INVALID, "splitters must not contain nulls");
  if (!type_is_numeric(values->type)) return set_error(B2_NOT_IMPLEMENTED, "b2_range_partition: type id %d", values->type);
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = values->length;
  Temp ids(ctx, s);
  B2_RETURN_NOT_OK(ids.alloc(sizeof(uint32_t) * (size_t)n));
  if (n > 0) {
    uint32_t* o = ids.as<uint32_t>();
    B2_RETURN_NOT_OK(visit_type(NumericTypes{}, values->type,
                                [&](auto tag) { return run_range<decltype(tag)>(values, splitters, order, o, s); }));
  }
  fill_out(out_ids, B2_UINT32, n, 0, nullptr, ids.release());
  return B2_OK;
}
