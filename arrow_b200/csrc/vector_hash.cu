// vector_hash.cu -- unique / value_counts / dictionary_encode over one fixed-width or utf8 / binary column.
//
// Replaces (SURVEY section 8f rank 1):
//   UniqueAction / ValueCountsAction / DictEncodeAction + RegularHashKernel
//                                     kernels/vector_hash.cc:65-235,236-470
//   "unique" / "value_counts" / "dictionary_encode" registration   :782-830
//   DictionaryEncodeOptions{MASK, ENCODE}          compute/api_vector.h:66-82
// Semantics kept: the dictionary (= the uniques) lists the distinct values in FIRST-OCCURRENCE
// order; unique and value_counts treat null as a value (ShouldEncodeNulls() == true), so a
// null entry sits where the first null row was; dictionary_encode emits int32 indices and
// with MASK (the default) null rows become null indices and the dictionary holds no null,
// with ENCODE null rows point at a null dictionary entry; counts are int64, never null.
// Values group by BYTES like the Grouper (-0.0 != +0.0, NaNs by payload); the reference's
// memo table compares floats with == after a bit-pattern hash, i.e. the same except for
// hash-colliding NaN payloads / signed zeros.
//
// Design: the Grouper (grouper.cu) already yields dense first-occurrence ids and the
// uniques in id order, so this file only adds the id -> int32 index remap (skipping the null
// group for MASK) and a count-per-id pass (global atomics, L2-resident for dictionaries up
// to ~10M entries); the MASK dictionary is the uniques filtered by their own validity.
#include "bitmap.h"
#include "selection.cuh"

namespace b2 {

// index of the (single) zero bit of a validity bitmap = the id of the null group
__global__ void __launch_bounds__(kBlock) find_null_entry_kernel(const uint32_t* __restrict__ bits, int64_t n,
                                                                 unsigned long long* out) {
  const int64_t nw = (n + 31) >> 5;
  for (int64_t w = blockIdx.x * (int64_t)kBlock + threadIdx.x; w < nw; w += (int64_t)gridDim.x * kBlock) {
    uint32_t inv = ~bits[w];
    if (((w + 1) << 5) > n) inv &= (1u << (n & 31)) - 1u;  // ignore the padding of the last word
    if (inv) atomicMin(out, static_cast<unsigned long long>((w << 5) + __ffs(inv) - 1));
  }
}

// ids -> int32 dictionary indices; with skip_null the null group's id is removed from the numbering
__global__ void __launch_bounds__(kBlock) remap_ids_kernel(const uint32_t* __restrict__ ids, int64_t n,
                                                           uint32_t null_id, bool skip_null, int32_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const uint32_t g = __ldcs(ids + i);
    int32_t v = static_cast<int32_t>(g);
    if (skip_null) v = g == null_id ? 0 : static_cast<int32_t>(g > null_id ? g - 1 : g);
    out[i] = v;
  }
}

// counts[id] += 1 per row.  Lanes of a warp holding the same id are merged first (MATCH.ANY, one
// atomic per distinct id per warp): a hot value would otherwise serialise tens of millions of atomics
// on one L2 address.  The null entry -- the usual hot value, 10 % of the rows
// even after the merge still means one atomic per warp on ONE address -- is counted in registers
// and added once per warp at the end.
// MERGE = false (large dictionaries): equal ids inside one warp are rare, so the MATCH.ANY (bench_micro/smem_probe.cu
// measures its cost) costs more than the atomics it saves; every row is one RED into the L2-resident counts.
template <bool MERGE>
__global__ void __launch_bounds__(kBlock) count_ids_kernel(const uint32_t* __restrict__ ids, int64_t n,
                                                           uint32_t null_id, bool has_null,
                                                           unsigned long long* counts) {
  const unsigned lane = lane_id();
  const int64_t stride = (int64_t)gridDim.x * kBlock;
  unsigned long long nulls = 0;
  for (int64_t base = blockIdx.x * (int64_t)kBlock + (threadIdx.x & ~31u); base < n; base += stride) {
    const int64_t i = base + lane;
    bool in = i < n;
    const uint32_t g = in ? __ldcs(ids + i) : 0u;
    if (has_null) {
      const bool is_null = in && g == null_id;
      nulls += __popc(__ballot_sync(0xffffffffu, is_null));
      in = in && !is_null;
    }
    const unsigned live = __ballot_sync(0xffffffffu, in);
    if (in) {
      if (MERGE) {
        const unsigned peers = __match_any_sync(live, g);
        if ((peers & lanemask_lt()) == 0) atomicAdd(&counts[g], static_cast<unsigned long long>(__popc(peers)));
      } else {
        atomicAdd(&counts[g], 1ull);
      }
    }
  }
  if (has_null && lane == 0 && nulls) atomicAdd(&counts[null_id], nulls);
}

}  // namespace b2

using namespace b2;

namespace {
struct GrouperGuard {
  B2Grouper* g = nullptr;
  ~GrouperGuard() {
    if (g) b2_grouper_destroy(g);
  }
};
}  // namespace

extern "C" int b2_vector_hash(B2Context* ctx, const B2Array* values, int null_encoding, B2Array* out_indices,
                              B2Array* out_dictionary, B2Array* out_counts, void* stream) {
  if (!ctx || !values || !out_dictionary) return set_error(B2_INVALID, "b2_vector_hash: null argument");
  if (null_encoding != 0 && null_encoding != 1) return set_error(B2_INVALID, "b2_vector_hash: null_encoding must be 0 (MASK) or 1 (ENCODE)");
  if (type_width(values->type) == 0 && !type_is_binary_like(values->type))
    return set_error(B2_NOT_IMPLEMENTED, "unique/value_counts/dictionary_encode: type id %d is neither fixed-width nor utf8 / binary", values->type);
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->pick(stream);
  const int64_t n = values->length;
  const bool mask_nulls = null_encoding == 0;

  GrouperGuard gg;
  const int32_t kt = values->type;
  B2_RETURN_NOT_OK(b2_grouper_create(ctx, &kt, 1, &gg.g));
  PoolArray ids(ctx, s), uniq(ctx, s);
  B2_RETURN_NOT_OK(b2_grouper_consume(gg.g, values, &ids.a, s));
  B2_RETURN_NOT_OK(b2_grouper_uniques(gg.g, &uniq.a, s));
  uint32_t n_groups = 0;
  B2_RETURN_NOT_OK(b2_grouper_num_groups(gg.g, &n_groups));
  if (n_groups > 0x7fffffffu) return set_error(B2_CAPACITY_ERROR, "dictionary of %u entries does not fit int32 indices", n_groups);

  // id of the null group, if there is one
  uint32_t null_id = 0;
  const bool has_null = uniq.a.null_count > 0;
  if (has_null) {
    ScalarSlot slot(ctx);
    B2_RETURN_NOT_OK(slot.zero(s));
    B2_CUDA(cudaMemsetAsync(slot.dev(), 0xff, sizeof(int64_t), s));
    find_null_entry_kernel<<<grid_for((n_groups + 31) / 32, kBlock, kSMs * 4), kBlock, 0, s>>>(
        static_cast<const uint32_t*>(uniq.a.validity), n_groups, reinterpret_cast<unsigned long long*>(slot.dev()));
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(slot.fetch(s));
    null_id = static_cast<uint32_t>(slot.host()[0]);
  }

  // dictionary first (the only step below that can still fail in a kernel-visible way)
  PoolArray dict(ctx, s);
  if (mask_nulls && has_null) {
    // uniques without the null entry: filter the uniques by their own validity bitmap
    B2Array keep{};
    keep.data = uniq.a.validity;
    keep.length = n_groups;
    keep.type = B2_BOOL;
    B2Array plain = uniq.a;
    plain.validity = nullptr;
    plain.null_count = 0;
    B2_RETURN_NOT_OK(b2_filter(ctx, &plain, &keep, 0, &dict.a, s));
  }

  Temp counts(ctx, s), idx(ctx, s), idx_valid(ctx, s);
  int64_t idx_nulls = 0;
  if (out_counts) {
    B2_RETURN_NOT_OK(counts.alloc(sizeof(int64_t) * (size_t)(n_groups ? n_groups : 1)));
    B2_CUDA(cudaMemsetAsync(counts.ptr, 0, sizeof(int64_t) * (size_t)(n_groups ? n_groups : 1), s));
    if (n > 0) {
      const int cgrid = grid_for(n, kBlock * 4, kSMs * 16);
      const uint32_t* idp = static_cast<const uint32_t*>(ids.a.data);
      if (n_groups >= 65536) count_ids_kernel<false><<<cgrid, kBlock, 0, s>>>(idp, n, null_id, has_null, counts.as<unsigned long long>());
      else count_ids_kernel<true><<<cgrid, kBlock, 0, s>>>(idp, n, null_id, has_null, counts.as<unsigned long long>());
      B2_LAUNCHED();
    }
  }
  if (out_indices) {
    B2_RETURN_NOT_OK(idx.alloc(sizeof(int32_t) * (size_t)(n ? n : 1)));
    if (n > 0) {
      remap_ids_kernel<<<grid_for(n, kBlock * 4, kSMs * 16), kBlock, 0, s>>>(
          static_cast<const uint32_t*>(ids.a.data), n, null_id, mask_nulls && has_null, idx.as<int32_t>());
      B2_LAUNCHED();
    }
    if (mask_nulls && has_null) {  // indices are null exactly where the values were
      void* validity = nullptr;
      B2_RETURN_NOT_OK(make_validity(ctx, values, nullptr, n, &validity, &idx_nulls, s));
      idx_valid.ptr = validity;
    }
  }
  // nothing can fail from here on: hand the buffers over
  if (out_counts) fill_out(out_counts, B2_INT64, n_groups, 0, nullptr, counts.release());
  if (out_indices) fill_out(out_indices, B2_INT32, n, idx_nulls, idx_valid.release(), idx.release());
  ((mask_nulls && has_null) ? dict : uniq).give(out_dictionary);
  return B2_OK;
}
