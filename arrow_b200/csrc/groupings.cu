// groupings.cu -- group-major order and the list-valued hash aggregates.
//
// Replaces:
//   Grouper::MakeGroupings / ApplyGroupings     compute/row/grouper.h:141-194, row/grouper.cc:975-1025
//   GroupedListImpl (hash_list)                 compute/kernels/hash_aggregate.cc:1858-2047
//   GroupedDistinctImpl (hash_distinct)         compute/kernels/hash_aggregate.cc:1400-1539
// Semantics kept: groupings entry g = the row numbers whose id is g, in row order; groups without rows are empty lists;
// null ids are Invalid.  hash_list keeps nulls as elements, in consume order then merge order; hash_distinct lists the
// (value, group) pairs CountOptions::mode admits in the pair Grouper's first-occurrence order.  List slots are never null.
//
// Design:
//   make_groupings : one stable radix sort of the ids carrying row numbers (radix_passes, sort_indices.cu): the ids are
//                    the keys as they are, the first executed pass makes row numbers from positions, only the digits
//                    that vary are sorted (1 pass for <= 256 groups, 3 for 10M) and the last pass writes int32 rows plus
//                    the sorted ids.  Offsets come from the run boundaries of the sorted ids -- where sorted[i] differs
//                    from sorted[i-1], offsets[sorted[i-1]+1 .. sorted[i]] = i -- coalesced, no atomics, no scan.  A
//                    boundary fills at most kGapInline empty groups; when sparse ids leave a longer gap, every offset is
//                    found by binary search instead (log2 n reads per group).  The largest id is sorted[n-1]: an id >=
//                    num_groups is found there and reported with the same one read-back.
//   hash_list      : consume appends values (fixed width: a copy; bool and validity: bits at any bit offset; strings:
//                    rebased offsets + their bytes) and ids to amortised growable device buffers; finalize =
//                    make_groupings + b2_take of the values through the rows.
//   hash_distinct  : hash_count_distinct's pair Grouper; finalize keeps the pairs the mode admits with one b2_filter, then
//                    groups them as hash_list does.
#include "bitmap.h"
#include "groupings.h"

namespace b2 {

// A run boundary fills at most this many empty groups itself; longer gaps (sparse ids) are left to the binary search below,
// so no thread's work grows with num_groups
constexpr int64_t kGapInline = 64;

// offsets[0 .. num_groups] of the groups in `sorted` (ascending ids, n >= 1).  flags[0] = 1 when the largest id is out of
// range (offsets are then only written inside [0, num_groups]); flags[1] = 1 when a gap longer than kGapInline was skipped.
__global__ void __launch_bounds__(kBlock) groupings_offsets_kernel(const uint32_t* __restrict__ sorted, int64_t n,
                                                                   int64_t num_groups, int32_t* __restrict__ offsets,
                                                                   int64_t* flags) {
  const int64_t tid = blockIdx.x * (int64_t)kBlock + threadIdx.x, stride = (int64_t)gridDim.x * kBlock;
  const int64_t first = sorted[0], last = sorted[n - 1];
  if (tid == 0 && last >= num_groups) flags[0] = 1;
  // groups before the first id start at 0, groups after the last end at n: the whole grid fills them (they may be long)
  for (int64_t g = tid; g <= first && g <= num_groups; g += stride) offsets[g] = 0;
  for (int64_t g = last + 1 + tid; g <= num_groups; g += stride) offsets[g] = static_cast<int32_t>(n);
  for (int64_t i = 1 + tid; i < n; i += stride) {
    const int64_t prev = __ldcs(sorted + i - 1), cur = __ldcs(sorted + i);
    const int64_t hi = cur < num_groups ? cur : num_groups;
    if (hi - prev > kGapInline) {
      flags[1] = 1;
      continue;
    }
    for (int64_t g = prev + 1; g <= hi; ++g) offsets[g] = static_cast<int32_t>(i);
  }
}

// offsets[g] = #ids < g by binary search, one thread per group: the sparse case, where run boundaries are far apart
__global__ void __launch_bounds__(kBlock) groupings_search_kernel(const uint32_t* __restrict__ sorted, int64_t n,
                                                                  int64_t num_groups, int32_t* __restrict__ offsets) {
  for (int64_t g = blockIdx.x * (int64_t)kBlock + threadIdx.x; g <= num_groups; g += (int64_t)gridDim.x * kBlock) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if ((int64_t)__ldg(sorted + mid) < g) lo = mid + 1;
      else hi = mid;
    }
    offsets[g] = static_cast<int32_t>(lo);
  }
}

// dst bits [dst_off, dst_off + n) = logical bits [0, n) of src; other bits of dst are kept.  One thread per 32-bit dst
// word, so appends at any bit offset need no atomics.
__global__ void __launch_bounds__(kBlock) append_bits_kernel(uint32_t* __restrict__ dst, int64_t dst_off, BitmapReader src,
                                                             int64_t n) {
  const int64_t w0 = dst_off >> 5, w1 = (dst_off + n - 1) >> 5;
  for (int64_t w = w0 + blockIdx.x * (int64_t)kBlock + threadIdx.x; w <= w1; w += (int64_t)gridDim.x * kBlock) {
    const int64_t q = (w << 5) - dst_off;  // logical src bit that lands on bit 0 of this word (negative in the first word)
    const int64_t qs = q < 0 ? 0 : q;
    const int64_t i = qs >> 6;
    const int sh = static_cast<int>(qs & 63);
    uint64_t bits = src.word(i) >> sh;
    if (sh) bits |= src.word(i + 1) << (64 - sh);
    uint32_t v = static_cast<uint32_t>(bits);
    uint64_t mask = 0xffffffffull;
    if (q < 0) {
      v <<= -q;
      mask = (mask << -q) & 0xffffffffull;
    }
    const int64_t end = dst_off + n - (w << 5);  // bits of this word inside the range
    if (end < 32) mask &= (1ull << end) - 1ull;
    const uint32_t m = static_cast<uint32_t>(mask);
    dst[w] = m == 0xffffffffu ? v : ((dst[w] & ~m) | (v & m));
  }
}

// dst[i + 1] = base + src[i + 1] - src[0] for i < n (dst[0] was written by the previous append)
template <typename O>
__global__ void __launch_bounds__(kBlock) rebase_offsets_kernel(O* __restrict__ dst, const O* __restrict__ src, int64_t n,
                                                                int64_t base) {
  const O start = src[0];
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock)
    dst[i + 1] = static_cast<O>(base + static_cast<int64_t>(src[i + 1] - start));
}

// Groupings of n ids (no nulls) into freshly allocated offsets / rows buffers
static int make_groupings(B2Context* ctx, const uint32_t* ids, int64_t n, int64_t num_groups, int32_t** out_offsets,
                          int32_t** out_rows, cudaStream_t s) {
  if (n > INT32_MAX)
    return set_error(B2_CAPACITY_ERROR, "MakeGroupings: %lld ids exceed the int32 offsets of a list", (long long)n);
  Temp offsets(ctx, s), rows(ctx, s), sorted(ctx, s);
  B2_RETURN_NOT_OK(offsets.alloc(sizeof(int32_t) * (size_t)(num_groups + 1)));
  B2_RETURN_NOT_OK(rows.alloc(sizeof(int32_t) * (size_t)n));
  if (n == 0) {
    B2_CUDA(cudaMemsetAsync(offsets.ptr, 0, sizeof(int32_t) * (size_t)(num_groups + 1), s));
  } else {
    B2_RETURN_NOT_OK(sorted.alloc(sizeof(uint32_t) * (size_t)n));
    bool ids_sorted = false;
    B2_RETURN_NOT_OK(radix_sort_ids(ctx, ids, n, rows.as<int32_t>(), sorted.as<uint32_t>(), &ids_sorted, s));
    ScalarSlot slot(ctx);
    B2_RETURN_NOT_OK(slot.zero(s));
    const int64_t work = n > num_groups ? n : num_groups + 1;
    const uint32_t* sorted_ids = ids_sorted ? sorted.as<uint32_t>() : ids;
    groupings_offsets_kernel<<<grid_for(work, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(sorted_ids, n, num_groups,
                                                                                    offsets.as<int32_t>(), slot.dev());
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(slot.fetch(s));
    if (!slot.host()[0] && slot.host()[1]) {
      groupings_search_kernel<<<grid_for(num_groups + 1, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(sorted_ids, n, num_groups,
                                                                                               offsets.as<int32_t>());
      B2_LAUNCHED();
    }
    if (slot.host()[0]) return set_error(B2_INDEX_ERROR, "MakeGroupings: a group id is >= num_groups (%lld)", (long long)num_groups);
  }
  *out_offsets = static_cast<int32_t*>(offsets.release());
  *out_rows = static_cast<int32_t*>(rows.release());
  return B2_OK;
}

// ---- hash_list state --------------------------------------------------------------------------------------------------
struct ListAgg {
  B2Context* ctx;
  int32_t type;
  int32_t byte_width = 0;  // fixed_size_binary: set by the first consume
  int64_t num_groups = 0;
  int64_t length = 0, cap = 0;          // rows
  int64_t chars = 0, chars_cap = 0;     // (large_)utf8 / binary bytes
  bool has_nulls = false;
  uint32_t* ids = nullptr;
  void* data = nullptr;                 // values / bit-packed bools / offsets (cap + 1 entries)
  uint32_t* validity = nullptr;         // always kept: bits of every row
  char* bytes = nullptr;

  int64_t row_bytes(int64_t rows) const {  // bytes of the data buffer for `rows` rows
    if (type == B2_BOOL) return bitmap_alloc_bytes(rows);
    if (type_is_binary_like(type)) return (rows + 1) * offset_width(type);
    return rows * (type == B2_FIXED_SIZE_BINARY ? byte_width : type_width(type));
  }
  B2Array values() const {
    B2Array v{};
    v.validity = validity;
    v.data = data;
    v.data2 = bytes;
    v.length = length;
    v.null_count = has_nulls ? -1 : 0;
    v.type = type;
    v.byte_width = byte_width;
    return v;
  }
};

static int regrow(B2Context* ctx, void** p, size_t keep, size_t bytes, cudaStream_t s) {
  void* q;
  B2_RETURN_NOT_OK(ctx->alloc(bytes, &q, s));
  if (keep) B2_CUDA(cudaMemcpyAsync(q, *p, keep, cudaMemcpyDeviceToDevice, s));
  if (*p) ctx->free(*p, s);
  *p = q;
  return B2_OK;
}

static int reserve_rows(ListAgg* l, int64_t need, cudaStream_t s) {
  if (need <= l->cap) return B2_OK;
  int64_t cap = l->cap * 2 > need ? l->cap * 2 : need;
  if (cap < 1024) cap = 1024;
  B2Context* ctx = l->ctx;
  void* ids = l->ids;
  void* validity = l->validity;
  B2_RETURN_NOT_OK(regrow(ctx, &ids, sizeof(uint32_t) * l->length, sizeof(uint32_t) * cap, s));
  l->ids = static_cast<uint32_t*>(ids);
  B2_RETURN_NOT_OK(regrow(ctx, &validity, bitmap_bytes(l->length), bitmap_alloc_bytes(cap), s));
  l->validity = static_cast<uint32_t*>(validity);
  const bool offsets = type_is_binary_like(l->type);
  const int64_t keep = l->cap == 0 ? 0 : l->type == B2_BOOL ? bitmap_bytes(l->length) : l->row_bytes(l->length);
  B2_RETURN_NOT_OK(regrow(ctx, &l->data, keep, l->row_bytes(cap), s));
  if (offsets && l->cap == 0) B2_CUDA(cudaMemsetAsync(l->data, 0, offset_width(l->type), s));  // offsets[0] = 0
  l->cap = cap;
  return B2_OK;
}

static int append_bits(uint32_t* dst, int64_t dst_off, const void* src, int64_t src_off, int64_t n, cudaStream_t s) {
  BitmapReader r(src, src_off, n);
  const int64_t words = ((dst_off + n - 1) >> 5) - (dst_off >> 5) + 1;
  append_bits_kernel<<<grid_for(words, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(dst, dst_off, r, n);
  B2_LAUNCHED();
  return B2_OK;
}

int list_create(B2Context* ctx, int32_t value_type, ListAgg** out) {
  const bool ok = type_width(value_type) > 0 || value_type == B2_BOOL || type_is_binary_like(value_type) ||
                  value_type == B2_FIXED_SIZE_BINARY;
  if (!ok) return set_error(B2_NOT_IMPLEMENTED, "hash_list over value type id %d", value_type);
  ListAgg* l = new ListAgg();
  l->ctx = ctx;
  l->type = value_type;
  *out = l;
  return B2_OK;
}

void list_destroy(ListAgg* l) {
  if (!l) return;
  cudaStream_t s = l->ctx->stream;
  for (void* p : {static_cast<void*>(l->ids), l->data, static_cast<void*>(l->validity), static_cast<void*>(l->bytes)})
    if (p) l->ctx->free(p, s);
  delete l;
}

int list_resize(ListAgg* l, int64_t num_groups) {
  l->num_groups = num_groups;
  return B2_OK;
}

int list_consume(ListAgg* l, const B2Array* values, const B2Array* ids, cudaStream_t s) {
  if (!values) return set_error(B2_INVALID, "hash aggregate needs a value column");
  const int64_t n = ids->length;
  if (values->length != n) return set_error(B2_INVALID, "values and group ids differ in length");
  if (values->type != l->type)
    return set_error(B2_TYPE_ERROR, "hash aggregate was created for type id %d, got %d", l->type, values->type);
  if (l->type == B2_FIXED_SIZE_BINARY) {
    const int w = values->byte_width;
    if (w != 1 && w != 2 && w != 4 && w != 8 && w != 16)
      return set_error(B2_NOT_IMPLEMENTED, "hash_list over fixed_size_binary(%d)", w);
    if (l->byte_width && l->byte_width != w) return set_error(B2_TYPE_ERROR, "fixed_size_binary width changed from %d to %d", l->byte_width, w);
    l->byte_width = w;
  }
  if (n == 0) return B2_OK;
  if (l->length + n > INT32_MAX)
    return set_error(B2_CAPACITY_ERROR, "hash_list: %lld values exceed the int32 offsets of a list", (long long)(l->length + n));
  B2Context* ctx = l->ctx;
  B2_RETURN_NOT_OK(reserve_rows(l, l->length + n, s));
  const int64_t len = l->length;
  B2_CUDA(cudaMemcpyAsync(l->ids + len, static_cast<const uint32_t*>(ids->data) + ids->offset, sizeof(uint32_t) * n,
                          cudaMemcpyDeviceToDevice, s));
  const bool nulls = values->null_count != 0 && values->validity;
  B2_RETURN_NOT_OK(append_bits(l->validity, len, nulls ? values->validity : nullptr, values->offset, n, s));
  l->has_nulls = l->has_nulls || nulls;
  if (l->type == B2_BOOL) {
    B2_RETURN_NOT_OK(append_bits(static_cast<uint32_t*>(l->data), len, values->data, values->offset, n, s));
  } else if (type_is_binary_like(l->type)) {
    // the one host read-back of a consume: where this batch's bytes start and how many there are
    const int ow = offset_width(l->type);
    const char* src = static_cast<const char*>(values->data) + values->offset * ow;
    ScalarSlot slot(ctx);
    B2_RETURN_NOT_OK(slot.zero(s));
    B2_CUDA(cudaMemcpyAsync(slot.dev(), src, ow, cudaMemcpyDeviceToDevice, s));
    B2_CUDA(cudaMemcpyAsync(slot.dev() + 1, src + n * ow, ow, cudaMemcpyDeviceToDevice, s));
    B2_RETURN_NOT_OK(slot.fetch(s));
    int64_t start, end;
    if (ow == 4) {
      start = *reinterpret_cast<volatile int32_t*>(slot.host());
      end = *reinterpret_cast<volatile int32_t*>(slot.host() + 1);
    } else {
      start = slot.host()[0];
      end = slot.host()[1];
    }
    const int64_t nb = end - start;
    if (ow == 4 && l->chars + nb > INT32_MAX)
      return set_error(B2_CAPACITY_ERROR, "hash_list: %lld bytes of string data exceed the int32 offsets of the value type",
                       (long long)(l->chars + nb));
    if (l->chars + nb > l->chars_cap) {
      int64_t cap = l->chars_cap * 2 > l->chars + nb ? l->chars_cap * 2 : l->chars + nb;
      if (cap < 4096) cap = 4096;
      if (ow == 4 && cap > INT32_MAX) cap = INT32_MAX;
      void* b = l->bytes;
      B2_RETURN_NOT_OK(regrow(ctx, &b, l->chars, cap, s));
      l->bytes = static_cast<char*>(b);
      l->chars_cap = cap;
    }
    if (nb) B2_CUDA(cudaMemcpyAsync(l->bytes + l->chars, static_cast<const char*>(values->data2) + start, nb,
                                    cudaMemcpyDeviceToDevice, s));
    const int grid = grid_for(n, kBlock * 4, kSMs * 8);
    if (ow == 4)
      rebase_offsets_kernel<int32_t><<<grid, kBlock, 0, s>>>(static_cast<int32_t*>(l->data) + len,
                                                             reinterpret_cast<const int32_t*>(src), n, l->chars);
    else
      rebase_offsets_kernel<int64_t><<<grid, kBlock, 0, s>>>(static_cast<int64_t*>(l->data) + len,
                                                             reinterpret_cast<const int64_t*>(src), n, l->chars);
    B2_LAUNCHED();
    l->chars += nb;
  } else {
    const int w = l->type == B2_FIXED_SIZE_BINARY ? l->byte_width : type_width(l->type);
    B2_CUDA(cudaMemcpyAsync(static_cast<char*>(l->data) + len * w, static_cast<const char*>(values->data) + values->offset * w,
                            (size_t)n * w, cudaMemcpyDeviceToDevice, s));
  }
  l->length += n;
  return B2_OK;
}

int list_merge(ListAgg* l, const ListAgg* other, const B2Array* group_id_mapping, cudaStream_t s) {
  // the other state's rows, ids mapped, after this state's rows (GroupedListImpl::Merge, hash_aggregate.cc:1912-1946)
  if (other->length == 0) return B2_OK;
  PoolArray mapped(l->ctx, s);
  B2Array oids{};
  oids.data = other->ids;
  oids.length = other->length;
  oids.type = B2_UINT32;
  B2_RETURN_NOT_OK(b2_take(l->ctx, group_id_mapping, &oids, 1, &mapped.a, s));
  const B2Array ov = other->values();
  return list_consume(l, &ov, &mapped.a, s);
}

// offsets (int32, num_groups + 1) + the values gathered through the rows: ApplyGroupings (grouper.cc:975-984)
static int grouped(B2Context* ctx, const B2Array* values, const B2Array* ids, int64_t num_groups, B2Array* out_offsets,
                   B2Array* out_values, cudaStream_t s) {
  int32_t *offsets = nullptr, *rows = nullptr;
  B2_RETURN_NOT_OK(make_groupings(ctx, static_cast<const uint32_t*>(ids->data) + ids->offset, ids->length, num_groups,
                                  &offsets, &rows, s));
  PoolArray off(ctx, s), idx(ctx, s);
  fill_out(&off.a, B2_INT32, num_groups + 1, 0, nullptr, offsets);
  fill_out(&idx.a, B2_INT32, ids->length, 0, nullptr, rows);
  B2_RETURN_NOT_OK(b2_take(ctx, values, &idx.a, /*boundscheck=*/0, out_values, s));
  off.give(out_offsets);
  return B2_OK;
}

int list_finalize(ListAgg* l, B2Array* out_offsets, B2Array* out_values, cudaStream_t s) {
  if (l->type == B2_FIXED_SIZE_BINARY && l->byte_width == 0) {  // no batch seen, so no width: num_groups empty lists
    int32_t *offsets = nullptr, *rows = nullptr;
    B2_RETURN_NOT_OK(make_groupings(l->ctx, nullptr, 0, l->num_groups, &offsets, &rows, s));
    l->ctx->free(rows, s);
    fill_out(out_offsets, B2_INT32, l->num_groups + 1, 0, nullptr, offsets);
    fill_out(out_values, l->type, 0, 0, nullptr, nullptr);
    return B2_OK;
  }
  B2Array ids{};
  ids.data = l->ids;
  ids.length = l->length;
  ids.type = B2_UINT32;
  const B2Array v = l->values();
  return grouped(l->ctx, &v, &ids, l->num_groups, out_offsets, out_values, s);
}

int distinct_finalize(B2Context* ctx, B2Grouper* pairs, int count_mode, int64_t num_groups, B2Array* out_offsets,
                      B2Array* out_values, cudaStream_t s) {
  B2Array u[2] = {};
  B2_RETURN_NOT_OK(b2_grouper_uniques(pairs, u, s));
  PoolArray vals(ctx, s), gids(ctx, s);
  vals.a = u[0];
  gids.a = u[1];
  if (count_mode != 2) {
    // the pair Grouper keeps at most one null per group, so dropping (ONLY_VALID) or keeping only (ONLY_NULL) the null
    // pairs before grouping gives what the reference's rewrite of the finished lists gives (hash_aggregate.cc:1494-1535)
    PoolArray mask(ctx, s), fv(ctx, s), fg(ctx, s);
    B2_RETURN_NOT_OK(b2_validity(ctx, count_mode == 0 ? B2_IS_VALID : B2_IS_NULL, &vals.a, 0, &mask.a, s));
    B2_RETURN_NOT_OK(b2_filter(ctx, &vals.a, &mask.a, 0, &fv.a, s));
    B2_RETURN_NOT_OK(b2_filter(ctx, &gids.a, &mask.a, 0, &fg.a, s));
    vals.take_from(fv);
    gids.take_from(fg);
  }
  return grouped(ctx, &vals.a, &gids.a, num_groups, out_offsets, out_values, s);
}

}  // namespace b2

using namespace b2;

extern "C" int b2_make_groupings(B2Context* ctx, const B2Array* ids, int64_t num_groups, B2Array* out_offsets,
                                 B2Array* out_rows, void* stream) {
  if (!ctx || !ids || !out_offsets || !out_rows) return set_error(B2_INVALID, "b2_make_groupings: null argument");
  if (ids->type != B2_UINT32) return set_error(B2_TYPE_ERROR, "MakeGroupings: ids must be uint32 (type id %d)", ids->type);
  if (ids->length < 0 || ids->offset < 0 || num_groups < 0) return set_error(B2_INVALID, "negative length/offset/num_groups");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  int64_t nulls = ids->validity ? ids->null_count : 0;
  if (nulls < 0) {
    int64_t valid = 0;
    B2_RETURN_NOT_OK(b2_bitmap_count(ctx, ids->validity, ids->offset, ids->length, &valid, s));
    nulls = ids->length - valid;
  }
  if (nulls > 0) return set_error(B2_INVALID, "MakeGroupings with null ids");
  int32_t *offsets = nullptr, *rows = nullptr;
  B2_RETURN_NOT_OK(make_groupings(ctx, static_cast<const uint32_t*>(ids->data) + ids->offset, ids->length, num_groups,
                                  &offsets, &rows, s));
  fill_out(out_offsets, B2_INT32, num_groups + 1, 0, nullptr, offsets);
  fill_out(out_rows, B2_INT32, ids->length, 0, nullptr, rows);
  return B2_OK;
}
