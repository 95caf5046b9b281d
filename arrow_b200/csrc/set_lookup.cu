// set_lookup.cu -- is_in / index_in: the membership of every row in a value set.
//
// Replaces:
//   SetLookupState::Init / AddArrayValueSet        kernels/scalar_set_lookup.cc:44-129
//   IndexInVisitor / ExecIndexIn                   :271-396
//   IsInVisitor / ExecIsIn                         :398-545
//   SetLookupOptions, GetNullMatchingBehavior      compute/api_scalar.h:279-324, api_scalar.cc:604-612
// Semantics kept: every distinct value maps to the position of its FIRST occurrence in the value set
// (memo_index_to_value_index); a null in the value set is recorded at its first position unless the behaviour is SKIP
// (null_index); numbers compare by bit pattern at their width (UnsignedIntType<sizeof>: -0.0 != +0.0, a NaN matches only
// the same payload), strings by bytes.  Per row:
//   is_in    valid, found -> true; valid, not found -> null if INCONCLUSIVE and null_index != -1, else false;
//            null -> true if MATCH and null_index != -1; false if SKIP or MATCH; null for EMIT_NULL / INCONCLUSIVE
//   index_in valid, found -> first position; not found -> null; null -> null_index if MATCH and != -1, else null
// Data under null slots is zero, as the reference writes it.
//
// Design.  The build runs once per b2_set_lookup_create: the Grouper dedupes the value set and numbers the distinct
// values in first-occurrence order, one kernel takes the first position of every id, and a second lays the distinct
// values out in an open-addressing table at load factor <= 1/2: 8-byte keys (the value's bits, or a string's 64-bit
// hash) followed by int32 payloads (the position, or a string's unique id whose bytes the probe compares).  A boolean
// value set needs no table: three first positions (false, true, null).
// The probe is one streaming pass.  Each warp owns 32-row groups, so the boolean result and the output validity are
// written as whole 32-bit words from one ballot each, without atomics.  A table small enough that two probe blocks still
// share an SM (shared_table_limit) is staged in shared memory once per block (the IN-list case); a larger one is probed
// in global memory, where it stays L2-resident up to a few million entries.
#include <algorithm>
#include <atomic>

#include "common.cuh"
#include "context.h"
#include "hash_table.cuh"

namespace b2 {

constexpr int kProbeBlock = 512;
constexpr int kProbeBlocksPerSM = 2;  // the register budget of __launch_bounds__(kProbeBlock, kProbeBlocksPerSM)
constexpr uint64_t kStringSeed = 0x452821e638d01377ull;
// value kinds of the probe: W > 0 = fixed width W; utf8 / binary by the width of their offsets; boolean
constexpr int kBoolKey = 0, kStr32 = -4, kStr64 = -8;

struct ProbeArgs {
  const void* data;         // fixed width: values at the input's offset; strings: offsets at the input's offset
  const uint8_t* bytes;     // strings: character data
  BitmapReader bits;        // boolean values
  BitmapReader valid;
  int64_t n;
  int64_t n_words;          // 32-bit output words written, padding included
  const unsigned long long* keys;
  const int32_t* vals;
  uint64_t mask;
  int64_t table_bytes;
  int32_t special_pos;      // 8-byte values whose bits are kEmptyKey live outside the table
  const void* u_offs;       // strings: the distinct values ...
  const uint8_t* u_bytes;
  const int32_t* first_pos; // ... and their first positions
  int32_t false_pos, true_pos;
  int32_t null_row_pos;     // the result of a null row when it is a position
  bool miss_valid;          // a valid row that is not found gives a valid result
  bool null_miss_valid;     // a null row with null_row_pos < 0 gives a valid result
  uint32_t* out_bits;       // is_in
  int32_t* out_index;       // index_in
  uint32_t* out_valid;      // NULL: the result has no nulls
  unsigned long long* null_count;
};

__device__ __forceinline__ uint64_t string_key(const uint8_t* p, int64_t len) {
  const uint64_t h = hash_bytes(p, len, kStringSeed);
  return h == kEmptyKey ? kEmptyKey - 1 : h;
}

template <int W>
__device__ __forceinline__ uint64_t load_value_bits(const void* data, int64_t i) {
  if constexpr (W == 1) return ld_stream(static_cast<const uint8_t*>(data) + i);
  if constexpr (W == 2) return ld_stream(static_cast<const uint16_t*>(data) + i);
  if constexpr (W == 4) return ld_stream(static_cast<const uint32_t*>(data) + i);
  if constexpr (W == 8) return ld_stream(static_cast<const unsigned long long*>(data) + i);
  return 0;
}

// position of fixed-width value bits `k`, or -1
__device__ __forceinline__ int32_t find_bits(const unsigned long long* keys, const int32_t* vals, uint64_t mask,
                                             int32_t special_pos, uint64_t k) {
  if (k == kEmptyKey) return special_pos;
  for (uint64_t slot = hash64(k) & mask;; slot = (slot + 1) & mask) {
    const uint64_t cur = keys[slot];
    if (cur == k) return vals[slot];
    if (cur == kEmptyKey) return -1;
  }
}

// position of string row i, or -1: the hash picks the candidates, the bytes decide
template <typename OffT>
__device__ __forceinline__ int32_t find_string(const ProbeArgs& a, const unsigned long long* keys, const int32_t* vals,
                                               int64_t i) {
  const OffT* offs = static_cast<const OffT*>(a.data);
  const int64_t o0 = static_cast<int64_t>(offs[i]), len = static_cast<int64_t>(offs[i + 1]) - o0;
  const uint64_t k = string_key(a.bytes + o0, len);
  const OffT* uoffs = static_cast<const OffT*>(a.u_offs);
  for (uint64_t slot = hash64(k) & a.mask;; slot = (slot + 1) & a.mask) {
    const uint64_t cur = keys[slot];
    if (cur == kEmptyKey) return -1;
    if (cur == k) {
      const int32_t id = vals[slot];
      const int64_t u0 = static_cast<int64_t>(uoffs[id]);
      if (static_cast<int64_t>(uoffs[id + 1]) - u0 == len && bytes_equal(a.bytes + o0, a.u_bytes + u0, len)) return a.first_pos[id];
    }
  }
}

// One pass over the values.  Warp w handles the U consecutive 32-row groups starting at group w * U, then strides by
// the grid; fixed-width values of all U groups are loaded before the first probe, so the loads overlap.
template <int KIND, bool SMEM, bool INDEX>
__global__ void __launch_bounds__(kProbeBlock, kProbeBlocksPerSM) set_probe_kernel(const ProbeArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const unsigned long long* keys;
  const int32_t* vals;
  if constexpr (SMEM) {
    const uint4* src = reinterpret_cast<const uint4*>(a.keys);
    uint4* dst = reinterpret_cast<uint4*>(smem);
    for (int64_t k = threadIdx.x; k < (a.table_bytes >> 4); k += kProbeBlock) dst[k] = __ldg(src + k);
    __syncthreads();
    keys = reinterpret_cast<const unsigned long long*>(smem);
    vals = reinterpret_cast<const int32_t*>(smem + (a.mask + 1) * sizeof(unsigned long long));
  } else {
    keys = a.keys;
    vals = a.vals;
  }
  constexpr int U = KIND >= kBoolKey ? 4 : 1;
  const unsigned lane = lane_id();
  const int64_t warp = (blockIdx.x * (int64_t)kProbeBlock + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * kProbeBlock) >> 5;
  unsigned long long nulls = 0;
  for (int64_t w0 = warp * U; w0 < a.n_words; w0 += n_warps * U) {
    uint64_t key[U];
    uint32_t vw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = ((w0 + u) << 5) + lane;
      vw[u] = a.valid.word32(w0 + u);  // zero past n
      if constexpr (KIND > 0) key[u] = i < a.n ? load_value_bits<KIND>(a.data, i) : 0;
      if constexpr (KIND == kBoolKey) key[u] = (a.bits.word32(w0 + u) >> lane) & 1u;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t w = w0 + u;
      if (w >= a.n_words) break;  // warp-uniform
      const int64_t i = (w << 5) + lane;
      const bool in = i < a.n;
      const bool row_valid = (vw[u] >> lane) & 1u;
      int32_t pos = in ? a.null_row_pos : -1;
      if (row_valid) {
        if constexpr (KIND > 0) pos = find_bits(keys, vals, a.mask, a.special_pos, key[u]);
        if constexpr (KIND == kBoolKey) pos = key[u] ? a.true_pos : a.false_pos;
        if constexpr (KIND == kStr32) pos = find_string<int32_t>(a, keys, vals, i);
        if constexpr (KIND == kStr64) pos = find_string<int64_t>(a, keys, vals, i);
      }
      const bool found = pos >= 0;
      if constexpr (INDEX) {
        if (in) st_stream(a.out_index + i, found ? pos : 0);
      } else {
        const unsigned word = __ballot_sync(0xffffffffu, found);
        if (lane == 0) st_stream(a.out_bits + w, word);
      }
      if (a.out_valid) {
        const bool ovalid = found || (in && (row_valid ? a.miss_valid : a.null_miss_valid));
        const unsigned word = __ballot_sync(0xffffffffu, ovalid);
        const unsigned live = __ballot_sync(0xffffffffu, in);
        if (lane == 0) {
          st_stream(a.out_valid + w, word);
          nulls += __popc(live & ~word);
        }
      }
    }
  }
  if (a.out_valid && lane == 0 && nulls) atomicAdd(a.null_count, nulls);
}

// first[id] = min row with that id
__global__ void __launch_bounds__(kBlock) first_position_kernel(const uint32_t* __restrict__ ids, int64_t n, unsigned* first) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock)
    atomicMin(first + ids[i], static_cast<unsigned>(i));
}

// Lays the distinct values out in the table.  slots[0] = first position of the null, slots[1] = that of the value
// whose bits are kEmptyKey (both stay ~0 when absent).
template <int KIND>
__global__ void __launch_bounds__(kBlock) set_layout_kernel(const void* __restrict__ data, const uint8_t* __restrict__ bytes,
                                                            BitmapReader valid, int64_t n_uniques, const unsigned* __restrict__ first,
                                                            unsigned long long* keys, int32_t* vals, uint64_t mask,
                                                            unsigned long long* slots) {
  for (int64_t u = blockIdx.x * (int64_t)kBlock + threadIdx.x; u < n_uniques; u += (int64_t)gridDim.x * kBlock) {
    const unsigned fp = first[u];
    if (!valid.bit(u)) {
      slots[0] = fp;
      continue;
    }
    uint64_t k;
    if constexpr (KIND > 0) {
      k = load_key_bits(data, KIND, u);
      if (k == kEmptyKey) {
        slots[1] = fp;
        continue;
      }
    } else {
      using OffT = std::conditional_t<KIND == kStr32, int32_t, int64_t>;
      const OffT* offs = static_cast<const OffT*>(data);
      const int64_t o0 = static_cast<int64_t>(offs[u]);
      k = string_key(bytes + o0, static_cast<int64_t>(offs[u + 1]) - o0);
    }
    // the uniques are distinct, so every one claims a slot of its own (equal string hashes included)
    uint64_t slot = hash64(k) & mask;
    while (atomicCAS(keys + slot, (unsigned long long)kEmptyKey, (unsigned long long)k) != kEmptyKey) slot = (slot + 1) & mask;
    vals[slot] = KIND > 0 ? static_cast<int32_t>(fp) : static_cast<int32_t>(u);
  }
}

// slots[0] / [1] / [2] = first position of false / true / null
__global__ void __launch_bounds__(kBlock) bool_positions_kernel(BitmapReader bits, BitmapReader valid, int64_t n,
                                                                unsigned long long* slots) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock)
    atomicMin(slots + (valid.bit(i) ? (bits.bit(i) ? 1 : 0) : 2), static_cast<unsigned long long>(i));
}

inline bool set_type_supported(int t) { return t == B2_BOOL || type_is_numeric(t) || type_is_binary_like(t); }

inline int kind_of(int t) {
  if (t == B2_BOOL) return kBoolKey;
  if (type_is_binary_like(t)) return offset_width(t) == 8 ? kStr64 : kStr32;
  return type_width(t);
}

}  // namespace b2

using namespace b2;

struct B2SetLookup {
  B2Context* ctx = nullptr;
  int32_t type = 0;
  int null_matching = 0;
  int32_t null_index = -1;
  int32_t special_pos = -1;
  int32_t false_pos = -1, true_pos = -1;
  uint64_t mask = 0;
  int64_t table_bytes = 0;
  bool shared = false;
  void* table = nullptr;      // keys[mask + 1] then vals[mask + 1]
  void* first_pos = nullptr;  // strings: the first position of every distinct value
  B2Array uniques{};          // strings: the distinct values (owned buffers)
};

namespace {
struct GrouperGuard {
  B2Grouper* g = nullptr;
  ~GrouperGuard() {
    if (g) b2_grouper_destroy(g);
  }
};

void free_state(B2SetLookup* s) {
  cudaStream_t st = s->ctx->stream;
  for (const void* p : {static_cast<const void*>(s->table), static_cast<const void*>(s->first_pos), s->uniques.validity,
                        s->uniques.data, s->uniques.data2})
    if (p) s->ctx->free(const_cast<void*>(p), st);
  delete s;
}

int32_t slot_pos(volatile int64_t* v) { return v[0] == -1 ? -1 : static_cast<int32_t>(v[0]); }

// The largest table the probe stages in shared memory: one that still lets kProbeBlocksPerSM blocks share an SM (the
// registers allow no more), so staging the table never costs occupancy.  On the H100: 113 KB, 8192 slots, at most 4096
// distinct values.
int shared_table_limit(int device, int* out) {
  int per_sm = 0, per_block_optin = 0, reserved = 0;
  B2_CUDA(cudaDeviceGetAttribute(&per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, device));
  B2_CUDA(cudaDeviceGetAttribute(&per_block_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  B2_CUDA(cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, device));
  *out = std::min(per_sm / kProbeBlocksPerSM - reserved, per_block_optin);
  return B2_OK;
}

int build(B2SetLookup* st, const B2Array* vs, cudaStream_t s) {
  B2Context* ctx = st->ctx;
  const int64_t n = vs->length;
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  B2_CUDA(cudaMemsetAsync(slot.dev(), 0xff, 3 * sizeof(int64_t), s));
  unsigned long long* slots = reinterpret_cast<unsigned long long*>(slot.dev());
  const BitmapReader valid(vs->null_count == 0 ? nullptr : vs->validity, vs->offset, n);

  if (vs->type == B2_BOOL) {
    if (n > 0) {
      bool_positions_kernel<<<grid_for(n, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(BitmapReader(vs->data, vs->offset, n), valid, n, slots);
      B2_LAUNCHED();
    }
    B2_RETURN_NOT_OK(slot.fetch(s));
    st->false_pos = slot_pos(slot.host());
    st->true_pos = slot_pos(slot.host() + 1);
    st->null_index = slot_pos(slot.host() + 2);
    return B2_OK;
  }

  GrouperGuard gg;
  PoolArray ids(ctx, s), uniq(ctx, s);
  uint32_t n_uniques = 0;
  if (n > 0) {
    B2_RETURN_NOT_OK(b2_grouper_create(ctx, &vs->type, 1, &gg.g));
    B2_RETURN_NOT_OK(b2_grouper_consume(gg.g, vs, &ids.a, s));
    B2_RETURN_NOT_OK(b2_grouper_uniques(gg.g, &uniq.a, s));
    B2_RETURN_NOT_OK(b2_grouper_num_groups(gg.g, &n_uniques));
  }
  Temp first(ctx, s), table(ctx, s);
  B2_RETURN_NOT_OK(first.alloc(sizeof(unsigned) * n_uniques));
  if (n_uniques > 0) {
    B2_CUDA(cudaMemsetAsync(first.ptr, 0xff, sizeof(unsigned) * n_uniques, s));
    first_position_kernel<<<grid_for(n, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(static_cast<const uint32_t*>(ids.a.data), n,
                                                                              first.as<unsigned>());
    B2_LAUNCHED();
  }
  const uint64_t n_valid = n_uniques - (uniq.a.null_count > 0 ? 1 : 0);  // the null group takes no slot
  const uint64_t cap = next_pow2(std::max<uint64_t>(16, 2ull * n_valid));
  st->mask = cap - 1;
  st->table_bytes = static_cast<int64_t>(cap * (sizeof(unsigned long long) + sizeof(int32_t)));
  B2_RETURN_NOT_OK(table.alloc(st->table_bytes));
  B2_CUDA(cudaMemsetAsync(table.ptr, 0xff, cap * sizeof(unsigned long long), s));
  unsigned long long* keys = table.as<unsigned long long>();
  int32_t* vals = reinterpret_cast<int32_t*>(keys + cap);
  if (n_uniques > 0) {
    const BitmapReader uvalid(uniq.a.null_count == 0 ? nullptr : uniq.a.validity, 0, n_uniques);
    const int grid = grid_for(n_uniques, kBlock, kSMs * 8);
    const void* d = uniq.a.data;
    const uint8_t* b = static_cast<const uint8_t*>(uniq.a.data2);
    switch (kind_of(vs->type)) {
      case 1: set_layout_kernel<1><<<grid, kBlock, 0, s>>>(d, b, uvalid, n_uniques, first.as<unsigned>(), keys, vals, st->mask, slots); break;
      case 2: set_layout_kernel<2><<<grid, kBlock, 0, s>>>(d, b, uvalid, n_uniques, first.as<unsigned>(), keys, vals, st->mask, slots); break;
      case 4: set_layout_kernel<4><<<grid, kBlock, 0, s>>>(d, b, uvalid, n_uniques, first.as<unsigned>(), keys, vals, st->mask, slots); break;
      case 8: set_layout_kernel<8><<<grid, kBlock, 0, s>>>(d, b, uvalid, n_uniques, first.as<unsigned>(), keys, vals, st->mask, slots); break;
      case kStr32: set_layout_kernel<kStr32><<<grid, kBlock, 0, s>>>(d, b, uvalid, n_uniques, first.as<unsigned>(), keys, vals, st->mask, slots); break;
      default: set_layout_kernel<kStr64><<<grid, kBlock, 0, s>>>(d, b, uvalid, n_uniques, first.as<unsigned>(), keys, vals, st->mask, slots); break;
    }
    B2_LAUNCHED();
  }
  B2_RETURN_NOT_OK(slot.fetch(s));
  st->null_index = slot_pos(slot.host());
  st->special_pos = slot_pos(slot.host() + 1);
  int smem_limit = 0;
  B2_RETURN_NOT_OK(shared_table_limit(ctx->device, &smem_limit));
  st->shared = st->table_bytes <= smem_limit;
  st->table = table.release();
  if (type_is_binary_like(vs->type)) {
    st->first_pos = first.release();
    uniq.give(&st->uniques);
  }
  return B2_OK;
}

template <int KIND, bool SMEM, bool INDEX>
int launch_probe(B2Context* ctx, const ProbeArgs& a, cudaStream_t s) {
  auto kernel = set_probe_kernel<KIND, SMEM, INDEX>;
  const int smem = SMEM ? static_cast<int>(a.table_bytes) : 0;
  if constexpr (SMEM) {
    // raised once per device to the largest table the shared path takes, never per call: callers on other threads
    // may be launching the same kernel with other table sizes
    static std::atomic<uint64_t> raised{0};
    if (!(raised.load() & (1ull << ctx->device))) {
      int limit = 0;
      B2_RETURN_NOT_OK(shared_table_limit(ctx->device, &limit));
      B2_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, limit));
      raised.fetch_or(1ull << ctx->device);
    }
  }
  int per_sm = 0;
  B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kProbeBlock, smem));
  constexpr int U = KIND >= kBoolKey ? 4 : 1;
  const int grid = grid_for(a.n_words, (kProbeBlock / 32) * U, ctx->sm_count * std::max(per_sm, 1));
  kernel<<<grid, kProbeBlock, smem, s>>>(a);
  B2_LAUNCHED();
  return B2_OK;
}

template <int KIND>
int dispatch_probe(B2Context* ctx, const ProbeArgs& a, bool shared, bool index, cudaStream_t s) {
  if (shared) return index ? launch_probe<KIND, true, true>(ctx, a, s) : launch_probe<KIND, true, false>(ctx, a, s);
  return index ? launch_probe<KIND, false, true>(ctx, a, s) : launch_probe<KIND, false, false>(ctx, a, s);
}

int probe(B2SetLookup* st, const B2Array* values, bool index, B2Array* out, void* stream) {
  const char* fn = index ? "b2_index_in" : "b2_is_in";
  if (!st || !values || !out) return set_error(B2_INVALID, "%s: null argument", fn);
  if (values->type != st->type)
    return set_error(B2_TYPE_ERROR, "Array type doesn't match type of values set: type id %d vs %d", values->type, st->type);
  B2Context* ctx = st->ctx;
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->pick(stream);
  const int64_t n = values->length;
  const int nm = st->null_matching;
  const bool match = nm == 0, skip = nm == 1, inconclusive = nm == 3;

  ProbeArgs a{};
  a.n = n;
  a.n_words = bitmap_alloc_bytes(n) / 4;
  a.valid = BitmapReader(values->null_count == 0 ? nullptr : values->validity, values->offset, n);
  a.special_pos = st->special_pos;
  a.false_pos = st->false_pos;
  a.true_pos = st->true_pos;
  a.null_row_pos = match ? st->null_index : -1;
  a.miss_valid = index ? false : !(inconclusive && st->null_index != -1);
  a.null_miss_valid = index ? false : (match || skip);
  // the result can hold a null: index_in always; is_in where a miss or a null row gives one
  const bool input_nulls = a.valid.base != nullptr;
  const bool want_valid = index || !a.miss_valid || (input_nulls && !a.null_miss_valid && a.null_row_pos < 0);

  const int kind = kind_of(st->type);
  if (kind > 0) {
    a.data = static_cast<const uint8_t*>(values->data) + values->offset * kind;
  } else if (kind == kBoolKey) {
    a.bits = BitmapReader(values->data, values->offset, n);
  } else {
    a.data = static_cast<const uint8_t*>(values->data) + values->offset * (kind == kStr64 ? 8 : 4);
    a.bytes = static_cast<const uint8_t*>(values->data2);
    a.u_offs = st->uniques.data;
    a.u_bytes = static_cast<const uint8_t*>(st->uniques.data2);
    a.first_pos = static_cast<const int32_t*>(st->first_pos);
  }
  a.keys = static_cast<const unsigned long long*>(st->table);
  a.vals = st->table ? reinterpret_cast<const int32_t*>(a.keys + st->mask + 1) : nullptr;
  a.mask = st->mask;
  a.table_bytes = st->table_bytes;

  Temp data(ctx, s), validity(ctx, s);
  B2_RETURN_NOT_OK(data.alloc(index ? sizeof(int32_t) * n : bitmap_alloc_bytes(n)));
  if (want_valid) B2_RETURN_NOT_OK(validity.alloc(bitmap_alloc_bytes(n)));
  a.out_bits = index ? nullptr : data.as<uint32_t>();
  a.out_index = index ? data.as<int32_t>() : nullptr;
  a.out_valid = validity.as<uint32_t>();
  int64_t nulls = 0;
  if (n > 0) {
    ScalarSlot slot(ctx);
    if (want_valid) {
      B2_RETURN_NOT_OK(slot.zero(s));
      a.null_count = reinterpret_cast<unsigned long long*>(slot.dev());
    }
    switch (kind) {
      case 1: B2_RETURN_NOT_OK(dispatch_probe<1>(ctx, a, st->shared, index, s)); break;
      case 2: B2_RETURN_NOT_OK(dispatch_probe<2>(ctx, a, st->shared, index, s)); break;
      case 4: B2_RETURN_NOT_OK(dispatch_probe<4>(ctx, a, st->shared, index, s)); break;
      case 8: B2_RETURN_NOT_OK(dispatch_probe<8>(ctx, a, st->shared, index, s)); break;
      case kBoolKey: B2_RETURN_NOT_OK(dispatch_probe<kBoolKey>(ctx, a, false, index, s)); break;
      case kStr32: B2_RETURN_NOT_OK(dispatch_probe<kStr32>(ctx, a, st->shared, index, s)); break;
      default: B2_RETURN_NOT_OK(dispatch_probe<kStr64>(ctx, a, st->shared, index, s)); break;
    }
    if (want_valid) {
      B2_RETURN_NOT_OK(slot.fetch(s));
      nulls = slot.host()[0];
    }
  }
  if (nulls == 0 && validity.ptr) {
    ctx->free(validity.ptr, s);  // all valid: drop the bitmap like the reference
    validity.ptr = nullptr;
  }
  fill_out(out, index ? B2_INT32 : B2_BOOL, n, nulls, validity.release(), data.release());
  return B2_OK;
}
}  // namespace

extern "C" int b2_set_lookup_create(B2Context* ctx, const B2Array* value_set, int null_matching, B2SetLookup** out,
                                    void* stream) {
  if (!ctx || !value_set || !out) return set_error(B2_INVALID, "b2_set_lookup_create: null argument");
  if (null_matching < 0 || null_matching > 3)
    return set_error(B2_INVALID, "b2_set_lookup_create: null_matching must be 0 (MATCH), 1 (SKIP), 2 (EMIT_NULL) or 3 (INCONCLUSIVE)");
  if (!set_type_supported(value_set->type))
    return set_error(B2_NOT_IMPLEMENTED, "is_in / index_in: no device kernel for value set type id %d", value_set->type);
  if (value_set->length > INT32_MAX)
    return set_error(B2_CAPACITY_ERROR, "is_in / index_in: a value set of %lld values does not fit int32 positions",
                     static_cast<long long>(value_set->length));
  B2_CUDA(cudaSetDevice(ctx->device));
  auto* st = new B2SetLookup();
  st->ctx = ctx;
  st->type = value_set->type;
  st->null_matching = null_matching;
  const int status = build(st, value_set, ctx->pick(stream));
  if (status != B2_OK) {
    free_state(st);
    return status;
  }
  if (null_matching == 1) st->null_index = -1;  // SKIP: a null in the value set is not recorded
  *out = st;
  return B2_OK;
}

extern "C" void b2_set_lookup_destroy(B2SetLookup* s) {
  if (!s) return;
  cudaSetDevice(s->ctx->device);
  free_state(s);
}

extern "C" int b2_set_lookup_table(const B2SetLookup* s, int64_t* table_bytes, int32_t* shared) {
  if (!s) return set_error(B2_INVALID, "b2_set_lookup_table: null argument");
  if (table_bytes) *table_bytes = s->table_bytes;
  if (shared) *shared = s->shared ? 1 : 0;
  return B2_OK;
}

extern "C" int b2_is_in(B2SetLookup* s, const B2Array* values, B2Array* out, void* stream) {
  return probe(s, values, false, out, stream);
}

extern "C" int b2_index_in(B2SetLookup* s, const B2Array* values, B2Array* out, void* stream) {
  return probe(s, values, true, out, stream);
}
