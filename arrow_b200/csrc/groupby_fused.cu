// groupby_fused.cu -- one-pass (key, value) -> {sum, count} group-by.
//
// This is the aggregate node's per-batch Consume (grouper->Consume followed by
// kernel->consume for each aggregate, cpp/src/arrow/acero/groupby_aggregate_node.cc:210-253)
// for the `hash_sum` + `hash_count(ONLY_VALID)` pair of BASELINE config 3, fused so the
// uint32 id column is never materialised: each row claims/finds its 32-byte slot
// {key, sum, count, first_row} with one CAS and updates sum and count in the same
// 32-byte sector (one DRAM sector RMW per row when the table exceeds L2).
// Results are identical to Grouper + GroupedSumImpl + GroupedCountImpl
// (kernels/hash_aggregate_numeric.cc:274-295, kernels/hash_aggregate.cc:61-245):
// integer sums wrap in 64 bits, float sums accumulate in double, the null key is its own
// group, sum is null for groups whose count is 0 (min_count = 1).  Group ORDER is
// unspecified (as under use_threads in the reference, whose tests sort by key).
//
// Algorithmic bytes: 16.125 B/row + 24.25 B/group (SURVEY section 8d).
#include <type_traits>

#include "bitmap.h"
#include "hash_table.cuh"
#include "groupby_partitioned.cuh"
#include "groupby_compact.cuh"
#include "groupby_dense.cuh"

namespace b2 {

constexpr int kSlotWords = 4;  // 32-byte slots: key, sum, count, spare
constexpr int64_t kChunkRows = 1ll << 26;

struct FusedTable {
  unsigned long long* slots;  // [(cap + 2) * 4]
  uint64_t mask;
};

__global__ void __launch_bounds__(kBlock) fused_init_kernel(FusedTable t) {
  for (uint64_t i = blockIdx.x * (uint64_t)kBlock + threadIdx.x; i < t.mask + 3; i += (uint64_t)gridDim.x * kBlock) {
    ulonglong4 v;
    v.x = kEmptyKey;
    v.y = 0;
    v.z = 0;
    v.w = 0;
    *reinterpret_cast<ulonglong4*>(t.slots + i * kSlotWords) = v;
  }
}

// rows: either [row0, row0 + n) or the explicit list `pending_in`
template <typename V, int KW>
__global__ void __launch_bounds__(kBlock) fused_consume_kernel(const void* __restrict__ keys,
                                                               BitmapReader key_valid,
                                                               const V* __restrict__ values,
                                                               BitmapReader val_valid, int64_t row0, int64_t n,
                                                               const uint32_t* pending_in, FusedTable t,
                                                               uint32_t* pending_out, unsigned long long* counters) {
  for (int64_t j = blockIdx.x * (int64_t)kBlock + threadIdx.x; j < n; j += (int64_t)gridDim.x * kBlock) {
    const int64_t i = pending_in ? row0 + pending_in[j] : row0 + j;
    const bool knull = !key_valid.bit(i);
    const uint64_t key = knull ? 0 : load_key_bits(keys, KW, i);
    bool inserted;
    int64_t slot = table_find_or_insert(t.slots, t.mask, kSlotWords, key, knull, &inserted);
    if (slot < 0) {
      unsigned long long k = atomicAdd(&counters[0], 1ull);
      pending_out[k] = static_cast<uint32_t>(i - row0);
      continue;
    }
    if (inserted) atomicAdd(&counters[1], 1ull);
    if (val_valid.bit(i)) {
      unsigned long long* p = t.slots + slot * kSlotWords;
      const V v = values[i];
      if constexpr (std::is_floating_point<V>::value) atomicAdd(reinterpret_cast<double*>(p + 1), static_cast<double>(v));
      else if constexpr (std::is_signed<V>::value) atomicAdd(p + 1, static_cast<unsigned long long>(static_cast<long long>(v)));
      else atomicAdd(p + 1, static_cast<unsigned long long>(v));
      atomicAdd(p + 2, 1ull);
    }
  }
}

// partial states (key, sum, count) of another group-by -- a peer GPU's groups after the exchange, or another
// thread's table -- added into this table: the fused twin of HashAggregateKernel::merge
// (compute/kernel.h:720-725, GroupByNode::Merge acero/groupby_aggregate_node.cc:255-298)
template <bool IS_FLOAT, int KW>
__global__ void __launch_bounds__(kBlock) fused_merge_kernel(const void* __restrict__ keys, BitmapReader key_valid,
                                                             const unsigned long long* __restrict__ sums,
                                                             const long long* __restrict__ counts, int64_t n, const uint32_t* pending_in,
                                                             FusedTable t, uint32_t* pending_out, unsigned long long* counters) {
  for (int64_t j = blockIdx.x * (int64_t)kBlock + threadIdx.x; j < n; j += (int64_t)gridDim.x * kBlock) {
    const int64_t i = pending_in ? pending_in[j] : j;
    const bool knull = !key_valid.bit(i);
    const uint64_t key = knull ? 0 : load_key_bits(keys, KW, i);
    bool inserted;
    int64_t slot = table_find_or_insert(t.slots, t.mask, kSlotWords, key, knull, &inserted);
    if (slot < 0) {
      unsigned long long k = atomicAdd(&counters[0], 1ull);
      pending_out[k] = static_cast<uint32_t>(i);
      continue;
    }
    if (inserted) atomicAdd(&counters[1], 1ull);
    const long long c = counts[i];
    if (c > 0) {  // a partial with count 0 only asserts that the group exists (its sum slot is null)
      unsigned long long* p = t.slots + slot * kSlotWords;
      if (IS_FLOAT) atomicAdd(reinterpret_cast<double*>(p + 1), __longlong_as_double((long long)sums[i]));
      else atomicAdd(p + 1, sums[i]);
      atomicAdd(p + 2, static_cast<unsigned long long>(c));
    }
  }
}

// move every occupied slot of `src` into `dst` (growth)
__global__ void __launch_bounds__(kBlock) fused_rehash_kernel(FusedTable src, FusedTable dst, int64_t* overflow) {
  for (uint64_t i = blockIdx.x * (uint64_t)kBlock + threadIdx.x; i < src.mask + 3; i += (uint64_t)gridDim.x * kBlock) {
    const unsigned long long* p = src.slots + i * kSlotWords;
    unsigned long long k = p[0];
    const bool special = i > src.mask;
    if (special ? (k != 0ull) : (k == kEmptyKey)) continue;
    bool inserted;
    int64_t slot = special ? table_find_or_insert(dst.slots, dst.mask, kSlotWords, kEmptyKey, i == src.mask + 2, &inserted)
                           : table_find_or_insert(dst.slots, dst.mask, kSlotWords, k, false, &inserted);
    if (slot < 0) {
      *overflow = 1;
      continue;
    }
    unsigned long long* q = dst.slots + slot * kSlotWords;
    q[1] = p[1];
    q[2] = p[2];
  }
}

// occupied slots -> dense output rows (order = slot order); rank via atomic ticket per warp
__global__ void __launch_bounds__(kBlock) fused_emit_kernel(FusedTable t, int key_width, void* out_keys,
                                                            uint32_t* key_validity, unsigned long long* out_sums,
                                                            uint32_t* sum_validity, long long* out_counts,
                                                            unsigned long long* ticket) {
  const uint64_t total = t.mask + 3;
  for (uint64_t base = (blockIdx.x * (uint64_t)kBlock + threadIdx.x) & ~31ull; base < total;
       base += (uint64_t)gridDim.x * kBlock) {
    const uint64_t i = base + lane_id();
    bool occ = false;
    unsigned long long k = 0, sum = 0, cnt = 0;
    if (i < total) {
      const unsigned long long* p = t.slots + i * kSlotWords;
      k = p[0];
      occ = (i > t.mask) ? (k == 0ull) : (k != kEmptyKey);
      sum = p[1];
      cnt = p[2];
    }
    const unsigned m = __ballot_sync(0xffffffffu, occ);
    if (m == 0) continue;
    unsigned long long start = 0;
    if (lane_id() == 0) start = atomicAdd(ticket, (unsigned long long)__popc(m));
    start = __shfl_sync(0xffffffffu, start, 0);
    if (occ) {
      const uint64_t g = start + __popc(m & lanemask_lt());
      const bool is_null = i == t.mask + 2;
      const uint64_t kv = i == t.mask + 1 ? kEmptyKey : (is_null ? 0ull : k);
      switch (key_width) {
        case 1: static_cast<uint8_t*>(out_keys)[g] = static_cast<uint8_t>(kv); break;
        case 2: static_cast<uint16_t*>(out_keys)[g] = static_cast<uint16_t>(kv); break;
        case 4: static_cast<uint32_t*>(out_keys)[g] = static_cast<uint32_t>(kv); break;
        default: static_cast<uint64_t*>(out_keys)[g] = kv; break;
      }
      out_sums[g] = sum;
      out_counts[g] = static_cast<long long>(cnt);
      // validity bitmaps start all-ones; clear the few null bits atomically
      if (is_null) atomicAnd(&key_validity[g >> 5], ~(1u << (g & 31)));
      if (cnt == 0) atomicAnd(&sum_validity[g >> 5], ~(1u << (g & 31)));
    }
  }
}

// counts the zero bits among the first n and clears everything past n (the bitmap started as all-ones;
// Arrow output padding bits are zero -- common.cuh); alloc_words = 32-bit words in the allocation
__global__ void __launch_bounds__(kBlock) count_zero_bits_kernel(uint32_t* bits, int64_t n, int64_t alloc_words, int64_t* out) {
  int64_t nw = (n + 31) >> 5;
  int64_t local = 0;
  for (int64_t w = blockIdx.x * (int64_t)kBlock + threadIdx.x; w < alloc_words; w += (int64_t)gridDim.x * kBlock) {
    if (w >= nw) {
      bits[w] = 0u;
      continue;
    }
    uint32_t v = bits[w];
    int64_t rem = n - (w << 5);
    if (rem < 32) {
      bits[w] = v & ((1u << rem) - 1u);
      v |= ~((1u << rem) - 1u);
    }
    local += 32 - __popc(v);
  }
  int64_t s = block_sum<kBlock>(local);
  if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(out), (unsigned long long)s);
}

}  // namespace b2

using namespace b2;

// Which paths a group-by may take, from the environment (tests force each path)
struct PathSettings {
  bool compact = true;                    // B2_GROUPBY_COMPACT=0 forces the general path
  bool dense = true;                      // B2_GROUPBY_DENSE=0 skips the direct-addressed path
  int64_t dense_band_bytes = 24ll << 20;  // B2_DENSE_BAND_MB: packed state applied per launch (about half the 50 MB L2)
};

static PathSettings path_settings_from_env() {
  PathSettings p;
  const char* e = getenv("B2_GROUPBY_COMPACT");
  p.compact = !(e && e[0] == '0');
  const char* d = getenv("B2_GROUPBY_DENSE");
  p.dense = !(d && d[0] == '0');
  const char* bm = getenv("B2_DENSE_BAND_MB");
  if (bm && atoll(bm) > 0) p.dense_band_bytes = atoll(bm) << 20;
  return p;
}

struct B2GroupBySumCount {
  B2Context* ctx;
  int key_type, value_type;
  PathSettings paths;  // read once, at create
  FusedTable table{};
  uint64_t cap = 0;
  uint64_t groups = 0;
  int64_t hint = 0;  // expected number of groups (0 = unknown); refined after every chunk
  bool hint_given = false;
  int64_t chunks_compact = 0, chunks_general = 0, chunks_atomic = 0, chunks_dense = 0;  // which path consumed each chunk
  // Direct-addressed state (groupby_dense.cuh) accumulated by dense chunks.  It coexists with the hash table: finalize
  // emits straight from it when the table was never needed, otherwise flushes it into the table first.
  struct Dense {
    bool active = false;
    unsigned long long kmin = 0, kflip = 0, range = 0;
    unsigned long long* sums = nullptr;
    unsigned long long* counts = nullptr;
    uint32_t* exists = nullptr;
    unsigned long long null_sum = 0, null_cnt = 0, null_rows = 0;  // the null-key group (host copies)
  } dense;
};

constexpr int64_t kPartMinRows = 1ll << 21;  // below this the plain atomic path is cheaper than 5 launches
template <typename V>
static int fused_consume_partitioned(B2GroupBySumCount* g, const RawColumns& raw, int64_t n, cudaStream_t s);

static int fused_alloc(B2Context* ctx, uint64_t cap, FusedTable* t, cudaStream_t s) {
  void* p;
  B2_RETURN_NOT_OK(ctx->alloc((cap + 2) * kSlotWords * 8, &p, s));
  t->slots = static_cast<unsigned long long*>(p);
  t->mask = cap - 1;
  fused_init_kernel<<<grid_for((int64_t)cap + 2, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(*t);
  B2_LAUNCHED();
  return B2_OK;
}

static int fused_grow(B2GroupBySumCount* g, uint64_t cap, cudaStream_t s) {
  while (true) {
    FusedTable nt;
    B2_RETURN_NOT_OK(fused_alloc(g->ctx, cap, &nt, s));
    ScalarSlot slot(g->ctx);
    B2_RETURN_NOT_OK(slot.zero(s));
    fused_rehash_kernel<<<grid_for((int64_t)g->cap + 2, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(g->table, nt, slot.dev());
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(slot.fetch(s));
    if (slot.host()[0]) {
      g->ctx->free(nt.slots, s);
      cap *= 2;
      continue;
    }
    g->ctx->free(g->table.slots, s);
    g->table = nt;
    g->cap = cap;
    return B2_OK;
  }
}

template <typename V>
static int launch_fused(int kw, int grid, cudaStream_t s, const void* keys, BitmapReader kv, const V* values,
                        BitmapReader vv, int64_t row0, int64_t n, const uint32_t* pin, FusedTable t, uint32_t* pout,
                        unsigned long long* counters) {
  return visit_width<1, 2, 4, 8>(kw, [&](auto w) {
    fused_consume_kernel<V, w><<<grid, kBlock, 0, s>>>(keys, kv, values, vv, row0, n, pin, t, pout, counters);
    return B2_OK;
  });
}

template <bool IS_FLOAT>
static int launch_merge(int kw, int grid, cudaStream_t s, const void* keys, BitmapReader kv, const unsigned long long* sums,
                        const long long* counts, int64_t n, const uint32_t* pin, FusedTable t, uint32_t* pout,
                        unsigned long long* counters) {
  return visit_width<1, 2, 4, 8>(kw, [&](auto w) {
    fused_merge_kernel<IS_FLOAT, w><<<grid, kBlock, 0, s>>>(keys, kv, sums, counts, n, pin, t, pout, counters);
    return B2_OK;
  });
}

// Inserts n rows into the table with launch(grid, todo, pending_in, pending_out, counters), a fused_consume_kernel or
// fused_merge_kernel launch over g->table.  The kernel parks a row whose neighbourhood hit the probe limit in pending_out
// (counters: [0] parked, [1] inserted); the table then grows and only the parked rows are retried.  The table also grows
// when its load passes 1/2.
template <typename Launch>
static int insert_with_retry(B2GroupBySumCount* g, int64_t n, cudaStream_t s, Launch launch) {
  B2Context* ctx = g->ctx;
  Temp pend_a(ctx, s), pend_b(ctx, s);
  B2_RETURN_NOT_OK(pend_a.alloc(sizeof(uint32_t) * (size_t)n));
  const uint32_t* pin = nullptr;
  uint32_t* pout = pend_a.as<uint32_t>();
  int64_t todo = n;
  while (todo > 0) {
    ScalarSlot slot(ctx);
    B2_RETURN_NOT_OK(slot.zero(s));
    B2_RETURN_NOT_OK(launch(grid_for(todo, kBlock * 4, kSMs * 16), todo, pin, pout, reinterpret_cast<unsigned long long*>(slot.dev())));
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(slot.fetch(s));
    const int64_t pending = slot.host()[0];
    g->groups += static_cast<uint64_t>(slot.host()[1]);
    if (pending == 0 && g->groups * 2 <= g->cap) break;
    B2_RETURN_NOT_OK(fused_grow(g, next_pow2(g->groups * 4 > g->cap * 2 ? g->groups * 4 : g->cap * 2), s));
    if (pending == 0) break;
    if (!pend_b.ptr) B2_RETURN_NOT_OK(pend_b.alloc(sizeof(uint32_t) * (size_t)n));
    pin = pout;
    pout = (pout == pend_a.as<uint32_t>()) ? pend_b.as<uint32_t>() : pend_a.as<uint32_t>();
    todo = pending;
  }
  return B2_OK;
}

template <typename V>
static int fused_consume(B2GroupBySumCount* g, const B2Array* keys, const B2Array* values, cudaStream_t s) {
  const int kw = type_width(g->key_type);
  const int64_t n = keys->length;
  RawColumns raw{};
  raw.keys = static_cast<const char*>(keys->data) + keys->offset * kw;
  raw.values = static_cast<const V*>(values->data) + values->offset;
  raw.key_valid = BitmapReader(keys->null_count == 0 ? nullptr : keys->validity, keys->offset, n);
  raw.val_valid = BitmapReader(values->null_count == 0 ? nullptr : values->validity, values->offset, n);
  if (n >= kPartMinRows) return fused_consume_partitioned<V>(g, raw, n, s);
  if (!g->table.slots) B2_RETURN_NOT_OK(fused_alloc(g->ctx, g->cap, &g->table, s));
  ++g->chunks_atomic;
  for (int64_t row0 = 0; row0 < n; row0 += kChunkRows) {
    const int64_t cn = n - row0 < kChunkRows ? n - row0 : kChunkRows;
    B2_RETURN_NOT_OK(insert_with_retry(g, cn, s, [&](int grid, int64_t todo, const uint32_t* pin, uint32_t* pout,
                                                     unsigned long long* counters) {
      return launch_fused<V>(kw, grid, s, raw.keys, raw.key_valid, static_cast<const V*>(raw.values), raw.val_valid, row0, todo, pin, g->table,
                      pout, counters);
    }));
  }
  return B2_OK;
}

// ---- partitioned path (groupby_partitioned.cuh) -------------------------------------------------

template <typename V, int KW>
static int run_partitioned_chunk(B2GroupBySumCount* g, const RawColumns& raw, int64_t cn, int passes, cudaStream_t s,
                                 unsigned long long* d_counters, unsigned long long* ovf_pairs, unsigned int* ovf_counts,
                                 uint64_t ovf_cap) {
  B2Context* ctx = g->ctx;
  constexpr bool kFloat = std::is_floating_point<V>::value;
  FusedTableRef tref{g->table.slots, g->table.mask, ovf_pairs, ovf_counts, ovf_cap};
  const int pre_grid = ctx->sm_count * 4;
  if (passes == 0) {
    preagg_kernel<true, kFloat, V, KW><<<pre_grid, kBlock, 0, s>>>(raw, Tuples{}, cn, tref, d_counters);
    B2_LAUNCHED();
    return B2_OK;
  }
  Temp hist(ctx, s), dbase(ctx, s), lookback(ctx, s);
  Temp ka(ctx, s), va(ctx, s), fa(ctx, s), kb(ctx, s), vb(ctx, s), fb(ctx, s);
  B2_RETURN_NOT_OK(hist.alloc(sizeof(unsigned long long) * 2 * kPartRadix));
  B2_RETURN_NOT_OK(dbase.alloc(sizeof(uint32_t) * 2 * kPartRadix));
  B2_CUDA(cudaMemsetAsync(hist.ptr, 0, sizeof(unsigned long long) * 2 * kPartRadix, s));
  part_hist_kernel<KW><<<grid_for(cn, kBlock * 16, ctx->sm_count * 8), kBlock, 0, s>>>(raw, cn, passes, hist.as<unsigned long long>());
  B2_LAUNCHED();
  part_scan_kernel<<<passes, kPartRadix, 0, s>>>(hist.as<unsigned long long>(), dbase.as<uint32_t>());
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(ka.alloc(8 * (size_t)cn));
  B2_RETURN_NOT_OK(va.alloc(8 * (size_t)cn));
  B2_RETURN_NOT_OK(fa.alloc((size_t)cn));
  if (passes > 1) {
    B2_RETURN_NOT_OK(kb.alloc(8 * (size_t)cn));
    B2_RETURN_NOT_OK(vb.alloc(8 * (size_t)cn));
    B2_RETURN_NOT_OK(fb.alloc((size_t)cn));
  }
  const uint32_t n_tiles = (uint32_t)((cn + kPartTile - 1) / kPartTile);
  const size_t lb_bytes = (size_t)n_tiles * kPartRadix * sizeof(uint32_t) + 256;
  B2_RETURN_NOT_OK(lookback.alloc(lb_bytes));
  constexpr size_t smem = part_smem_bytes();
  PartArgs a;
  a.raw = raw;
  a.n = (uint32_t)cn;
  a.lookback = lookback.as<uint32_t>();
  a.ticket = reinterpret_cast<uint32_t*>(lookback.as<char>() + (size_t)n_tiles * kPartRadix * sizeof(uint32_t));
  // pass 1: user columns -> tuples A, ordered by hash bits 0..7
  B2_CUDA(cudaMemsetAsync(lookback.ptr, 0, lb_bytes, s));
  a.in = Tuples{};
  a.out = Tuples{ka.as<unsigned long long>(), va.as<unsigned long long>(), fa.as<uint8_t>()};
  a.shift = 0;
  a.digit_base = dbase.as<uint32_t>();
  B2_CUDA(cudaFuncSetAttribute(part_pass_kernel<true, V, KW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  part_pass_kernel<true, V, KW><<<n_tiles, kPartThreads, smem, s>>>(a);
  B2_LAUNCHED();
  Tuples sorted = a.out;
  if (passes > 1) {  // pass 2: A -> B, ordered by (hash bits 8..15, hash bits 0..7)
    B2_CUDA(cudaMemsetAsync(lookback.ptr, 0, lb_bytes, s));
    a.in = a.out;
    a.out = Tuples{kb.as<unsigned long long>(), vb.as<unsigned long long>(), fb.as<uint8_t>()};
    a.shift = 8;
    a.digit_base = dbase.as<uint32_t>() + kPartRadix;
    B2_CUDA(cudaFuncSetAttribute(part_pass_kernel<false, int64_t, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    part_pass_kernel<false, int64_t, 8><<<n_tiles, kPartThreads, smem, s>>>(a);
    B2_LAUNCHED();
    sorted = a.out;
  }
  preagg_kernel<false, kFloat, int64_t, 8><<<pre_grid, kBlock, 0, s>>>(RawColumns{}, sorted, cn, tref, d_counters);
  B2_LAUNCHED();
  return B2_OK;
}

// ---- shared helpers of the partitioned / dense paths ---------------------------------------------------
static int ensure_table(B2GroupBySumCount* g, uint64_t min_cap, cudaStream_t s) {
  if (g->table.slots) return B2_OK;
  if (min_cap > g->cap) g->cap = min_cap;
  return fused_alloc(g->ctx, g->cap, &g->table, s);
}

// After kernels that insert through global_accumulate: read the counters, grow the table and replay whatever was parked
// because a neighbourhood hit the probe limit.  counters = slot: [0] parked, [1] inserted, [2] did not fit the parking area.
template <bool IS_FLOAT>
static int absorb_parked(B2GroupBySumCount* g, ScalarSlot& slot, Temp& ovf_pairs, Temp& ovf_counts, cudaStream_t s) {
  B2Context* ctx = g->ctx;
  unsigned long long* dc = reinterpret_cast<unsigned long long*>(slot.dev());
  B2_RETURN_NOT_OK(slot.fetch(s));
  if (slot.host()[2] != 0)
    return set_error(B2_CAPACITY_ERROR, "group-by: %lld more groups than the table sized from expected_groups=%lld can absorb in one batch; "
                     "pass a larger expected_groups (or 0 to let the table grow chunk by chunk)", (long long)slot.host()[2], (long long)g->hint);
  int64_t parked = slot.host()[0];
  g->groups += static_cast<uint64_t>(slot.host()[1]);
  while (parked > 0) {
    // the table filled up: grow it and replay the parked (key, sum, count) entries.  At least double it: parked entries
    // of keys whose hashes share more low bits than the table has would otherwise meet the same full neighbourhood in a
    // table of the same (or a smaller) size on every replay
    const uint64_t want = 4 * (g->groups + (uint64_t)parked);
    B2_RETURN_NOT_OK(fused_grow(g, next_pow2(want > g->cap * 2 ? want : g->cap * 2), s));
    Temp p2(ctx, s), c2(ctx, s);
    B2_RETURN_NOT_OK(p2.alloc(16 * (size_t)parked));
    B2_RETURN_NOT_OK(c2.alloc(4 * (size_t)parked));
    FusedTableRef tref{g->table.slots, g->table.mask, p2.as<unsigned long long>(), c2.as<unsigned int>(), (uint64_t)parked};
    B2_RETURN_NOT_OK(slot.zero(s));
    replay_overflow_kernel<IS_FLOAT><<<grid_for(parked, kBlock * 4, ctx->sm_count * 8), kBlock, 0, s>>>(
        tref, ovf_pairs.as<unsigned long long>(), ovf_counts.as<unsigned int>(), parked, dc);
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(slot.fetch(s));
    g->groups += static_cast<uint64_t>(slot.host()[1]);
    const int64_t again = slot.host()[0];
    if (again > 0) {  // (only if the grown table is somehow still too small) keep the remainder parked
      B2_CUDA(cudaMemcpyAsync(ovf_pairs.ptr, p2.ptr, 16 * (size_t)again, cudaMemcpyDeviceToDevice, s));
      B2_CUDA(cudaMemcpyAsync(ovf_counts.ptr, c2.ptr, 4 * (size_t)again, cudaMemcpyDeviceToDevice, s));
    }
    parked = again;
  }
  if (g->groups * 2 > g->cap) B2_RETURN_NOT_OK(fused_grow(g, next_pow2(g->groups * 4), s));
  return B2_OK;
}

static void dense_release(B2GroupBySumCount* g, cudaStream_t s) {
  auto& d = g->dense;
  if (d.sums) g->ctx->free(d.sums, s);
  if (d.counts) g->ctx->free(d.counts, s);
  if (d.exists) g->ctx->free(d.exists, s);
  d = B2GroupBySumCount::Dense();
}

// number of groups held by the dense state (incl. those whose every value was null), and how many have count 0
static int dense_count(B2GroupBySumCount* g, int64_t* groups, int64_t* empty, cudaStream_t s) {
  ScalarSlot slot(g->ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  dense_count_kernel<<<grid_for((int64_t)g->dense.range, kBlock * 8, g->ctx->sm_count * 8), kBlock, 0, s>>>(g->dense.counts, g->dense.exists,
                                                                                                       g->dense.range, slot.dev());
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(slot.fetch(s));
  *groups = slot.host()[0];
  *empty = slot.host()[1];
  return B2_OK;
}

// dense state -> the global table (one insert per group), then the dense arrays are released
static int flush_dense(B2GroupBySumCount* g, cudaStream_t s) {
  auto& d = g->dense;
  if (!d.active) return B2_OK;
  B2Context* ctx = g->ctx;
  int64_t nd = 0, empty = 0;
  B2_RETURN_NOT_OK(dense_count(g, &nd, &empty, s));
  const uint64_t want = next_pow2(2 * (g->groups + (uint64_t)nd + 1));
  B2_RETURN_NOT_OK(ensure_table(g, want, s));
  if (want > g->cap) B2_RETURN_NOT_OK(fused_grow(g, want, s));
  Temp ovf_pairs(ctx, s), ovf_counts(ctx, s);
  const uint64_t ovf_cap = (uint64_t)nd + 2;
  B2_RETURN_NOT_OK(ovf_pairs.alloc(16 * (size_t)ovf_cap));
  B2_RETURN_NOT_OK(ovf_counts.alloc(4 * (size_t)ovf_cap));
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  unsigned long long* dc = reinterpret_cast<unsigned long long*>(slot.dev());
  FusedTableRef tref{g->table.slots, g->table.mask, ovf_pairs.as<unsigned long long>(), ovf_counts.as<unsigned int>(), ovf_cap};
  if (d.null_rows) {
    dense_null_flush_kernel<<<1, 32, 0, s>>>(tref, d.null_sum, d.null_cnt, dc);
    B2_LAUNCHED();
  }
  dense_flush_kernel<<<grid_for((int64_t)d.range, kBlock * 4, ctx->sm_count * 16), kBlock, 0, s>>>(d.sums, d.counts, d.exists, d.range, d.kmin,
                                                                                                 d.kflip, tref, dc);
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(absorb_parked<false>(g, slot, ovf_pairs, ovf_counts, s));
  dense_release(g, s);
  return B2_OK;
}

// ---- value windows of the dense and compact paths ----------------------------------------------
static inline int bit_width_u64(unsigned long long v) {
  int b = 0;
  while (v) {
    ++b;
    v >>= 1;
  }
  return b;
}

// The window a packed value field holds: v' = value bits - vbase < 2^vb.  Values of at most 4 bytes take their type's
// whole range (nothing to verify).  64-bit values take 4x the sampled range, centred on it (rows outside it are caught
// by the kernels' per-row check), at most vb_cap bits; false when the sampled range itself does not fit.
struct ValueWindow {
  int vb;
  unsigned long long vbase;
};

static bool value_window(const CompactStats& st, int vw, bool vsigned, int vb_cap, ValueWindow* w) {
  if (vw <= 4) {
    w->vb = 8 * vw;
    w->vbase = vsigned ? static_cast<unsigned long long>(-(1ll << (8 * vw - 1))) : 0ull;
    return true;
  }
  if (st.sampled == 0) {
    w->vb = 8;
    w->vbase = 0;
    return true;
  }
  const unsigned long long flip = vsigned ? 0x8000000000000000ull : 0ull;
  const unsigned long long range = st.vmax - st.vmin;  // in the order-preserving domain
  const int need = bit_width_u64(range);
  int vb = need + 2 < 8 ? 8 : need + 2;
  if (vb > vb_cap) vb = vb_cap;
  if (vb < need || vb < 1 || vb > 62) return false;
  w->vb = vb;
  w->vbase = (st.vmin ^ flip) - ((((1ull << vb) - 1ull) - range) / 2);  // wrap-around is fine: v' = bits - vbase (mod 2^64)
  return true;
}

// ---- dense path (groupby_dense.cuh) -------------------------------------------------------------
static void launch_dense_consume(const DenseArgs& a, int grid, cudaStream_t s) {
  if (a.kw == 8 && a.vw == 8) dense_consume_kernel<8, 8><<<grid, kBlock, 0, s>>>(a);
  else if (a.kw == 4 && a.vw == 8) dense_consume_kernel<4, 8><<<grid, kBlock, 0, s>>>(a);
  else if (a.kw == 4 && a.vw == 4) dense_consume_kernel<4, 4><<<grid, kBlock, 0, s>>>(a);
  else dense_consume_kernel<0, 0><<<grid, kBlock, 0, s>>>(a);
}

// One batch's dense state: 64-bit sums and counts and the exists bitmap over `range` slots, and the null-key group
struct DenseBatch {
  Temp sums, counts, exists;
  unsigned long long null_sum = 0, null_cnt = 0, null_rows = 0;
  bool ok = false;  // false: declined, the arrays hold nothing
  DenseBatch(B2Context* ctx, cudaStream_t s) : sums(ctx, s), counts(ctx, s), exists(ctx, s) {}
};

// Runs the packed dense accumulation of n rows.  Row i has key (or group id) keys[row0 + i] of kw bytes and value
// vals[row0 + i] of vw bytes, and both bitmaps are addressed with row0 + i; its slot is (key bits ^ kflip) - kmin.
// Declines (out->ok stays false, nothing else touched) when the window leaves too few bits for 2^22-row sub-batches or a
// row fell outside [0, range) or outside the value window.
static int dense_accumulate(B2Context* ctx, const void* keys, int kw, BitmapReader key_valid, const void* vals, int vw,
                            bool vsigned, BitmapReader val_valid, int64_t row0, int64_t n, unsigned long long kmin,
                            unsigned long long kflip, unsigned long long range, ValueWindow w, int64_t band_bytes,
                            cudaStream_t s, DenseBatch* out) {
  const int m = (63 - w.vb) / 2;  // rows per sub-batch = 2^m: count needs m + 1 bits, sum needs vb + m bits
  if (m < 22) return B2_OK;       // wide values: a drain every < 4M rows costs more than it saves
  const int64_t sub = m >= 30 ? (1ll << 30) : (1ll << m);
  const int sb = w.vb + m;
  Temp packed(ctx, s);
  const size_t words = (size_t)range;
  B2_RETURN_NOT_OK(packed.alloc(words * 8));
  B2_RETURN_NOT_OK(out->sums.alloc(words * 8));
  B2_RETURN_NOT_OK(out->counts.alloc(words * 8));
  B2_RETURN_NOT_OK(out->exists.alloc((words / 32 + 2) * 4));
  B2_CUDA(cudaMemsetAsync(packed.ptr, 0, words * 8, s));
  B2_CUDA(cudaMemsetAsync(out->sums.ptr, 0, words * 8, s));
  B2_CUDA(cudaMemsetAsync(out->counts.ptr, 0, words * 8, s));
  B2_CUDA(cudaMemsetAsync(out->exists.ptr, 0, (words / 32 + 2) * 4, s));
  ScalarSlot sslot(ctx);
  B2_RETURN_NOT_OK(sslot.zero(s));  // [0] overflow flag, [1..3] null-key accumulator, [4] max count
  DenseArgs a{};
  a.kw = kw;
  a.vw = vw;
  a.vsigned = vsigned;
  a.key_valid = key_valid;
  a.val_valid = val_valid;
  a.kmin = kmin;
  a.kflip = kflip;
  a.range = range;
  a.vbase = w.vbase;
  a.vb = w.vb;
  a.sb = sb;
  a.table = packed.as<unsigned long long>();
  a.exists = out->exists.as<uint32_t>();
  a.overflow = reinterpret_cast<unsigned int*>(sslot.dev());
  a.null_acc = reinterpret_cast<unsigned long long*>(sslot.dev() + 1);
  const unsigned long long band_keys = (unsigned long long)(band_bytes / 8);
  const int bands = (int)((range + band_keys - 1) / band_keys);
  const int grid = grid_for(n < sub ? n : sub, kBlock * 16, ctx->sm_count * 8);
  const int dgrid = grid_for((int64_t)range, kBlock * 8, ctx->sm_count * 8);
  unsigned long long* d_max = reinterpret_cast<unsigned long long*>(sslot.dev() + 4);
  for (int64_t off = 0; off < n; off += sub) {
    a.row0 = row0 + off;
    a.n = n - off < sub ? n - off : sub;
    a.keys = static_cast<const uint8_t*>(keys) + (size_t)a.row0 * kw;
    a.vals = static_cast<const uint8_t*>(vals) + (size_t)a.row0 * vw;
    for (int b = 0; b < bands; ++b) {
      a.band_lo = (unsigned long long)b * band_keys;
      a.band_hi = b == bands - 1 ? range : a.band_lo + band_keys;
      launch_dense_consume(a, grid, s);
      B2_LAUNCHED();
    }
    // Fold the packed words into the 64-bit arrays only when the NEXT sub-batch could overflow a count field (2^m rows of
    // one key): a cheap max-count pass (reads the table once) guards the drain; the last sub-batch always drains.
    const bool last = off + sub >= n;
    if (!last) {
      B2_CUDA(cudaMemsetAsync(d_max, 0, 8, s));
      dense_maxcount_kernel<<<dgrid, kBlock, 0, s>>>(packed.as<unsigned long long>(), range, sb, d_max);
      B2_LAUNCHED();
    }
    const int64_t next_rows = last ? 0 : (n - off - sub < sub ? n - off - sub : sub);
    dense_drain_kernel<<<dgrid, kBlock, 0, s>>>(packed.as<unsigned long long>(), range, sb, w.vbase, out->sums.as<unsigned long long>(),
                                                out->counts.as<unsigned long long>(), last ? nullptr : d_max,
                                                (unsigned long long)next_rows, 1ull << m);
    B2_LAUNCHED();
  }
  B2_RETURN_NOT_OK(sslot.fetch(s));
  if (sslot.host()[0] != 0) return B2_OK;
  out->null_sum = static_cast<unsigned long long>(sslot.host()[1]);
  out->null_cnt = static_cast<unsigned long long>(sslot.host()[2]);
  out->null_rows = static_cast<unsigned long long>(sslot.host()[3]);
  out->ok = true;
  return B2_OK;
}

// Runs one chunk on the direct-addressed path when a sample says the keys are dense and the values narrow.
// *done = false: not applicable, or a row fell outside the sampled windows -- nothing has touched the group-by's state.
template <int KW>
static int try_dense_chunk(B2GroupBySumCount* g, const RawColumns& raw, int64_t cn, cudaStream_t s, bool* done) {
  *done = false;
  B2Context* ctx = g->ctx;
  if (!g->paths.dense || cn < (1 << 22)) return B2_OK;
  const int vt = g->value_type;
  if (vt == B2_FLOAT || vt == B2_DOUBLE) return B2_OK;
  const int vw = type_width(vt);
  const bool vsigned = type_is_signed_int(vt);
  const unsigned long long kflip = type_is_signed_int(g->key_type) ? (1ull << (8 * KW - 1)) : 0ull;
  // sample keys (and 64-bit values)
  ScalarSlot sslot(ctx);
  B2_RETURN_NOT_OK(sslot.zero(s));
  CompactStats* d_stats = reinterpret_cast<CompactStats*>(sslot.dev());
  B2_CUDA(cudaMemsetAsync(&d_stats->kmin, 0xff, 8, s));
  B2_CUDA(cudaMemsetAsync(&d_stats->vmin, 0xff, 8, s));
  const int64_t step = cn > 65536 ? cn / 65536 : 1;
  dense_sample_kernel<KW><<<64, kBlock, 0, s>>>(raw.keys, raw.key_valid, static_cast<const unsigned long long*>(raw.values), raw.val_valid,
                                                raw.row0, cn, step, kflip, vw == 8, vsigned, d_stats);
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(sslot.fetch(s));
  CompactStats st;
  memcpy(&st, const_cast<const int64_t*>(reinterpret_cast<volatile int64_t*>(sslot.host())), sizeof(st));
  if (st.kmax < st.kmin) return B2_OK;  // no valid key in the sample
  const unsigned long long krange = st.kmax - st.kmin + 1;
  if (krange == 0 || krange > kDenseMaxRange) return B2_OK;
  const unsigned long long slack = krange / 64 + 1024;  // rows outside the padded window are caught by the kernel's check
  unsigned long long kmin = st.kmin > slack ? st.kmin - slack : 0ull;
  unsigned long long range = (st.kmax - kmin) + 1 + slack;
  // a later batch whose sample falls inside the window of the state already held keeps that window: its result is
  // added to the state element-wise instead of going through the hash table
  const bool reuse = g->dense.active && g->dense.kflip == kflip && st.kmin >= g->dense.kmin && st.kmax < g->dense.kmin + g->dense.range;
  if (reuse) {
    kmin = g->dense.kmin;
    range = g->dense.range;
  }
  if (range > kDenseMaxRange + kDenseMaxRange / 32) return B2_OK;
  if ((unsigned long long)cn < 4 * range) return B2_OK;  // too few rows per slot: flushing the table would dominate
  // value_window may cut a window down to the 62-bit cap instead of refusing it; dense_accumulate still declines such a
  // window, as its sub-batches of at least 2^22 rows need vb <= 19
  ValueWindow w;
  if (!value_window(st, vw, vsigned, 62, &w)) return B2_OK;
  DenseBatch b(ctx, s);
  B2_RETURN_NOT_OK(dense_accumulate(ctx, raw.keys, KW, raw.key_valid, raw.values, vw, vsigned, raw.val_valid, raw.row0, cn, kmin,
                                    kflip, range, w, g->paths.dense_band_bytes, s, &b));
  if (!b.ok) return B2_OK;  // values too wide, or a row outside the sampled windows: partitioned path
  auto& d = g->dense;
  if (reuse) {
    dense_merge_kernel<<<grid_for((int64_t)range, kBlock * 8, ctx->sm_count * 8), kBlock, 0, s>>>(
        d.sums, d.counts, d.exists, b.sums.as<unsigned long long>(), b.counts.as<unsigned long long>(), b.exists.as<uint32_t>(), range);
    B2_LAUNCHED();
  } else {
    B2_RETURN_NOT_OK(flush_dense(g, s));  // a state with another window goes to the hash table first
    d.active = true;
    d.kmin = kmin;
    d.kflip = kflip;
    d.range = range;
    d.sums = static_cast<unsigned long long*>(b.sums.release());
    d.counts = static_cast<unsigned long long*>(b.counts.release());
    d.exists = static_cast<uint32_t*>(b.exists.release());
  }
  d.null_sum += b.null_sum;
  d.null_cnt += b.null_cnt;
  d.null_rows += b.null_rows;
  *done = true;
  return B2_OK;
}

// Runs one chunk on the compact path when the measured key range and the (verified) value window fit one
// 64-bit tuple.  *done = false means "not applicable" (or the value window was violated): nothing has
// touched the global table and the caller runs the general path on the same chunk.
template <int KW>
static int try_compact_chunk(B2GroupBySumCount* g, const RawColumns& raw, int64_t cn, int passes, cudaStream_t s,
                             unsigned long long* d_counters, unsigned long long* ovf_pairs, unsigned int* ovf_counts,
                             uint64_t ovf_cap, bool* done) {
  *done = false;
  B2Context* ctx = g->ctx;
  if (!g->paths.compact || passes == 0) return B2_OK;
  const int vt = g->value_type;
  if (vt == B2_FLOAT || vt == B2_DOUBLE) return B2_OK;  // float sums accumulate in double: general path
  const int vw = type_width(vt);
  const bool vsigned = type_is_signed_int(vt);
  const unsigned long long kflip = type_is_signed_int(g->key_type) ? (1ull << (8 * KW - 1)) : 0ull;

  // 1. stats: exact key range, null keys, both digit histograms; a sample of the 64-bit value range
  Temp hist(ctx, s), dbase(ctx, s);
  B2_RETURN_NOT_OK(hist.alloc(sizeof(unsigned long long) * 2 * kPartRadix));
  B2_RETURN_NOT_OK(dbase.alloc(sizeof(uint32_t) * 2 * kPartRadix));
  B2_CUDA(cudaMemsetAsync(hist.ptr, 0, sizeof(unsigned long long) * 2 * kPartRadix, s));
  ScalarSlot sslot(ctx);
  B2_RETURN_NOT_OK(sslot.zero(s));
  CompactStats* d_stats = reinterpret_cast<CompactStats*>(sslot.dev());
  static_assert(sizeof(CompactStats) <= 64, "CompactStats must fit the front of a scalar slot");
  B2_CUDA(cudaMemsetAsync(&d_stats->kmin, 0xff, 8, s));
  B2_CUDA(cudaMemsetAsync(&d_stats->vmin, 0xff, 8, s));
  compact_stats_kernel<KW><<<grid_for(cn, kBlock * 16, ctx->sm_count * 8), kBlock, 0, s>>>(
      raw.keys, raw.key_valid, raw.row0, cn, kflip, passes, hist.as<unsigned long long>(), d_stats);
  B2_LAUNCHED();
  if (vw == 8) {
    const int64_t step = cn > 65536 ? cn / 65536 : 1;
    compact_value_sample_kernel<<<64, kBlock, 0, s>>>(static_cast<const unsigned long long*>(raw.values), raw.val_valid, raw.row0,
                                                     cn, step, vsigned, d_stats);
    B2_LAUNCHED();
  }
  part_scan_kernel<<<passes, kPartRadix, 0, s>>>(hist.as<unsigned long long>(), dbase.as<uint32_t>());
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(sslot.fetch(s));
  CompactStats st;
  memcpy(&st, const_cast<const int64_t*>(reinterpret_cast<volatile int64_t*>(sslot.host())), sizeof(st));
  const int64_t n_tuples = cn - (int64_t)st.null_keys;
  if (n_tuples <= 0) return B2_OK;  // every key null: general path

  // 2. tuple encoding
  CompactEnc enc;
  enc.kmin = st.kmin;
  enc.kflip = kflip;
  enc.kb = bit_width_u64(st.kmax - st.kmin);
  if (enc.kb < 1) enc.kb = 1;
  ValueWindow w;
  if (!value_window(st, vw, vsigned, 63 - enc.kb, &w)) return B2_OK;
  enc.vb = w.vb;
  enc.vbase = w.vbase;
  if (enc.kb + enc.vb + 1 > 64) return B2_OK;

  // 3. passes
  const uint32_t n_tiles_in = (uint32_t)((cn + kCTile - 1) / kCTile);
  const uint32_t n_tiles_t = (uint32_t)((n_tuples + kCTile - 1) / kCTile);
  Temp bufA(ctx, s), bufB(ctx, s), lookback(ctx, s);
  B2_RETURN_NOT_OK(bufA.alloc((size_t)n_tiles_t * kCTile * 8 + 256));
  if (passes > 1) B2_RETURN_NOT_OK(bufB.alloc((size_t)n_tiles_t * kCTile * 8 + 256));
  const size_t lb_bytes = (size_t)n_tiles_in * kPartRadix * sizeof(uint32_t) + 256;
  B2_RETURN_NOT_OK(lookback.alloc(lb_bytes));
  B2_CUDA(cudaMemsetAsync(lookback.ptr, 0, lb_bytes, s));
  B2_RETURN_NOT_OK(sslot.zero(s));  // reuse the slot: [0] overflow flag, [1..3] null-key accumulator
  CompactArgs a{};
  a.keys = static_cast<const uint8_t*>(raw.keys) + (size_t)raw.row0 * KW;
  a.vals = static_cast<const uint8_t*>(raw.values) + (size_t)raw.row0 * vw;
  a.kw = KW;
  a.vw = vw;
  a.vsigned = vsigned;
  a.bulk_ok = aligned_to(a.keys, 16) && aligned_to(a.vals, 16);
  a.key_valid = raw.key_valid;
  a.val_valid = raw.val_valid;
  a.row0 = raw.row0;
  a.in = nullptr;
  a.out = bufA.as<unsigned long long>();
  a.n = (uint32_t)cn;
  a.enc = enc;
  a.shift = 24;
  a.digit_base = dbase.as<uint32_t>();
  a.lookback = lookback.as<uint32_t>();
  a.ticket = reinterpret_cast<uint32_t*>(lookback.as<char>() + (size_t)n_tiles_in * kPartRadix * sizeof(uint32_t));
  a.overflow = reinterpret_cast<unsigned int*>(sslot.dev());
  a.null_acc = reinterpret_cast<unsigned long long*>(sslot.dev() + 1);
  const int max_ctas = ctx->sm_count * 2;
  {
    const int grid1 = (int)n_tiles_in < max_ctas ? (int)n_tiles_in : max_ctas;
    const size_t sm1 = compact_pass_smem(true);
    if (KW == 8 && vw == 8) {
      B2_CUDA(cudaFuncSetAttribute(compact_pass_kernel<true, 8, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1));
      compact_pass_kernel<true, 8, 8><<<grid1, kCThreads, sm1, s>>>(a);
    } else if (KW == 4 && vw == 4) {
      B2_CUDA(cudaFuncSetAttribute(compact_pass_kernel<true, 4, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1));
      compact_pass_kernel<true, 4, 4><<<grid1, kCThreads, sm1, s>>>(a);
    } else {
      B2_CUDA(cudaFuncSetAttribute(compact_pass_kernel<true, 0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1));
      compact_pass_kernel<true, 0, 0><<<grid1, kCThreads, sm1, s>>>(a);
    }
  }
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(sslot.fetch(s));
  if (sslot.host()[0] != 0) return B2_OK;  // a value outside the sampled window: redo the chunk on the general path
  FusedTableRef tref{g->table.slots, g->table.mask, ovf_pairs, ovf_counts, ovf_cap};
  if (st.null_keys) {
    compact_null_flush_kernel<<<1, 32, 0, s>>>(tref, reinterpret_cast<const unsigned long long*>(sslot.dev() + 1), d_counters);
    B2_LAUNCHED();
  }
  const unsigned long long* sorted = bufA.as<unsigned long long>();
  if (passes > 1) {
    const size_t lb2 = (size_t)n_tiles_t * kPartRadix * sizeof(uint32_t) + 256;
    B2_CUDA(cudaMemsetAsync(lookback.ptr, 0, lb2, s));
    a.in = bufA.as<unsigned long long>();
    a.out = bufB.as<unsigned long long>();
    a.n = (uint32_t)n_tuples;
    a.shift = 16;
    a.digit_base = dbase.as<uint32_t>() + kPartRadix;
    a.ticket = reinterpret_cast<uint32_t*>(lookback.as<char>() + (size_t)n_tiles_t * kPartRadix * sizeof(uint32_t));
    B2_CUDA(cudaFuncSetAttribute(compact_pass_kernel<false, 0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)compact_pass_smem(false)));
    compact_pass_kernel<false, 0, 0><<<(int)n_tiles_t < max_ctas ? (int)n_tiles_t : max_ctas, kCThreads, compact_pass_smem(false), s>>>(a);
    B2_LAUNCHED();
    sorted = bufB.as<unsigned long long>();
  }
  const bool narrow = enc.kb <= 31 && enc.vb <= 19;
  if (narrow) {
    B2_CUDA(cudaFuncSetAttribute(compact_preagg_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)compact_preagg_smem<true>()));
    compact_preagg_kernel<true><<<max_ctas, kCThreads, compact_preagg_smem<true>(), s>>>(sorted, (uint32_t)n_tuples, enc, tref, d_counters);
  } else {
    B2_CUDA(cudaFuncSetAttribute(compact_preagg_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)compact_preagg_smem<false>()));
    compact_preagg_kernel<false><<<max_ctas, kCThreads, compact_preagg_smem<false>(), s>>>(sorted, (uint32_t)n_tuples, enc, tref, d_counters);
  }
  B2_LAUNCHED();
  *done = true;
  return B2_OK;
}

// Consumes rows [0, n) of `raw` chunk by chunk: each chunk goes to the dense path, else the compact path, else the
// general path
template <typename V, int KW>
static int consume_chunks(B2GroupBySumCount* g, RawColumns raw, int64_t n, int64_t max_chunk, cudaStream_t s) {
  B2Context* ctx = g->ctx;
  constexpr bool kFloat = std::is_floating_point<V>::value;
  for (int64_t row0 = 0; row0 < n;) {
    const int64_t remaining = n - row0;
    raw.row0 = row0;
    // the direct-addressed path needs no per-row scratch memory: it is offered everything that is left, whatever the
    // memory-driven chunk size of the partitioned paths
    bool done = false;
    B2_RETURN_NOT_OK(try_dense_chunk<KW>(g, raw, remaining, s, &done));
    if (done) {
      ++g->chunks_dense;
      break;
    }
    const int64_t cn = remaining < max_chunk ? remaining : max_chunk;
    const uint64_t ovf_cap = static_cast<uint64_t>(cn < kChunkRows ? cn : kChunkRows);
    const int64_t est = g->hint > 0 ? g->hint : (g->groups > 0 ? (int64_t)g->groups : (1ll << 40));
    const int passes = est <= 1500 ? 0 : (est <= 200000 ? 1 : 2);
    // parking space for entries that hit the probe limit (worst case: every row of the chunk)
    Temp ovf_pairs(ctx, s), ovf_counts(ctx, s);
    B2_RETURN_NOT_OK(ovf_pairs.alloc(16 * (size_t)ovf_cap));
    B2_RETURN_NOT_OK(ovf_counts.alloc(4 * (size_t)ovf_cap));
    ScalarSlot slot(ctx);
    B2_RETURN_NOT_OK(slot.zero(s));
    unsigned long long* dc = reinterpret_cast<unsigned long long*>(slot.dev());
    unsigned long long* op = ovf_pairs.as<unsigned long long>();
    unsigned int* oc = ovf_counts.as<unsigned int>();
    // the partitioned paths insert into the global table: create it on first use
    B2_RETURN_NOT_OK(ensure_table(g, next_pow2(2 * (uint64_t)(g->hint > (1 << 19) ? g->hint : (1 << 19))), s));
    B2_RETURN_NOT_OK(try_compact_chunk<KW>(g, raw, cn, passes, s, dc, op, oc, ovf_cap, &done));
    if (done) {
      ++g->chunks_compact;
    } else {
      ++g->chunks_general;
      B2_RETURN_NOT_OK((run_partitioned_chunk<V, KW>(g, raw, cn, passes, s, dc, op, oc, ovf_cap)));
    }
    B2_RETURN_NOT_OK(absorb_parked<kFloat>(g, slot, ovf_pairs, ovf_counts, s));
    if (g->hint <= 0 || (int64_t)g->groups > g->hint) g->hint = (int64_t)g->groups;  // measured cardinality
    row0 += cn;
  }
  return B2_OK;
}

template <typename V>
static int fused_consume_partitioned(B2GroupBySumCount* g, const RawColumns& raw, int64_t n, cudaStream_t s) {
  B2Context* ctx = g->ctx;
  // Chunking.  Pre-aggregation pays off in proportion to how often a key repeats INSIDE one chunk, so
  // chunks should be as large as memory allows (tuples: 2 x 17 B/row).  Entries that hit a full table
  // are parked and replayed after growth; the parking area holds min(chunk, 64M) entries, so without a
  // cardinality hint chunks stay at 64M rows (worst case fully parkable), while a caller that passes
  // expected_groups gets one chunk of up to 2^30 rows and a capacity error only if the true cardinality
  // exceeds the hint by more than the table slack + 64M groups inside a single chunk.
  size_t free_b = 0, total_b = 0;
  cudaMemGetInfo(&free_b, &total_b);
  const int64_t mem_rows = static_cast<int64_t>((free_b + (size_t)(ctx->bytes_reserved - ctx->bytes_in_use)) / 48);
  int64_t max_chunk = g->hint_given ? ((1ll << 30) - kPartTile) : kChunkRows;
  if (max_chunk > mem_rows) max_chunk = mem_rows > kChunkRows ? mem_rows / kPartTile * kPartTile : kChunkRows;
  return visit_width<1, 2, 4, 8>(type_width(g->key_type), [&](auto w) { return consume_chunks<V, w>(g, raw, n, max_chunk, s); });
}

// The dense path with GROUP IDS as keys: the consume of a hash_sum HashAggregateKernel over an integer column
// (hash_aggregate.cu) -- sums[id] += value, counts[id] += 1 for the valid values -- as ONE packed RED per row into an
// L2-resident table instead of two atomics into two arrays.  *done = false:
// not applicable (floats, too few rows per group, values wider than the packed word allows or outside the sampled
// window); nothing has been added to sums / counts and the caller runs its own kernel.
int b2::dense_sum_count_by_id(B2Context* ctx, const uint32_t* ids, uint64_t num_groups, const void* values, int value_type,
                              BitmapReader val_valid, int64_t n, unsigned long long* sums, unsigned long long* counts,
                              cudaStream_t s, bool* done) {
  *done = false;
  const PathSettings paths = path_settings_from_env();
  if (!paths.dense) return B2_OK;
  const int vt = value_type;
  if (vt == B2_FLOAT || vt == B2_DOUBLE || n < (1 << 22) || num_groups == 0) return B2_OK;
  if (num_groups > kDenseMaxRange || (uint64_t)n < 4 * num_groups) return B2_OK;
  const int vw = type_width(vt);
  const bool vsigned = type_is_signed_int(vt);
  CompactStats st{};
  if (vw == 8) {  // narrower values take their type's whole range: nothing to sample
    ScalarSlot sslot(ctx);
    B2_RETURN_NOT_OK(sslot.zero(s));
    CompactStats* d_stats = reinterpret_cast<CompactStats*>(sslot.dev());
    B2_CUDA(cudaMemsetAsync(&d_stats->vmin, 0xff, 8, s));
    const int64_t step = n > 65536 ? n / 65536 : 1;
    compact_value_sample_kernel<<<64, kBlock, 0, s>>>(static_cast<const unsigned long long*>(values), val_valid, 0, n, step, vsigned,
                                                     d_stats);
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(sslot.fetch(s));
    memcpy(&st, const_cast<const int64_t*>(reinterpret_cast<volatile int64_t*>(sslot.host())), sizeof(st));
  }
  // value_window may cut a window down to the 62-bit cap instead of refusing it; dense_accumulate still declines such a
  // window, as its sub-batches of at least 2^22 rows need vb <= 19
  ValueWindow w;
  if (!value_window(st, vw, vsigned, 62, &w)) return B2_OK;
  // ids are never null; an id >= num_groups raises the overflow flag, and the caller's kernel then reports it its own way
  const unsigned long long range = num_groups;
  DenseBatch b(ctx, s);
  B2_RETURN_NOT_OK(dense_accumulate(ctx, ids, 4, BitmapReader(nullptr, 0, n), values, vw, vsigned, val_valid, 0, n, 0, 0, range, w,
                                    paths.dense_band_bytes, s, &b));
  if (!b.ok) return B2_OK;  // values too wide, a value outside the sampled window or a bad id: the caller's kernel runs the batch
  dense_merge_kernel<<<grid_for((int64_t)range, kBlock * 8, ctx->sm_count * 8), kBlock, 0, s>>>(
      sums, counts, b.exists.as<uint32_t>(), b.sums.as<unsigned long long>(), b.counts.as<unsigned long long>(), b.exists.as<uint32_t>(),
      range);
  B2_LAUNCHED();
  *done = true;
  return B2_OK;
}

extern "C" {

int b2_groupby_sumcount_create(B2Context* ctx, int32_t key_type, int32_t value_type, int64_t expected_groups,
                               B2GroupBySumCount** out) {
  if (!ctx || !out) return set_error(B2_INVALID, "b2_groupby_sumcount_create: null argument");
  if (type_width(key_type) == 0) return set_error(B2_NOT_IMPLEMENTED, "group-by key type id %d", key_type);
  if (!type_is_numeric(value_type)) return set_error(B2_NOT_IMPLEMENTED, "group-by value type id %d", value_type);
  B2_CUDA(cudaSetDevice(ctx->device));
  B2GroupBySumCount* g = new B2GroupBySumCount();
  g->ctx = ctx;
  g->key_type = key_type;
  g->value_type = value_type;
  g->paths = path_settings_from_env();
  uint64_t cap = next_pow2(expected_groups > 0 ? (uint64_t)expected_groups * 2 : (1u << 16));
  if (cap < 1024) cap = 1024;
  // the table is allocated and initialised lazily on the first consume, on the CALLER's stream:
  // an init kernel queued on the context stream would race with a consume on another stream
  g->cap = cap;
  g->hint = expected_groups;
  g->hint_given = expected_groups > 0;
  *out = g;
  return B2_OK;
}

void b2_groupby_sumcount_destroy(B2GroupBySumCount* g) {
  if (!g) return;
  cudaSetDevice(g->ctx->device);
  if (g->table.slots) g->ctx->free(g->table.slots, g->ctx->stream);
  dense_release(g, g->ctx->stream);
  delete g;
}

int b2_groupby_sumcount_consume(B2GroupBySumCount* g, const B2Array* keys, const B2Array* values, void* stream) {
  if (!g || !keys || !values) return set_error(B2_INVALID, "b2_groupby_sumcount_consume: null argument");
  if (keys->type != g->key_type || values->type != g->value_type)
    return set_error(B2_TYPE_ERROR, "group-by was created for (key %d, value %d), got (%d, %d)", g->key_type,
                     g->value_type, keys->type, values->type);
  if (keys->length != values->length) return set_error(B2_INVALID, "keys and values differ in length");
  cudaStream_t s = g->ctx->pick(stream);
  B2_CUDA(cudaSetDevice(g->ctx->device));
  if (keys->length == 0) return B2_OK;
  return visit_type(NumericTypes{}, values->type, [&](auto tag) { return fused_consume<decltype(tag)>(g, keys, values, s); });
}

int b2_groupby_sumcount_merge(B2GroupBySumCount* g, const B2Array* keys, const B2Array* sums, const B2Array* counts, void* stream) {
  if (!g || !keys || !sums || !counts) return set_error(B2_INVALID, "b2_groupby_sumcount_merge: null argument");
  if (keys->type != g->key_type) return set_error(B2_TYPE_ERROR, "merge: key type id %d, expected %d", keys->type, g->key_type);
  const int sum_type = sum_type_of(g->value_type);
  if (sums->type != sum_type || counts->type != B2_INT64)
    return set_error(B2_TYPE_ERROR, "merge: sums must have type id %d and counts int64 (got %d, %d)", sum_type, sums->type, counts->type);
  if (sums->length != keys->length || counts->length != keys->length) return set_error(B2_INVALID, "merge: columns differ in length");
  if (keys->length >= (1ll << 32)) return set_error(B2_NOT_IMPLEMENTED, "merge: at most 2^32 - 1 partial groups per call");
  B2Context* ctx = g->ctx;
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = keys->length;
  if (n == 0) return B2_OK;
  // size the table for the partials up front: every partial may be a new group
  const uint64_t want = next_pow2(2 * (g->groups + (uint64_t)n));
  B2_RETURN_NOT_OK(ensure_table(g, want, s));
  if (want > g->cap) B2_RETURN_NOT_OK(fused_grow(g, want, s));
  const int kw = type_width(g->key_type);
  const void* kdata = static_cast<const char*>(keys->data) + keys->offset * kw;
  const unsigned long long* sdata = static_cast<const unsigned long long*>(sums->data) + sums->offset;
  const long long* cdata = static_cast<const long long*>(counts->data) + counts->offset;
  BitmapReader kv(keys->null_count == 0 ? nullptr : keys->validity, keys->offset, n);
  // the table was sized for every partial above, so its load stays at most 1/2 and it grows only when a neighbourhood
  // hits the probe limit, to twice its size
  const auto launch = sum_type == B2_DOUBLE ? launch_merge<true> : launch_merge<false>;
  B2_RETURN_NOT_OK(insert_with_retry(g, n, s, [&](int grid, int64_t todo, const uint32_t* pin, uint32_t* pout,
                                                  unsigned long long* counters) {
    return launch(kw, grid, s, kdata, kv, sdata, cdata, todo, pin, g->table, pout, counters);
  }));
  if (g->hint <= 0 || (int64_t)g->groups > g->hint) g->hint = (int64_t)g->groups;
  return B2_OK;
}

int b2_groupby_sumcount_path_counts(const B2GroupBySumCount* g, int64_t* dense, int64_t* compact, int64_t* general, int64_t* atomic) {
  if (!g) return set_error(B2_INVALID, "b2_groupby_sumcount_path_counts: null argument");
  if (dense) *dense = g->chunks_dense;
  if (compact) *compact = g->chunks_compact;
  if (general) *general = g->chunks_general;
  if (atomic) *atomic = g->chunks_atomic;
  return B2_OK;
}

int b2_groupby_sumcount_finalize(B2GroupBySumCount* g, B2Array* out_keys, B2Array* out_sums, B2Array* out_counts,
                                 void* stream) {
  if (!g || !out_keys || !out_sums || !out_counts) return set_error(B2_INVALID, "b2_groupby_sumcount_finalize: null argument");
  B2Context* ctx = g->ctx;
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  // dense state: emitted directly when the hash table was never needed (the single-batch dense case: no table is ever
  // allocated, initialised or scanned); otherwise it joins the table first
  const bool dense_direct = g->dense.active && g->table.slots == nullptr;
  int64_t n_dense = 0, dense_empty = 0;
  if (g->dense.active && !dense_direct) B2_RETURN_NOT_OK(flush_dense(g, s));
  if (dense_direct) B2_RETURN_NOT_OK(dense_count(g, &n_dense, &dense_empty, s));
  if (!dense_direct && !g->table.slots) B2_RETURN_NOT_OK(fused_alloc(ctx, g->cap, &g->table, s));
  const int dense_null = dense_direct && g->dense.null_rows ? 1 : 0;
  const int64_t n = dense_direct ? n_dense + dense_null : static_cast<int64_t>(g->groups);
  const int kw = type_width(g->key_type);
  const int sum_type = sum_type_of(g->value_type);
  Temp keys(ctx, s), sums(ctx, s), counts(ctx, s), kbits(ctx, s), sbits(ctx, s);
  B2_RETURN_NOT_OK(keys.alloc((size_t)n * kw));
  B2_RETURN_NOT_OK(sums.alloc((size_t)n * 8));
  B2_RETURN_NOT_OK(counts.alloc((size_t)n * 8));
  int64_t key_nulls = 0, sum_nulls = 0;
  if (n > 0) {
    const size_t bb = bitmap_alloc_bytes(n);
    B2_RETURN_NOT_OK(kbits.alloc(bb));
    B2_RETURN_NOT_OK(sbits.alloc(bb));
    B2_CUDA(cudaMemsetAsync(kbits.ptr, 0xff, bb, s));
    B2_CUDA(cudaMemsetAsync(sbits.ptr, 0xff, bb, s));
    ScalarSlot slot(ctx);
    B2_RETURN_NOT_OK(slot.zero(s));
    if (dense_direct) {
      const auto& d = g->dense;
      dense_emit_kernel<<<grid_for((int64_t)d.range, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(
          d.sums, d.counts, d.exists, d.range, d.kmin, d.kflip, kw, keys.ptr, kbits.as<uint32_t>(), sums.as<unsigned long long>(),
          sbits.as<uint32_t>(), counts.as<long long>(), reinterpret_cast<unsigned long long*>(slot.dev()), dense_null, d.null_sum, d.null_cnt,
          (unsigned long long)n_dense);
    } else {
      fused_emit_kernel<<<grid_for((int64_t)g->cap + 2, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(
          g->table, kw, keys.ptr, kbits.as<uint32_t>(), sums.as<unsigned long long>(), sbits.as<uint32_t>(),
          counts.as<long long>(), reinterpret_cast<unsigned long long*>(slot.dev()));
    }
    B2_LAUNCHED();
    count_zero_bits_kernel<<<grid_for(n, kBlock * 32 * 4, kSMs * 4), kBlock, 0, s>>>(kbits.as<uint32_t>(), n, (int64_t)(bb / 4), slot.dev() + 1);
    B2_LAUNCHED();
    count_zero_bits_kernel<<<grid_for(n, kBlock * 32 * 4, kSMs * 4), kBlock, 0, s>>>(sbits.as<uint32_t>(), n, (int64_t)(bb / 4), slot.dev() + 2);
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(slot.fetch(s));
    const int64_t emitted = slot.host()[0] + dense_null;
    if (emitted != n) return set_error(B2_UNKNOWN_ERROR, "group-by emitted %lld of %lld groups", (long long)emitted, (long long)n);
    key_nulls = slot.host()[1];
    sum_nulls = slot.host()[2];
  }
  fill_out(out_keys, g->key_type, n, key_nulls, key_nulls ? kbits.release() : nullptr, keys.release());
  fill_out(out_sums, sum_type, n, sum_nulls, sum_nulls ? sbits.release() : nullptr, sums.release());
  fill_out(out_counts, B2_INT64, n, 0, nullptr, counts.release());
  return B2_OK;
}

}  // extern "C"
