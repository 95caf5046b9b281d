// sort_strings.cu -- a uint32 rank per row of a (large_)utf8 / (large_)binary column, so that every sort by a string
// key (sort_indices, sort_payload, the multi-key sort, select_k) is the numeric radix sort of sort_indices.cu run on
// the ranks.
//
// Replaces, for base-binary keys:
//   ArrayCompareSorter<BinaryType / LargeBinaryType / StringType / LargeStringType>   kernels/vector_array_sort.cc:144-178
//   (std::stable_sort with an indirect comparator over the string views; registration :494-500, 588-592)
// Order kept: byte-lexicographic on UNSIGNED bytes, a proper prefix first, NUL bytes ordinary bytes.  Ties, descending
// order and nulls are the numeric sort's business: equal strings get equal ranks, and the rank column carries the
// input's validity.
//
// Design: prefix radix sorting with tie refinement.  Positions are slots of the sorted order; the rank of a row is the
// sorted position of the first row of its run of equal strings (monotone, equal for equal strings, no compaction).
//   round 0  : every row gets the 64-bit key  (7 bytes from depth 0, big-endian, zero-padded) << 8 | min(len, 8);
//              a null row gets all ones, above every string key (a tag is at most 8).  The keys are read in row order
//              and sorted by the numeric radix sort; a run is a stretch of equal keys in sorted order.
//   refinement: only rows of an OPEN run (two or more rows, tag 8) take part.  Each open run first gets the longest
//              common prefix of its members with its first member from the depth already matched (aligned 8-byte
//              loads, atomicMin per run); then every member builds its next key at that depth, and the members are
//              sorted by (run, key) with the multi-key sort.  Runs split where the key changes; a row's rank is the
//              sorted position of its sub-run's first row.  Ranks of closed rows never change again.  One
//              device-to-host read per round: the number of rows still open.
// Why the 7+1 key is exact.  Let two strings be equal in their first d bytes and compare their keys at depth d.
//   * If the keys first differ in the data bytes, at byte i < 7: a string that ended before i is padded with zero
//     there, and it is a proper prefix of the other, so it sorts first either way; otherwise both hold real bytes at i
//     and the first differing byte decides, as it does for the strings.
//   * If only the tags differ, the data bytes are equal, so the string with the smaller tag ended inside the chunk and
//     is a proper prefix of the other: it sorts first, as its key does.
//   * Equal keys with a tag below 8 are equal strings: both ended at the same length with the same bytes.
// So the key order is the string order wherever keys differ, and only equal keys with tag 8 ("continues") are left
// undecided -- which is what lets each round close runs locally.
// Round bound.  After the common-prefix step, a run of identical strings reaches their end (its next key has tag 0 and
// closes it), and a run whose members differ splits at the first byte where some member differs from the first one,
// however deep that byte is.  So a long shared prefix costs one round, not one round per 7 bytes.
#include "sort_strings.h"

#include "common.cuh"

namespace b2 {

namespace {

constexpr int kRunItems = 8;
constexpr int kRunTile = kBlock * kRunItems;  // positions per CTA of the run-start scan
constexpr uint32_t kOpenDepth0 = 7;           // bytes every row of a run left open by round 0 shares

B2Array plain(int type, const void* data, int64_t length) {
  B2Array a{};
  a.type = type;
  a.data = data;
  a.length = length;
  return a;
}

template <typename OffT>
struct StrCol {
  const OffT* offs;      // advanced by the array's offset; entries index `bytes` directly
  const uint8_t* bytes;  // the character buffer (any alignment)
  __device__ __forceinline__ int64_t start(int64_t row) const { return static_cast<int64_t>(offs[row]); }
  __device__ __forceinline__ int64_t len(int64_t row) const { return static_cast<int64_t>(offs[row + 1]) - static_cast<int64_t>(offs[row]); }
};

__device__ __forceinline__ uint64_t bswap64(uint64_t v) {
  const uint32_t lo = static_cast<uint32_t>(v), hi = static_cast<uint32_t>(v >> 32);
  return (static_cast<uint64_t>(__byte_perm(lo, 0, 0x0123)) << 32) | __byte_perm(hi, 0, 0x0123);
}

// (up to 7 bytes at p, big-endian, zero-padded) << 8 | min(rem, 8); rem = bytes left in the string from p
__device__ __forceinline__ uint64_t chunk_key(const uint8_t* p, int64_t rem) {
  const int nb = rem < 7 ? static_cast<int>(rem) : 7;
  const uint64_t v = nb > 0 ? load_bytes8(p, nb) : 0;  // byte 7 of v is zero, so it lands in the tag byte as 0
  return bswap64(v) | static_cast<uint64_t>(rem < 8 ? rem : 8);
}

// length of the common prefix of a[0, lim) and b[0, lim)
__device__ __forceinline__ int64_t common_prefix(const uint8_t* a, const uint8_t* b, int64_t lim) {
  for (int64_t o = 0; o < lim; o += 8) {
    const int nb = lim - o >= 8 ? 8 : static_cast<int>(lim - o);
    const uint64_t x = load_bytes8(a + o, nb) ^ load_bytes8(b + o, nb);
    if (x) return o + ((__ffsll(static_cast<long long>(x)) - 1) >> 3);  // little-endian: lowest set byte = first difference
  }
  return lim;
}

// ---- round 0: one key per row, in row order ---------------------------------------------------------------------
template <typename OffT>
__global__ void __launch_bounds__(kBlock) rank_key0_kernel(StrCol<OffT> c, BitmapReader valid, int64_t n, uint64_t* __restrict__ keys) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock)
    keys[i] = valid.bit(i) ? chunk_key(c.bytes + c.start(i), c.len(i)) : ~0ull;
}

// ---- apply a sort: sorted keys and the rows at their positions ----------------------------------------------------
// order[j] = the element at sorted slot j; element i is row rows_in[i] (NULL: row i) and sits at position act[j] of the
// global order (NULL: j).
__global__ void __launch_bounds__(kBlock) rank_permute_kernel(const uint64_t* __restrict__ order, const uint32_t* __restrict__ act,
                                                              const uint64_t* __restrict__ key_in, const uint32_t* __restrict__ rows_in,
                                                              int64_t m, uint64_t* __restrict__ key_s, uint32_t* __restrict__ perm) {
  for (int64_t j = blockIdx.x * (int64_t)kBlock + threadIdx.x; j < m; j += (int64_t)gridDim.x * kBlock) {
    const uint64_t i = order[j];
    key_s[j] = key_in[i];
    perm[act ? act[j] : j] = rows_in ? rows_in[i] : static_cast<uint32_t>(i);
  }
}

// ---- run starts: a max-scan of head positions over the sorted elements ---------------------------------------------
struct RunArgs {
  const uint64_t* key;  // [m] keys in sorted order
  const uint32_t* grp;  // [m] run start before this round (the runs being split), NULL in round 0
  const uint32_t* pos;  // [m] global position of element j (ascending), NULL = j
  int64_t m;
  uint32_t* tile_last;  // [tiles] last head position of the tile, then the exclusive max over earlier tiles
  uint32_t* rs;         // [n] run start of every position
  uint32_t* open;       // [tiles * kRunTile / 32] bit j: element j is in an open run
  uint32_t* lcp;        // [n] set to ~0 at the first position of every open run
};

__device__ __forceinline__ bool is_head(const RunArgs& a, int64_t j) {
  if (j == 0 || j >= a.m) return true;
  return a.key[j] != a.key[j - 1] || (a.grp && a.grp[j] != a.grp[j - 1]);
}
__device__ __forceinline__ uint32_t pos_of(const RunArgs& a, int64_t j) { return a.pos ? a.pos[j] : static_cast<uint32_t>(j); }

// positions grow with j, so the largest head position in a tile is its last head (0 when it has none)
__global__ void __launch_bounds__(kBlock) run_tile_kernel(RunArgs a) {
  __shared__ uint32_t s_w[kWarpsPerBlock];
  const int64_t base = blockIdx.x * (int64_t)kRunTile;
  uint32_t best = 0;
#pragma unroll
  for (int k = 0; k < kRunItems; ++k) {
    const int64_t j = base + k * kBlock + threadIdx.x;
    if (j < a.m && is_head(a, j)) best = max(best, pos_of(a, j));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (lane_id() == 0) s_w[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t r = 0;
    for (int w = 0; w < kWarpsPerBlock; ++w) r = max(r, s_w[w]);
    a.tile_last[blockIdx.x] = r;
  }
}

// one CTA: exclusive max-scan of the tiles' last heads, in place
constexpr int kScanThreads = 1024;
__global__ void __launch_bounds__(kScanThreads) run_tile_scan_kernel(uint32_t* t, int64_t nt) {
  __shared__ uint32_t s_w[kScanThreads / 32];
  const int64_t per = (nt + kScanThreads - 1) / kScanThreads;
  const int64_t lo = threadIdx.x * per, hi = lo + per < nt ? lo + per : nt;
  uint32_t local = 0;
  for (int64_t i = lo; i < hi; ++i) local = max(local, t[i]);
  uint32_t incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane_id() >= (unsigned)o) incl = max(incl, v);
  }
  if (lane_id() == 31) s_w[threadIdx.x >> 5] = incl;
  __syncthreads();
  uint32_t run = __shfl_up_sync(0xffffffffu, incl, 1);  // exclusive over the lanes below
  if (lane_id() == 0) run = 0;
  for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) run = max(run, s_w[w]);
  for (int64_t i = lo; i < hi; ++i) {
    const uint32_t v = t[i];
    t[i] = run;
    run = max(run, v);
  }
}

// run start of every element (= position of the last head at or before it), open bits, lcp reset of open runs
__global__ void __launch_bounds__(kBlock) run_finish_kernel(RunArgs a) {
  __shared__ uint32_t s_w[kWarpsPerBlock];
  const int64_t base = blockIdx.x * (int64_t)kRunTile;
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  uint32_t carry = a.tile_last[blockIdx.x];
  for (int k = 0; k < kRunItems; ++k) {
    const int64_t j = base + k * kBlock + threadIdx.x;
    const bool in = j < a.m;
    const bool h = in && is_head(a, j);
    const uint32_t p = in ? pos_of(a, j) : 0;
    uint32_t v = h ? p : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= (unsigned)o) v = max(v, t);
    }
    if (lane == 31) s_w[warp] = v;
    __syncthreads();
    uint32_t before = carry, total = carry;
#pragma unroll
    for (int w = 0; w < kWarpsPerBlock; ++w) {
      if (w < (int)warp) before = max(before, s_w[w]);
      total = max(total, s_w[w]);
    }
    bool open = false;
    if (in) {
      a.rs[p] = max(before, v);
      open = (a.key[j] & 0xff) == 8 && !(h && is_head(a, j + 1));
      if (open && h) a.lcp[p] = ~0u;
    }
    const unsigned bits = __ballot_sync(0xffffffffu, open);
    if (lane == 0) a.open[(base + k * kBlock) / 32 + warp] = bits;
    carry = total;
    __syncthreads();  // s_w is rewritten by the next slice
  }
}

// ---- refinement ------------------------------------------------------------------------------------------------
// element i = the row at open position act[i]; its run starts at g.  Every member but the first lowers the run's common
// prefix (from the matched depth) to what it shares with the first member.
template <typename OffT>
__global__ void __launch_bounds__(kBlock) rank_lcp_kernel(StrCol<OffT> c, const uint32_t* __restrict__ act, int64_t m,
                                                          const uint32_t* __restrict__ perm, const uint32_t* __restrict__ rs,
                                                          const uint64_t* __restrict__ depth, uint32_t* __restrict__ rows_i,
                                                          uint32_t* __restrict__ g_i, uint32_t* lcp) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < m; i += (int64_t)gridDim.x * kBlock) {
    const uint32_t p = act[i];
    const uint32_t row = perm[p], g = rs[p];
    rows_i[i] = row;
    g_i[i] = g;
    if (p == g) continue;
    const uint32_t first = perm[g];
    const int64_t d = depth ? static_cast<int64_t>(depth[i]) : kOpenDepth0;
    int64_t lim = c.len(row) - d;
    const int64_t lf = c.len(first) - d;
    if (lf < lim) lim = lf;
    if (lim > 0xffffffffll) lim = 0xffffffffll;  // a longer prefix is skipped in the next round
    const int64_t l = common_prefix(c.bytes + c.start(row) + d, c.bytes + c.start(first) + d, lim);
    atomicMin(lcp + g, static_cast<uint32_t>(l));
  }
}

// the next key of every element, at the matched depth plus its run's common prefix
template <typename OffT>
__global__ void __launch_bounds__(kBlock) rank_chunk_kernel(StrCol<OffT> c, int64_t m, const uint32_t* __restrict__ rows_i,
                                                            const uint32_t* __restrict__ g_i, const uint32_t* __restrict__ lcp,
                                                            const uint64_t* __restrict__ depth_in, uint64_t* __restrict__ depth_out,
                                                            uint64_t* __restrict__ key_i) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < m; i += (int64_t)gridDim.x * kBlock) {
    const uint32_t row = rows_i[i];
    const int64_t d = (depth_in ? static_cast<int64_t>(depth_in[i]) : kOpenDepth0) + lcp[g_i[i]];
    key_i[i] = chunk_key(c.bytes + c.start(row) + d, c.len(row) - d);
    depth_out[i] = static_cast<uint64_t>(d + 7);  // what the members of a run this key leaves open share
  }
}

__global__ void __launch_bounds__(kBlock) rank_scatter_kernel(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ rs,
                                                              int64_t n, uint32_t* __restrict__ rank) {
  for (int64_t p = blockIdx.x * (int64_t)kBlock + threadIdx.x; p < n; p += (int64_t)gridDim.x * kBlock) rank[perm[p]] = rs[p];
}

// run starts and open bits of m sorted elements; bits gets a B2_BOOL-ready bitmap of m bits
int run_scan(B2Context* ctx, RunArgs a, Temp* bits, cudaStream_t s) {
  const int64_t tiles = (a.m + kRunTile - 1) / kRunTile;
  Temp tl(ctx, s);
  B2_RETURN_NOT_OK(tl.alloc(sizeof(uint32_t) * (size_t)tiles));
  B2_RETURN_NOT_OK(bits->alloc((size_t)tiles * (kRunTile / 8) + 8));
  a.tile_last = tl.as<uint32_t>();
  a.open = bits->as<uint32_t>();
  run_tile_kernel<<<(unsigned)tiles, kBlock, 0, s>>>(a);
  B2_LAUNCHED();
  run_tile_scan_kernel<<<1, kScanThreads, 0, s>>>(a.tile_last, tiles);
  B2_LAUNCHED();
  run_finish_kernel<<<(unsigned)tiles, kBlock, 0, s>>>(a);
  B2_LAUNCHED();
  return B2_OK;
}

template <typename OffT>
int rank_typed(B2Context* ctx, const B2Array* values, uint32_t* rank, cudaStream_t s) {
  const int64_t n = values->length;
  const int grid = grid_for(n, kBlock * 4, ctx->sm_count * 8);
  StrCol<OffT> c{static_cast<const OffT*>(values->data) + values->offset, static_cast<const uint8_t*>(values->data2)};
  Temp perm(ctx, s), rs(ctx, s), lcp(ctx, s);
  B2_RETURN_NOT_OK(perm.alloc(sizeof(uint32_t) * (size_t)n));
  B2_RETURN_NOT_OK(rs.alloc(sizeof(uint32_t) * (size_t)n));
  B2_RETURN_NOT_OK(lcp.alloc(sizeof(uint32_t) * (size_t)n));
  PoolArray act(ctx, s), depth(ctx, s);  // open positions (uint32, ascending) and the depth their runs matched (uint64)

  // round 0
  {
    Temp keys(ctx, s), key_s(ctx, s), bits(ctx, s);
    B2_RETURN_NOT_OK(keys.alloc(sizeof(uint64_t) * (size_t)n));
    rank_key0_kernel<OffT><<<grid, kBlock, 0, s>>>(c, BitmapReader(values->null_count == 0 ? nullptr : values->validity, values->offset, n),
                                                  n, keys.as<uint64_t>());
    B2_LAUNCHED();
    PoolArray order(ctx, s);
    const B2Array ka = plain(B2_UINT64, keys.ptr, n);
    B2_RETURN_NOT_OK(b2_sort_indices(ctx, &ka, 0, 1, &order.a, s));
    B2_RETURN_NOT_OK(key_s.alloc(sizeof(uint64_t) * (size_t)n));
    rank_permute_kernel<<<grid, kBlock, 0, s>>>(static_cast<const uint64_t*>(order.a.data), nullptr, keys.as<uint64_t>(), nullptr, n,
                                                key_s.as<uint64_t>(), perm.as<uint32_t>());
    B2_LAUNCHED();
    RunArgs ra{};
    ra.key = key_s.as<uint64_t>();
    ra.m = n;
    ra.rs = rs.as<uint32_t>();
    ra.lcp = lcp.as<uint32_t>();
    B2_RETURN_NOT_OK(run_scan(ctx, ra, &bits, s));
    const B2Array mask = plain(B2_BOOL, bits.ptr, n);
    B2_RETURN_NOT_OK(b2_filter_indices(ctx, &mask, 0, &act.a, s));
    if (act.a.type == B2_UINT16) {  // b2_filter_indices narrows the indices of masks up to 65535 rows
      PoolArray wide(ctx, s);
      B2CastOptions to_u32{B2_UINT32, 1, 1, 0};
      B2_RETURN_NOT_OK(b2_cast_numeric(ctx, &act.a, &to_u32, &wide.a, s));
      act.take_from(wide);
    }
  }

  // refinement rounds, until no run is open
  while (act.a.length > 0) {
    const int64_t m = act.a.length;
    const int gm = grid_for(m, kBlock * 4, ctx->sm_count * 8);
    const uint32_t* ap = static_cast<const uint32_t*>(act.a.data) + act.a.offset;
    const uint64_t* din = depth.a.data ? static_cast<const uint64_t*>(depth.a.data) + depth.a.offset : nullptr;
    Temp rows_i(ctx, s), g_i(ctx, s), key_i(ctx, s), dout(ctx, s), key_s(ctx, s), bits(ctx, s);
    B2_RETURN_NOT_OK(rows_i.alloc(sizeof(uint32_t) * (size_t)m));
    B2_RETURN_NOT_OK(g_i.alloc(sizeof(uint32_t) * (size_t)m));
    B2_RETURN_NOT_OK(key_i.alloc(sizeof(uint64_t) * (size_t)m));
    B2_RETURN_NOT_OK(dout.alloc(sizeof(uint64_t) * (size_t)m));
    rank_lcp_kernel<OffT><<<gm, kBlock, 0, s>>>(c, ap, m, perm.as<uint32_t>(), rs.as<uint32_t>(), din, rows_i.as<uint32_t>(),
                                               g_i.as<uint32_t>(), lcp.as<uint32_t>());
    B2_LAUNCHED();
    rank_chunk_kernel<OffT><<<gm, kBlock, 0, s>>>(c, m, rows_i.as<uint32_t>(), g_i.as<uint32_t>(), lcp.as<uint32_t>(), din,
                                                 dout.as<uint64_t>(), key_i.as<uint64_t>());
    B2_LAUNCHED();
    // stable sort by (run, key): the runs stay where they are, their members are reordered inside them
    PoolArray order(ctx, s);
    const B2Array ks[2] = {plain(B2_UINT32, g_i.ptr, m), plain(B2_UINT64, key_i.ptr, m)};
    const int32_t asc[2] = {0, 0};
    B2_RETURN_NOT_OK(b2_sort_indices_multi(ctx, ks, 2, asc, 1, &order.a, s));
    B2_RETURN_NOT_OK(key_s.alloc(sizeof(uint64_t) * (size_t)m));
    rank_permute_kernel<<<gm, kBlock, 0, s>>>(static_cast<const uint64_t*>(order.a.data), ap, key_i.as<uint64_t>(), rows_i.as<uint32_t>(),
                                              m, key_s.as<uint64_t>(), perm.as<uint32_t>());
    B2_LAUNCHED();
    order.reset();
    // the sort keeps the runs in place, so g_i is already the run of sorted element j
    RunArgs ra{};
    ra.key = key_s.as<uint64_t>();
    ra.grp = g_i.as<uint32_t>();
    ra.pos = ap;
    ra.m = m;
    ra.rs = rs.as<uint32_t>();
    ra.lcp = lcp.as<uint32_t>();
    B2_RETURN_NOT_OK(run_scan(ctx, ra, &bits, s));
    // dout[j] is the depth of element j's run too: every member of a run wrote the same value
    const B2Array mask = plain(B2_BOOL, bits.ptr, m);
    PoolArray nact(ctx, s), ndepth(ctx, s);
    B2_RETURN_NOT_OK(b2_filter(ctx, &act.a, &mask, 0, &nact.a, s));
    if (nact.a.length > 0) {
      const B2Array da = plain(B2_UINT64, dout.ptr, m);
      B2_RETURN_NOT_OK(b2_filter(ctx, &da, &mask, 0, &ndepth.a, s));
    }
    act.take_from(nact);
    depth.take_from(ndepth);
  }

  rank_scatter_kernel<<<grid, kBlock, 0, s>>>(perm.as<uint32_t>(), rs.as<uint32_t>(), n, rank);
  B2_LAUNCHED();
  return B2_OK;
}

}  // namespace

int string_rank(B2Context* ctx, const B2Array* values, Temp* rank, B2Array* out, cudaStream_t s) {
  if (!type_is_binary_like(values->type)) return set_error(B2_INVALID, "string_rank: type id %d is not utf8 / binary", values->type);
  if (values->length < 0 || values->offset < 0) return set_error(B2_INVALID, "negative length/offset");
  const int64_t n = values->length;
  if (n >= (1ll << 32) - 8192)  // positions and row numbers are uint32
    return set_error(B2_NOT_IMPLEMENTED, "sort_indices: arrays of 2^32 rows or more must be sorted as chunks");
  B2_CUDA(cudaSetDevice(ctx->device));
  // the rank column shares the input's bitmap: whole bytes of the offset move into the pointer, the rest stays an offset
  const int64_t lead = values->offset & 7;
  B2_RETURN_NOT_OK(rank->alloc(sizeof(uint32_t) * (size_t)(n + lead)));
  *out = B2Array{};
  out->type = B2_UINT32;
  out->data = rank->ptr;
  out->validity = values->validity ? static_cast<const uint8_t*>(values->validity) + (values->offset >> 3) : nullptr;
  out->offset = lead;
  out->length = n;
  out->null_count = values->validity ? values->null_count : 0;
  if (n == 0) return B2_OK;
  uint32_t* r = rank->as<uint32_t>() + lead;
  return offset_width(values->type) == 8 ? rank_typed<int64_t>(ctx, values, r, s) : rank_typed<int32_t>(ctx, values, r, s);
}

}  // namespace b2
