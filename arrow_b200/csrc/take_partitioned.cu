// take_partitioned.cu -- partitioned gather for large random fixed-width Take (b2_take, b2_take_cast_arith).
//
// A gather in row order makes one random DRAM access per row once the values are far larger than L2: the H100 sustains
// about 28 G of those per second (bench_micro/gather_probe.cu, 8 GB table), a quarter of its streaming bandwidth.  If the
// rows are first grouped by the band of `values` they read, each band is gathered while it sits in L2 and `values` is
// read from DRAM about once: with 256 bands of 32 MB the same probe sustains 74 G gathers/s.  Four passes:
//
//   H  histogram: one read of the indices counts the rows of each bucket (bucket = j >> shift, < 256) and finds the
//      first out-of-range valid index (atomicMin, the direct kernels' rule).  Null and out-of-range indices count
//      as index 0.
//   A  partition: onesweep-style -- 4096-row tiles claimed through an atomic ticket are ranked stably by bucket
//      (ballot matching, as sort_indices.cu's onesweep_kernel), the tile's bucket counts published for a decoupled
//      look-back, and the uint32 index j written in bucket order; each row's uint16 tile-local position (where the
//      ranking put it) is written in row order.  The look-back cells stay alive for pass C.
//   B  banded gather: positions in bucket order, tiles claimed in order through a ticket so the whole GPU works on
//      about one band at a time; gathers values[j] and its validity bit, casts to the output type, writes both in
//      bucket order.  Prefetching the next band into L2 (cp.async.bulk.prefetch.L2) measured slower, so there is none.
//   C  restore: the mirror image of A, without ranking again.  A tile takes its bucket counts from the look-back cells
//      of tiles t and t - 1, reads its runs of gathered values through shared memory, puts them back in row order with
//      A's positions and finishes: masks null indices, applies the arithmetic with `other` (fused) and writes the
//      result and its bitmap in row order.
//
// B and C issue each phase's global loads together, into registers or shared memory, before the first store that
// needs them: one memory round trip per phase rather than one per item.
//
// Results are bit-identical to the direct kernels of selection_take.cu.  Limits: n < 2^30 (30-bit look-back counts),
// values_length <= 2^32 (indices are carried as uint32).  Temporaries: n * 6 bytes (n * 14 for 8-byte results) + n / 8 +
// 1 KB per tile of look-back cells.
#include <type_traits>

#include "elementwise.cuh"
#include "take_partitioned.h"

namespace b2 {

constexpr int kPartThreads = 256;
constexpr int kPartWarps = kPartThreads / 32;
constexpr int kPartItems = 16;
constexpr int kPartTile = kPartThreads * kPartItems;  // 4096 rows
constexpr int kBucketBits = 8;
constexpr int kBuckets = 1 << kBucketBits;  // == kPartThreads: thread b owns bucket b
constexpr uint32_t kCellAgg = 1u << 30, kCellIncl = 2u << 30, kCellMask = (1u << 30) - 1u;

template <typename Idx>
__device__ __forceinline__ uint64_t index_u64(Idx raw) {
  return std::is_unsigned<Idx>::value ? static_cast<uint64_t>(raw) : static_cast<uint64_t>(static_cast<int64_t>(raw));
}

// exclusive scan of one value per thread over the 256 threads of the block
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* s_warp_tot) {
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  uint32_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) s_warp_tot[warp] = incl;
  __syncthreads();
  uint32_t woff = 0;
#pragma unroll
  for (int w = 0; w < kPartWarps; ++w)
    if (w < (int)warp) woff += s_warp_tot[w];
  __syncthreads();  // s_warp_tot is free again
  return woff + incl - v;
}

// Stable rank of the tile's items by bucket.  Item j of lane l in warp w is tile element w*512 + j*32 + l; lanes with the
// same bucket find each other with one ballot per bucket bit.  Afterwards the tile-local position of item j is
// s_cnt[warp * 256 + bkt[j]] + rank[j]; thread b returns bucket b's item count in the tile (*count) and the tile-local
// start of its run (*bin_off).  A bucket's items sit in tile-element order within its run (the layout pass C rebuilds
// from the bucket counts alone).
__device__ __forceinline__ void rank_tile(const unsigned (&bkt)[kPartItems], uint16_t (&rank)[kPartItems], uint32_t* s_cnt,
                                          uint32_t* s_warp_tot, uint32_t* count, uint32_t* bin_off) {
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < kPartWarps * kBuckets; i += kPartThreads) s_cnt[i] = 0;
  __syncthreads();
  uint32_t* wc = s_cnt + warp * kBuckets;
  const unsigned lt = lanemask_lt();
#pragma unroll
  for (int j = 0; j < kPartItems; ++j) {
    unsigned peers = 0xffffffffu;
#pragma unroll
    for (int b = 0; b < kBucketBits; ++b) {
      const bool bit = (bkt[j] >> b) & 1u;
      const unsigned bal = __ballot_sync(0xffffffffu, bit);
      peers &= bit ? bal : ~bal;
    }
    const int leader = __ffs(peers) - 1;
    unsigned prev = 0;
    if ((int)lane == leader) {
      prev = wc[bkt[j]];
      wc[bkt[j]] = prev + __popc(peers);
    }
    prev = __shfl_sync(0xffffffffu, prev, leader);
    rank[j] = static_cast<uint16_t>(prev + __popc(peers & lt));
    __syncwarp();  // the next item's leader may be another lane reading the counter just written
  }
  __syncthreads();
  uint32_t run = 0;
#pragma unroll
  for (int w = 0; w < kPartWarps; ++w) {
    const uint32_t c = s_cnt[w * kBuckets + tid];
    s_cnt[w * kBuckets + tid] = run;
    run += c;
  }
  const uint32_t off = block_excl_scan(run, s_warp_tot);
#pragma unroll
  for (int w = 0; w < kPartWarps; ++w) s_cnt[w * kBuckets + tid] += off;
  __syncthreads();
  *count = run;
  *bin_off = off;
}

// ---- pass H ---------------------------------------------------------------------------------------------------------
template <typename Idx>
__global__ void __launch_bounds__(kPartThreads) part_hist_kernel(PartTakeArgs a, uint32_t* __restrict__ hist) {
  __shared__ uint32_t s_h[kBuckets];
  s_h[threadIdx.x] = 0;
  __syncthreads();
  const Idx* __restrict__ idx = static_cast<const Idx*>(a.indices);
  const uint64_t vlen = static_cast<uint64_t>(a.values_length);
  constexpr int kItems = 4;
  for (int64_t t = (int64_t)blockIdx.x * kPartThreads * kItems; t < a.n; t += (int64_t)gridDim.x * kPartThreads * kItems) {
    Idx raw[kItems];
    uint32_t ivw[kItems];
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      const int64_t i = t + k * kPartThreads + threadIdx.x;
      raw[k] = i < a.n ? __ldcs(idx + i) : Idx(0);
      ivw[k] = a.idx_valid.word32((t + k * kPartThreads + (threadIdx.x & ~31u)) >> 5);  // the warp's 32 rows
    }
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      const int64_t i = t + k * kPartThreads + threadIdx.x;
      if (i >= a.n) break;
      const uint64_t j = index_u64(raw[k]);
      const bool iv = (ivw[k] >> lane_id()) & 1u;
      unsigned b = 0;
      if (iv) {
        if (j < vlen) b = static_cast<unsigned>(j >> a.shift);
        else atomicMin(a.first_bad, static_cast<unsigned long long>(i));
      }
      atomicAdd(&s_h[b], 1u);
    }
  }
  __syncthreads();
  if (s_h[threadIdx.x]) atomicAdd(&hist[threadIdx.x], s_h[threadIdx.x]);
}

// ---- pass A ---------------------------------------------------------------------------------------------------------
template <typename Idx>
__global__ void __launch_bounds__(kPartThreads) part_scatter_kernel(PartTakeArgs a, const uint32_t* __restrict__ hist,
                                                                    uint32_t* __restrict__ part, uint16_t* __restrict__ pos,
                                                                    uint32_t* lookback, uint32_t* ticket) {
  __shared__ uint32_t s_j[kPartTile];
  __shared__ __align__(16) uint16_t s_lp[kPartTile];
  __shared__ uint32_t s_cnt[kPartWarps * kBuckets];
  __shared__ uint32_t s_gbase[kBuckets];
  __shared__ uint64_t s_iv[kPartTile / 64];
  __shared__ uint32_t s_warp_tot[kPartWarps];
  __shared__ uint32_t s_tile;
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_tile = atomicAdd(ticket, 1u);
  __syncthreads();
  const uint32_t tile = s_tile;
  const uint32_t base = tile * kPartTile;
  const uint32_t tile_n = static_cast<uint32_t>(a.n - base) < (uint32_t)kPartTile ? static_cast<uint32_t>(a.n - base) : (uint32_t)kPartTile;
  const Idx* __restrict__ idx = static_cast<const Idx*>(a.indices);
  const uint64_t vlen = static_cast<uint64_t>(a.values_length);

  Idx raw[kPartItems];
#pragma unroll
  for (int j = 0; j < kPartItems; ++j) {
    const uint32_t i = warp * (32 * kPartItems) + j * 32 + lane;
    raw[j] = i < tile_n ? __ldcs(idx + base + i) : Idx(0);
  }
  if (tid < kPartTile / 64) s_iv[tid] = a.idx_valid.word((base >> 6) + tid);
  __syncthreads();
  const uint32_t* iv32 = reinterpret_cast<const uint32_t*>(s_iv);
  unsigned bkt[kPartItems];
  uint32_t jj[kPartItems];
#pragma unroll
  for (int j = 0; j < kPartItems; ++j) {
    const uint32_t i = warp * (32 * kPartItems) + j * 32 + lane;
    const bool iv = (iv32[i >> 5] >> lane) & 1u;
    const uint64_t u = index_u64(raw[j]);
    jj[j] = (iv && u < vlen) ? static_cast<uint32_t>(u) : 0u;  // null / out of range: index 0, masked (or raised) later
    bkt[j] = i < tile_n ? jj[j] >> a.shift : kBuckets - 1;     // padding sorts last
  }
  uint16_t rank[kPartItems];
  uint32_t count, bin_off;
  rank_tile(bkt, rank, s_cnt, s_warp_tot, &count, &bin_off);
  if (tid == kBuckets - 1) count -= kPartTile - tile_n;
  const uint32_t start = block_excl_scan(hist[tid], s_warp_tot);
  volatile uint32_t* lb = lookback;
  lb[(size_t)tile * kBuckets + tid] = (tile == 0 ? kCellIncl : kCellAgg) | count;
  // stage in bucket order first: the predecessors get time to publish before the look-back has to wait for them
#pragma unroll
  for (int j = 0; j < kPartItems; ++j) {
    const uint32_t lp = s_cnt[warp * kBuckets + bkt[j]] + rank[j];
    s_j[lp] = jj[j];
    s_lp[warp * (32 * kPartItems) + j * 32 + lane] = static_cast<uint16_t>(lp);
  }
  uint32_t excl = 0;
  if (tile > 0) {
    excl = lookback_exclusive(lb + tid, tile, kBuckets);
    lb[(size_t)tile * kBuckets + tid] = kCellIncl | (excl + count);
  }
  s_gbase[tid] = start + excl - bin_off;
  __syncthreads();
  // the positions of the whole tile, padding included (the buffer holds whole tiles), as 16-byte stores
  uint4* pos4 = reinterpret_cast<uint4*>(pos + base);
  __stcs(pos4 + tid, reinterpret_cast<const uint4*>(s_lp)[tid]);
  __stcs(pos4 + kPartThreads + tid, reinterpret_cast<const uint4*>(s_lp)[kPartThreads + tid]);
#pragma unroll
  for (int j = 0; j < kPartItems; ++j) {
    const uint32_t p = j * kPartThreads + tid;
    if (p < tile_n) {
      const uint32_t v = s_j[p];
      __stcs(part + s_gbase[v >> a.shift] + p, v);  // every real row's bucket is its j >> shift (index 0 for the masked ones)
    }
  }
}

// ---- pass B ---------------------------------------------------------------------------------------------------------
// A coherent ld.global: ptxas may not move it past a store that could alias it, so a batch of them stays ahead of the
// stores.  ptxas sinks ld.global.nc (__ldg) gathers next to the store that consumes each, and they then wait on one
// another.
template <typename T>
__device__ __forceinline__ T ld_before_stores(const T* p) {
  uint64_t v;
  if constexpr (sizeof(T) == 1) {
    uint32_t w;
    asm volatile("ld.global.u8 %0, [%1];" : "=r"(w) : "l"(p));
    v = w;
  } else if constexpr (sizeof(T) == 4) {
    uint32_t w;
    asm volatile("ld.global.u32 %0, [%1];" : "=r"(w) : "l"(p));
    v = w;
  } else {
    static_assert(sizeof(T) == 8, "1-, 4- or 8-byte loads");
    asm volatile("ld.global.u64 %0, [%1];" : "=l"(v) : "l"(p));
  }
  T out;
  memcpy(&out, &v, sizeof(T));  // little-endian: the loaded bytes are the low ones
  return out;
}

template <typename VT, typename OT>
__global__ void __launch_bounds__(kPartThreads) part_gather_kernel(PartTakeArgs a, const uint32_t* part, OT* g,
                                                                   uint32_t* __restrict__ gvalid,
                                                                   uint32_t* ticket) {
  __shared__ uint32_t s_tile;
  if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
  __syncthreads();
  const int64_t p0 = (int64_t)s_tile * kPartTile;
  const VT* __restrict__ vals = static_cast<const VT*>(a.values);
  uint32_t j[kPartItems];
#pragma unroll
  for (int k = 0; k < kPartItems; ++k) {
    const int64_t p = p0 + k * kPartThreads + threadIdx.x;
    j[k] = p < a.n ? __ldcs(part + p) : 0u;
  }
  // the value gathers and their validity probes in one batch, before the first store
  const uint8_t* vbits = reinterpret_cast<const uint8_t*>(a.values_valid.base);
  VT v[kPartItems];
  uint32_t vb[kPartItems];
#pragma unroll
  for (int k = 0; k < kPartItems; ++k) {
    v[k] = ld_before_stores(vals + j[k]);
    const int64_t bit = a.values_valid.bit0 + j[k];
    vb[k] = gvalid ? ld_before_stores(vbits + (bit >> 3)) >> (bit & 7) : 1u;
  }
#pragma unroll
  for (int k = 0; k < kPartItems; ++k) {
    const int64_t p = p0 + k * kPartThreads + threadIdx.x;
    if (p < a.n) __stcs(g + p, static_cast<OT>(v[k]));
    if (gvalid) {
      const unsigned w = __ballot_sync(0xffffffffu, p < a.n && (vb[k] & 1u));
      if (lane_id() == 0 && p < a.n) gvalid[p >> 5] = w;
    }
  }
}

// ---- pass C ---------------------------------------------------------------------------------------------------------
// OP: B2_ADD / B2_SUBTRACT / B2_MULTIPLY for b2_take_cast_arith, -1 for a plain take.
template <typename OT, int OP>
__global__ void __launch_bounds__(kPartThreads) part_restore_kernel(PartTakeArgs a, const uint32_t* __restrict__ hist,
                                                                    const uint16_t* __restrict__ pos,
                                                                    const uint32_t* __restrict__ lookback,
                                                                    const OT* __restrict__ g,
                                                                    const uint32_t* __restrict__ gvalid) {
  constexpr bool kFused = OP >= 0;
  __shared__ OT s_val[kPartTile];
  __shared__ __align__(16) uint16_t s_lp[kPartTile];  // each row's tile-local position (pass A)
  __shared__ uint8_t s_bkt[kPartTile];                // the bucket of each tile-local position
  __shared__ uint32_t s_gv[kPartTile / 32];           // gathered validity by tile-local position
  __shared__ uint64_t s_iv[kPartTile / 64], s_ov[kPartTile / 64];  // index / `other` validity by row
  __shared__ uint32_t s_gbase[kBuckets];
  __shared__ uint32_t s_warp_tot[kPartWarps];
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t tile = blockIdx.x;
  const uint32_t base = tile * kPartTile;
  const uint32_t tile_n = static_cast<uint32_t>(a.n - base) < (uint32_t)kPartTile ? static_cast<uint32_t>(a.n - base) : (uint32_t)kPartTile;
  // everything that does not depend on where the runs are: positions, bucket counts, bitmaps
  const uint4* pos4 = reinterpret_cast<const uint4*>(pos + base);
  const uint4 q0 = __ldcs(pos4 + tid), q1 = __ldcs(pos4 + kPartThreads + tid);
  const uint32_t incl = lookback[(size_t)tile * kBuckets + tid] & kCellMask;
  const uint32_t prev = tile > 0 ? lookback[(size_t)(tile - 1) * kBuckets + tid] & kCellMask : 0u;
  const uint32_t h = hist[tid];
  uint64_t bits = 0;
  if (tid < kPartTile / 64) bits = a.idx_valid.word((base >> 6) + tid);
  else if (kFused && tid < kPartTile / 32) bits = a.other_valid.word((base >> 6) + tid - kPartTile / 64);
  reinterpret_cast<uint4*>(s_lp)[tid] = q0;
  reinterpret_cast<uint4*>(s_lp)[kPartThreads + tid] = q1;
  if (tid < kPartTile / 64) s_iv[tid] = bits;
  else if (kFused && tid < kPartTile / 32) s_ov[tid - kPartTile / 64] = bits;
  // thread b owns bucket b: its run is [bin_off, bin_off + count) of the tile and starts at gathered element
  // start + prev, where pass A left it
  const uint32_t count = incl - prev;
  const uint32_t start = block_excl_scan(h, s_warp_tot);
  const uint32_t bin_off = block_excl_scan(count, s_warp_tot);
  s_gbase[tid] = start + prev - bin_off;
  for (uint32_t k = 0; k < count; ++k) s_bkt[bin_off + k] = static_cast<uint8_t>(tid);
  __syncthreads();
  // read the tile's runs of gathered values in bucket order, consecutive threads on consecutive elements of a run:
  // every load of the phase is issued before the first shared store
  OT v[kPartItems];
  uint32_t src[kPartItems], gw[kPartItems];
#pragma unroll
  for (int k = 0; k < kPartItems; ++k) {
    const uint32_t p = k * kPartThreads + tid;
    src[k] = s_gbase[s_bkt[p]] + p;  // past tile_n: a padding position, never read
    v[k] = p < tile_n ? g[src[k]] : OT{};
    gw[k] = (gvalid && p < tile_n) ? gvalid[src[k] >> 5] : ~0u;
  }
#pragma unroll
  for (int k = 0; k < kPartItems; ++k) {
    s_val[k * kPartThreads + tid] = v[k];
    const unsigned w = __ballot_sync(0xffffffffu, (gw[k] >> (src[k] & 31)) & 1u);
    if (lane == 0) s_gv[k * kPartWarps + warp] = w;
  }
  __syncthreads();
  OT* __restrict__ out = static_cast<OT*>(a.out);
  const OT* __restrict__ other = static_cast<const OT*>(a.other);
  const OT oscalar = static_cast<OT>(a.other_scalar);
  const uint32_t* iv32 = reinterpret_cast<const uint32_t*>(s_iv);
  const uint32_t* ov32 = reinterpret_cast<const uint32_t*>(s_ov);
  OT x[kPartItems];
  if (kFused) {
#pragma unroll
    for (int j = 0; j < kPartItems; ++j) {
      const uint32_t i = warp * (32 * kPartItems) + j * 32 + lane;
      x[j] = (other && i < tile_n) ? other[base + i] : oscalar;
    }
  }
  int64_t valid_local = 0;
#pragma unroll
  for (int j = 0; j < kPartItems; ++j) {
    const uint32_t i = warp * (32 * kPartItems) + j * 32 + lane;
    const uint32_t lp = s_lp[i];
    const bool iv = (iv32[i >> 5] >> lane) & 1u;
    const OT y = iv ? s_val[lp] : OT{};
    bool ok = i < tile_n && iv && ((s_gv[lp >> 5] >> (lp & 31)) & 1u);
    if (kFused) {
      x[j] = fused_apply<OT>(OP, y, x[j]);
      ok = ok && ((ov32[i >> 5] >> lane) & 1u);
    } else {
      x[j] = y;
    }
    if (a.out_validity) {
      const unsigned w = __ballot_sync(0xffffffffu, ok);
      if (lane == 0 && i < tile_n) {
        a.out_validity[(base + i) >> 5] = w;
        valid_local += __popc(w);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < kPartItems; ++j) {
    const uint32_t i = warp * (32 * kPartItems) + j * 32 + lane;
    if (i < tile_n) __stcs(out + base + i, x[j]);
  }
  if (a.out_validity) {
    const int64_t s = block_sum<kPartThreads>(valid_local);
    if (tid == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(a.valid_count), (unsigned long long)s);
  }
}

// ---- host -----------------------------------------------------------------------------------------------------------
template <typename OT, int OP>
static void launch_restore(const PartTakeArgs& a, uint32_t n_tiles, const uint32_t* hist, const uint16_t* pos,
                           const uint32_t* lookback, const OT* gathered, const uint32_t* gv, cudaStream_t s) {
  part_restore_kernel<OT, OP><<<n_tiles, kPartThreads, 0, s>>>(a, hist, pos, lookback, gathered, gv);
}

template <typename Idx, typename VT, typename OT, bool FUSED>
static int run_passes(B2Context* ctx, const PartTakeArgs& a, cudaStream_t s, bool* ran) {
  *ran = false;
  const int64_t n = a.n;
  const uint32_t n_tiles = static_cast<uint32_t>((n + kPartTile - 1) / kPartTile);
  const size_t lb_bytes = (size_t)n_tiles * kBuckets * sizeof(uint32_t);
  const size_t misc_bytes = kBuckets * sizeof(uint32_t) + 2 * sizeof(uint32_t);  // hist + two tickets
  // a 4-byte result overwrites the index it was gathered through (pass B reads part[p] before it writes g[p])
  constexpr bool kInPlace = sizeof(OT) == sizeof(uint32_t);
  Temp part(ctx, s), pos(ctx, s), g(ctx, s), gvalid(ctx, s), cells(ctx, s);
  if (part.alloc(sizeof(uint32_t) * (size_t)n) != B2_OK || pos.alloc(sizeof(uint16_t) * n_tiles * kPartTile) != B2_OK ||
      (!kInPlace && g.alloc(sizeof(OT) * (size_t)n) != B2_OK) || cells.alloc(lb_bytes + misc_bytes) != B2_OK ||
      ((a.values_valid.base != nullptr) && gvalid.alloc(bitmap_alloc_bytes(n)) != B2_OK))
    return B2_OK;  // the direct kernels run instead
  *ran = true;
  uint32_t* lookback = cells.as<uint32_t>();
  uint32_t* hist = lookback + (size_t)n_tiles * kBuckets;
  uint32_t* tickets = hist + kBuckets;
  B2_CUDA(cudaMemsetAsync(cells.ptr, 0, lb_bytes + misc_bytes, s));
  part_hist_kernel<Idx><<<grid_for(n, kPartThreads * 4, ctx->sm_count * 8), kPartThreads, 0, s>>>(a, hist);
  B2_LAUNCHED();
  part_scatter_kernel<Idx><<<n_tiles, kPartThreads, 0, s>>>(a, hist, part.as<uint32_t>(), pos.as<uint16_t>(), lookback, tickets);
  B2_LAUNCHED();
  uint32_t* gv = (a.values_valid.base != nullptr) ? gvalid.as<uint32_t>() : nullptr;
  OT* gathered = kInPlace ? part.as<OT>() : g.as<OT>();
  part_gather_kernel<VT, OT><<<n_tiles, kPartThreads, 0, s>>>(a, part.as<uint32_t>(), gathered, gv, tickets + 1);
  B2_LAUNCHED();
  const uint16_t* ps = pos.as<uint16_t>();
  if constexpr (!FUSED) launch_restore<OT, -1>(a, n_tiles, hist, ps, lookback, gathered, gv, s);
  else if (a.op == B2_ADD) launch_restore<OT, B2_ADD>(a, n_tiles, hist, ps, lookback, gathered, gv, s);
  else if (a.op == B2_SUBTRACT) launch_restore<OT, B2_SUBTRACT>(a, n_tiles, hist, ps, lookback, gathered, gv, s);
  else launch_restore<OT, B2_MULTIPLY>(a, n_tiles, hist, ps, lookback, gathered, gv, s);
  B2_LAUNCHED();
  return B2_OK;
}

template <typename VT, typename OT, bool FUSED>
static int run_idx(B2Context* ctx, const PartTakeArgs& a, int idx_type, cudaStream_t s, bool* ran) {
  switch (idx_type) {
    case B2_INT32: return run_passes<int32_t, VT, OT, FUSED>(ctx, a, s, ran);
    case B2_UINT32: return run_passes<uint32_t, VT, OT, FUSED>(ctx, a, s, ran);
    case B2_INT64: return run_passes<int64_t, VT, OT, FUSED>(ctx, a, s, ran);
    case B2_UINT64: return run_passes<uint64_t, VT, OT, FUSED>(ctx, a, s, ran);
    default: *ran = false; return B2_OK;
  }
}

template <typename OT>
static int run_fused(B2Context* ctx, const PartTakeArgs& a, int value_type, int idx_type, cudaStream_t s, bool* ran) {
  switch (value_type) {
    case B2_DOUBLE: return run_idx<double, OT, true>(ctx, a, idx_type, s, ran);
    case B2_FLOAT: return run_idx<float, OT, true>(ctx, a, idx_type, s, ran);
    case B2_INT64: return run_idx<int64_t, OT, true>(ctx, a, idx_type, s, ran);
    case B2_INT32: return run_idx<int32_t, OT, true>(ctx, a, idx_type, s, ran);
    default: *ran = false; return B2_OK;
  }
}

int take_partitioned(B2Context* ctx, const PartTakeArgs& a, int vw, int value_type, int idx_type, int out_type,
                     cudaStream_t s, bool* ran) {
  if (out_type == B2_FLOAT) return run_fused<float>(ctx, a, value_type, idx_type, s, ran);
  if (out_type == B2_DOUBLE) return run_fused<double>(ctx, a, value_type, idx_type, s, ran);
  if (vw == 4) return run_idx<uint32_t, uint32_t, false>(ctx, a, idx_type, s, ran);
  if (vw == 8) return run_idx<uint64_t, uint64_t, false>(ctx, a, idx_type, s, ran);
  *ran = false;
  return B2_OK;
}

}  // namespace b2
