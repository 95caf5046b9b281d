// take_partitioned.cu -- partitioned gather for large random fixed-width Take (b2_take, b2_take_cast_arith).
//
// A gather in row order makes one random DRAM access per row once the values are far larger than L2: the H100 sustains
// about 28 G of those per second (bench_micro/gather_probe.cu, 8 GB table), a quarter of its streaming bandwidth.  If the
// rows are first grouped by the band of `values` they read, each band is gathered while it sits in L2 and `values` is
// read from DRAM about once: with 256 bands of 32 MB the same probe sustains 74 G gathers/s.  Bucket = j >> shift
// (< 256); "bucket order" is the order of all n rows sorted stably by bucket.  Four passes, and a fifth for a cast to
// float32 of 8-byte values with nulls:
//
//   F  fold: a float32 copy of the values with each null row's slot a signalling NaN that names the row's cast in a
//      side table, so that B makes one random request per row instead of two (see "fold" below).  Its null counts
//      and their scan run before A; the copy itself is made inside B's launch, each band just ahead of its gathers
//      (see "fold under the gather").
//   A  tile partition: each 4096-row tile, in any order, is ranked stably by bucket (ballot matching, as
//      sort_indices.cu's onesweep_kernel) and written back in its own slot: the uint32 index j in the tile's bucket
//      order, each row's uint16 tile-local position in row order, and one cell per bucket holding the bucket's count
//      and the start of its run in the tile.  It also finds the first out-of-range valid index (atomicMin, the direct
//      kernels' rule).  Null and out-of-range indices count as index 0.  A needs nothing global: no histogram pass
//      and no look-back.
//   S  positions: the tiles x 256 cell matrix scanned in bucket-major order (column sums over groups of tiles, one
//      block scanning those, then each group walking its columns).  Per tile and bucket it gives where the run lands
//      in bucket order (tile-major, for C); per non-empty cell a run descriptor, compacted in bucket order (for B);
//      per 4096-position chunk of bucket order the run holding its first position.  Compaction keeps a chunk's runs
//      at most 4097 whatever the distribution: a skewed column leaves long stretches of empty cells.
//   B  banded gather: 4096-position chunks of bucket order claimed in order through a ticket so the whole GPU works
//      on about one band at a time.  A chunk loads its runs into shared memory, finds each position's run (a mark at
//      each run start, then a max-scan) and reads j from the run's tile slot; gathers values[j] and its validity bit,
//      casts to the output type, writes both in bucket order.  With F it gathers folded[j] instead, and side[...]
//      for a sentinel, and the same queue holds the fold items, each ahead of the chunks that read it.
//      Prefetching the next band into L2 (cp.async.bulk.prefetch.L2) measured slower, so there is none.
//   C  restore: the mirror image of A, without ranking again.  A tile takes its bucket counts from its cells and its
//      runs' places from S, reads its runs of gathered values through shared memory, puts them back in row order with
//      A's positions and finishes: masks null indices, applies the arithmetic with `other` (fused) and writes the
//      result and its bitmap in row order.
//
// B and C issue each phase's global loads together, into registers or shared memory, before the first store that
// needs them: one memory round trip per phase rather than one per item.
//
// Results are bit-identical to the direct kernels of selection_take.cu.  Limits: n < 2^30 (positions and run sources
// are uint32), values_length <= 2^32 (indices are carried as uint32).  Temporaries: about n * 11 bytes (n * 15 for
// 8-byte results): j 4, positions 2, gathered values 4 or 8, gathered validity 1/8, cells, run places and run
// descriptors 1; with F also values_length * 4 + null_count * 4 (the folded copy and the side table) and 4 bytes per
// 4096 values, and 2 KB for the fold groups' counters and places in B's queue.
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
// a cell: the bucket's count in the tile (bits 15:0) and the tile-local start of its run (bits 31:16), both <= 4096
constexpr uint32_t kCellCount = 0xffffu;
constexpr int kScanGroup = 256;     // tiles per group of pass S
constexpr int kScanBatch = 16;      // cells loaded together by a thread of pass S
constexpr int kScanThreads = 1024;  // the single block scanning the group sums

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

// The lanes whose `x & bit` equals this lane's: one predicate test, the ballot and a predicated complement.  Written
// in C++ (`bit ? bal : ~bal`), ptxas tests the bit twice and selects the complement, about 7 instructions a bit
// against 4; pass A is bound by instruction issue, and this is 8 of them per row.
__device__ __forceinline__ unsigned ballot_same_bit(unsigned x, unsigned bit) {
  unsigned bal;
  asm("{\n\t.reg .pred p;\n\t.reg .b32 t;\n\t"
      "and.b32 t, %1, %2;\n\t"
      "setp.ne.u32 p, t, 0;\n\t"
      "vote.sync.ballot.b32 %0, p, 0xffffffff;\n\t"
      "@!p not.b32 %0, %0;\n\t}"
      : "=r"(bal)
      : "r"(x), "r"(bit));
  return bal;
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
    for (int b = 0; b < kBucketBits; ++b) peers &= ballot_same_bit(bkt[j], 1u << b);
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

// ---- pass A ---------------------------------------------------------------------------------------------------------
template <typename Idx>
__global__ void __launch_bounds__(kPartThreads) part_tile_kernel(PartTakeArgs a, uint32_t* __restrict__ part,
                                                                 uint16_t* __restrict__ pos, uint32_t* __restrict__ cells) {
  __shared__ __align__(16) uint32_t s_j[kPartTile];
  __shared__ __align__(16) uint16_t s_lp[kPartTile];
  __shared__ uint32_t s_cnt[kPartWarps * kBuckets];
  __shared__ uint64_t s_iv[kPartTile / 64];
  __shared__ uint32_t s_warp_tot[kPartWarps];
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t tile = blockIdx.x;
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
    if (iv && u >= vlen && i < tile_n) atomicMin(a.first_bad, static_cast<unsigned long long>(base + i));
    jj[j] = (iv && u < vlen) ? static_cast<uint32_t>(u) : 0u;  // null / out of range: index 0, masked (or raised) later
    bkt[j] = i < tile_n ? jj[j] >> a.shift : kBuckets - 1;     // padding sorts last
  }
  uint16_t rank[kPartItems];
  uint32_t count, bin_off;
  rank_tile(bkt, rank, s_cnt, s_warp_tot, &count, &bin_off);
  if (tid == kBuckets - 1) count -= kPartTile - tile_n;
  cells[(size_t)tile * kBuckets + tid] = count | bin_off << 16;
#pragma unroll
  for (int j = 0; j < kPartItems; ++j) {
    const uint32_t lp = s_cnt[warp * kBuckets + bkt[j]] + rank[j];
    s_j[lp] = jj[j];
    s_lp[warp * (32 * kPartItems) + j * 32 + lane] = static_cast<uint16_t>(lp);
  }
  __syncthreads();
  // the whole tile, padding included (the buffers hold whole tiles), as 16-byte stores
  uint4* pos4 = reinterpret_cast<uint4*>(pos + base);
  __stcs(pos4 + tid, reinterpret_cast<const uint4*>(s_lp)[tid]);
  __stcs(pos4 + kPartThreads + tid, reinterpret_cast<const uint4*>(s_lp)[kPartThreads + tid]);
  uint4* part4 = reinterpret_cast<uint4*>(part + base);
#pragma unroll
  for (int k = 0; k < kPartTile / 4 / kPartThreads; ++k)
    __stcs(part4 + k * kPartThreads + tid, reinterpret_cast<const uint4*>(s_j)[k * kPartThreads + tid]);
}

// ---- pass S ---------------------------------------------------------------------------------------------------------
// Groups of kScanGroup tiles; the group sums are laid out bucket-major, [bucket][group], so that their exclusive scan in
// memory order gives each (bucket, group) its first position in bucket order and its first run.
// S1: per group and bucket, the rows and the non-empty cells.
__global__ void __launch_bounds__(kBuckets) part_colsum_kernel(const uint32_t* __restrict__ cells, uint32_t n_tiles,
                                                               uint32_t* __restrict__ grp_rows,
                                                               uint32_t* __restrict__ grp_runs) {
  const uint32_t g = blockIdx.x, b = threadIdx.x;
  const uint32_t t1 = min(n_tiles, (g + 1) * kScanGroup);
  uint32_t rows = 0, runs = 0;
  for (uint32_t t = g * kScanGroup; t < t1; t += kScanBatch) {
    uint32_t c[kScanBatch];
#pragma unroll
    for (int k = 0; k < kScanBatch; ++k) c[k] = t + k < t1 ? cells[(size_t)(t + k) * kBuckets + b] : 0u;
#pragma unroll
    for (int k = 0; k < kScanBatch; ++k) {
      rows += c[k] & kCellCount;
      runs += (c[k] & kCellCount) != 0;
    }
  }
  grp_rows[b * gridDim.x + g] = rows;
  grp_runs[b * gridDim.x + g] = runs;
}

// S2: one block scans both group-sum arrays (m entries, a multiple of 4) in place, exclusively.  The total of the runs
// closes the chunk table, and a sentinel run starting at n closes the run list.
__global__ void __launch_bounds__(kScanThreads) part_scan_kernel(uint32_t* grp_rows, uint32_t* grp_runs, uint32_t m,
                                                                 uint32_t n_tiles, uint32_t n, uint32_t* chunk_first,
                                                                 uint2* runs) {
  __shared__ uint2 s_warp[kScanThreads / 32];
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  uint32_t carry_rows = 0, carry_runs = 0;
  for (uint32_t i0 = 0; i0 < m; i0 += 4 * kScanThreads) {
    const uint32_t i = i0 + 4 * threadIdx.x;
    uint4 r = make_uint4(0, 0, 0, 0), q = make_uint4(0, 0, 0, 0);
    if (i < m) {
      r = *reinterpret_cast<const uint4*>(grp_rows + i);
      q = *reinterpret_cast<const uint4*>(grp_runs + i);
    }
    const uint32_t tr = r.x + r.y + r.z + r.w, tq = q.x + q.y + q.z + q.w;
    uint32_t ir = tr, iq = tq;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t ur = __shfl_up_sync(0xffffffffu, ir, o), uq = __shfl_up_sync(0xffffffffu, iq, o);
      if (lane >= o) {
        ir += ur;
        iq += uq;
      }
    }
    if (lane == 31) s_warp[warp] = make_uint2(ir, iq);
    __syncthreads();
    uint32_t er = carry_rows + ir - tr, eq = carry_runs + iq - tq;
#pragma unroll 8
    for (int w = 0; w < kScanThreads / 32; ++w) {
      const uint2 s = s_warp[w];
      if (w < (int)warp) {
        er += s.x;
        eq += s.y;
      }
      carry_rows += s.x;
      carry_runs += s.y;
    }
    __syncthreads();  // s_warp is free again
    if (i < m) {
      *reinterpret_cast<uint4*>(grp_rows + i) = make_uint4(er, er + r.x, er + r.x + r.y, er + r.x + r.y + r.z);
      *reinterpret_cast<uint4*>(grp_runs + i) = make_uint4(eq, eq + q.x, eq + q.x + q.y, eq + q.x + q.y + q.z);
    }
  }
  if (threadIdx.x == 0) {
    chunk_first[n_tiles] = carry_runs;
    runs[carry_runs] = make_uint2(n, 0u);
  }
}

// S3: each group walks its columns again from the scanned sums, 32 tiles at a time staged through shared memory so
// that a warp scans one bucket's column across 32 tiles (lane = tile) and the column's runs are stored together.
// gbase[t][b] = (position in bucket order of tile t's bucket-b run) - (the run's start in the tile), for C.  A non-empty
// cell becomes run descriptor {position in bucket order of its first row, source offset}: row p of bucket order in that
// run has its index at part[source offset + p] (mod 2^32).  chunk_first[c] is the run holding position 4096 * c (a run
// of at most 4096 rows holds at most one).
__global__ void __launch_bounds__(kBuckets) part_runs_kernel(const uint32_t* __restrict__ cells, uint32_t n_tiles,
                                                             const uint32_t* __restrict__ grp_rows,
                                                             const uint32_t* __restrict__ grp_runs,
                                                             uint32_t* __restrict__ gbase, uint2* __restrict__ runs,
                                                             uint32_t* __restrict__ chunk_first) {
  __shared__ uint32_t s_c[32][kBuckets + 1];  // [tile][bucket]: the cells, then gbase
  __shared__ uint32_t s_gp[kBuckets], s_r[kBuckets];
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t g = blockIdx.x;
  const uint32_t t1 = min(n_tiles, (g + 1) * kScanGroup);
  s_gp[tid] = grp_rows[tid * gridDim.x + g];
  s_r[tid] = grp_runs[tid * gridDim.x + g];
  for (uint32_t t0 = g * kScanGroup; t0 < t1; t0 += 32) {
    const uint32_t nt = min(32u, t1 - t0);
#pragma unroll
    for (int k = 0; k < 32; ++k) s_c[k][tid] = k < nt ? cells[(size_t)(t0 + k) * kBuckets + tid] : 0u;
    __syncthreads();
    // warp w owns buckets 32w .. 32w + 31: no other warp touches their s_gp / s_r
    for (int bb = 0; bb < 32; ++bb) {
      const uint32_t b = warp * 32 + bb;
      const uint32_t c = s_c[lane][b], count = c & kCellCount, bin_off = c >> 16;
      uint32_t incl = count;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
      }
      const unsigned ne = __ballot_sync(0xffffffffu, count != 0);
      const uint32_t gp = s_gp[b] + incl - count, r = s_r[b] + __popc(ne & lanemask_lt());
      s_c[lane][b] = gp - bin_off;
      if (count) {
        runs[r] = make_uint2(gp, (t0 + lane) * kPartTile + bin_off - gp);
        const uint32_t q = (gp + kPartTile - 1) / kPartTile;
        if (q * kPartTile < gp + count) chunk_first[q] = r;
      }
      __syncwarp();  // every lane has read s_gp[b] / s_r[b]
      if (lane == 31) {
        s_gp[b] = gp + count;
        s_r[b] = r + (count != 0);
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 32; ++k)
      if (k < nt) gbase[(size_t)(t0 + k) * kBuckets + tid] = s_c[k][tid];
    __syncthreads();
  }
}

// ---- fold (pass F) --------------------------------------------------------------------------------------------------
// b2_take_cast_arith to float32 from 8-byte values with nulls.  B would make two random requests per row, the value and
// its validity byte, and the banded gather is bound by the rate of those requests, not by their bytes.  F writes
// folded[j] = static_cast<float>(values[j]) for a valid row; a null row gets a signalling NaN naming its rank among its
// band's nulls, and its real cast goes to side[band_base[band] + rank], so that C still sees the value the direct
// kernels compute for it.  A conversion returns a quiet NaN and int -> float no NaN, so no valid row reads as a
// sentinel.  B then makes one request per row, and a second one, into a slice that stays in L2, for the null rows.
// Ranks: null counts over tiles of 2^tb values (tb = min(shift, 12), whole tiles per band), scanned by one block.
constexpr uint32_t kFoldHalf = (1u << 22) - 1;  // payloads per sign: a non-zero mantissa with the quiet bit clear

__device__ __forceinline__ uint32_t fold_sentinel(uint32_t rank) {  // rank < 2 * kFoldHalf
  return rank < kFoldHalf ? 0x7f800000u | (rank + 1) : 0xff800000u | (rank - kFoldHalf + 1);
}
__device__ __forceinline__ bool is_fold_sentinel(uint32_t x) {
  return (x & 0x7fc00000u) == 0x7f800000u && (x & 0x3fffffu) != 0;
}
__device__ __forceinline__ uint32_t fold_rank(uint32_t x) { return (x & 0x3fffffu) - 1 + (x >> 31) * kFoldHalf; }

// F1: one warp per tile of 2^tb values (2^(tb - 6) bitmap words): its null count
__global__ void __launch_bounds__(kPartThreads) fold_count_kernel(BitmapReader vv, uint32_t n_ct, int tb,
                                                                  uint32_t* __restrict__ counts) {
  const uint32_t t = blockIdx.x * kPartWarps + (threadIdx.x >> 5);
  if (t >= n_ct) return;  // whole warps
  const unsigned lane = lane_id();
  uint32_t nulls = 0;
  for (int w = lane; w < (1 << (tb - 6)); w += 32) {
    const int64_t wi = ((int64_t)t << (tb - 6)) + w;
    const int64_t rem = vv.nbits - (wi << 6);
    if (rem > 0) nulls += (rem < 64 ? static_cast<uint32_t>(rem) : 64u) - __popcll(vv.word(wi));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nulls += __shfl_xor_sync(0xffffffffu, nulls, o);
  if (lane == 0) counts[t] = nulls;
}

// F2: one block scans the n_ct tile counts in place, exclusively (base[n_ct] = all nulls), then gives each bucket the
// base of its first tile: band_base[b] = base[b << band_tiles_log2]
__global__ void __launch_bounds__(kScanThreads) fold_scan_kernel(uint32_t* base, uint32_t n_ct, int band_tiles_log2,
                                                                 uint32_t* __restrict__ band_base) {
  __shared__ uint32_t s_warp[kScanThreads / 32];
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  uint32_t carry = 0;
  for (uint32_t i0 = 0; i0 < n_ct; i0 += 4 * kScanThreads) {
    const uint32_t i = i0 + 4 * threadIdx.x;
    uint32_t c[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) c[q] = i + q < n_ct ? base[i + q] : 0u;
    const uint32_t t = c[0] + c[1] + c[2] + c[3];
    uint32_t incl = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t e = carry + incl - t;
#pragma unroll 8
    for (int w = 0; w < kScanThreads / 32; ++w) {
      if (w < (int)warp) e += s_warp[w];
      carry += s_warp[w];
    }
    __syncthreads();  // s_warp is free again
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (i + q < n_ct) base[i + q] = e;
      e += c[q];
    }
  }
  if (threadIdx.x == 0) base[n_ct] = carry;
  __syncthreads();  // the block's global stores are visible to the block
  if (threadIdx.x < kBuckets) {
    const uint32_t t = threadIdx.x << band_tiles_log2;
    band_base[threadIdx.x] = t < n_ct ? base[t] : carry;
  }
}

// F3, a fold item of pass B: 4096 values (a whole number of count tiles), streamed; the ranks within the item come from
// a scan of its 64 bitmap words.  folded and side get plain stores: the band is gathered from L2 soon after.
struct FoldArgs {
  const uint32_t* tile_base;  // per count tile: the nulls before it (pass F2)
  const uint32_t* band_base;  // per bucket: the nulls before its first row
  uint32_t* folded;           // float32 bits
  float* side;                // the null rows' casts, in row order
  uint32_t side_cap;          // values->null_count: a null count too small cannot write or read past the table
  int tb;                     // count tiles of 2^tb values
  // the queue of pass B (see "fold under the gather")
  int group_shift;              // fold group of row j = j >> group_shift
  uint32_t n_groups;            // <= 256
  uint32_t n_items;             // fold items: values_length / 4096, rounded up
  uint32_t* ticket;             // 0 initially
  uint32_t* fold_done;          // per group: its fold items that have finished, 0 initially
  const uint32_t* gather_end;   // per group g: the gather chunks whose last position reads a group <= g (part_sched_kernel)
};

template <typename VT>
__device__ __forceinline__ void fold_item(const VT* __restrict__ vals, const BitmapReader& vv, int shift, const FoldArgs& f,
                                          uint32_t item, uint64_t* s_w, uint32_t* s_pre) {
  // s_w: the item's 64 bitmap words; s_pre: nulls of the item before each word
  const unsigned tid = threadIdx.x, lane = tid & 31;
  const int64_t base = (int64_t)item * kPartTile;
  const int64_t vlen = vv.nbits;
  VT v[kPartItems];
#pragma unroll
  for (int k = 0; k < kPartItems; ++k) {
    const int64_t r = base + k * kPartThreads + tid;
    v[k] = r < vlen ? __ldcs(vals + r) : VT(0);
  }
  if (tid < 32) {  // lane l: words 2l and 2l + 1
    const uint64_t w0 = vv.word((base >> 6) + 2 * lane), w1 = vv.word((base >> 6) + 2 * lane + 1);
    const int64_t rem = vlen - base - 128 * (int64_t)lane;
    const uint32_t rows0 = rem <= 0 ? 0u : rem < 64 ? static_cast<uint32_t>(rem) : 64u;
    const uint32_t rows1 = rem <= 64 ? 0u : rem < 128 ? static_cast<uint32_t>(rem - 64) : 64u;
    const uint32_t c0 = rows0 - __popcll(w0), c1 = rows1 - __popcll(w1);
    uint32_t incl = c0 + c1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    s_w[2 * lane] = w0;
    s_w[2 * lane + 1] = w1;
    s_pre[2 * lane] = incl - c0 - c1;
    s_pre[2 * lane + 1] = incl - c1;
  }
  __syncthreads();
  const uint32_t block_nulls = f.tile_base[base >> f.tb];
#pragma unroll
  for (int k = 0; k < kPartItems; ++k) {
    const uint32_t r = k * kPartThreads + tid;
    const int64_t row = base + r;
    if (row >= vlen) break;
    const float c = static_cast<float>(v[k]);
    const uint64_t w = s_w[r >> 6];
    uint32_t x = __float_as_uint(c);
    if (!((w >> (r & 63)) & 1u)) {
      const uint32_t rank = block_nulls + s_pre[r >> 6] + __popcll(~w & ((1ull << (r & 63)) - 1));
      if (rank < f.side_cap) f.side[rank] = c;
      x = fold_sentinel(rank - f.band_base[row >> shift]);
    }
    f.folded[row] = x;
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

// The same, served by L2: for words another CTA of the same launch stored, which a stale L1 line must not answer.
__device__ __forceinline__ uint32_t ld_l2_before_stores(const uint32_t* p) {
  uint32_t w;
  asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(w) : "l"(p));
  return w;
}

// The shared memory of a gather chunk.  A fold item lays its 64 bitmap words and their null prefixes over `src`.
struct ChunkShared {
  __align__(16) uint32_t src[kPartTile + 1];  // the chunk's runs' source offsets
  __align__(16) uint16_t run[kPartTile];      // per position: a mark at each run start, then its run
  uint32_t warp_max[kPartWarps];
  uint32_t claimed;                           // the ticket
};

__device__ __forceinline__ void clear_marks(ChunkShared& sh) {
  reinterpret_cast<uint4*>(sh.run)[threadIdx.x] = make_uint4(0, 0, 0, 0);
  reinterpret_cast<uint4*>(sh.run)[kPartThreads + threadIdx.x] = make_uint4(0, 0, 0, 0);
}

// The indices of chunk c (positions 4096c .. 4096c + 4095 of bucket order): j[k] belongs to position
// 4096c + 256k + tid.  The marks are clear and the block has synchronised since.
__device__ __forceinline__ void chunk_indices(int64_t n, const uint32_t* __restrict__ part, const uint2* __restrict__ runs,
                                              const uint32_t* __restrict__ chunk_first, uint32_t c, ChunkShared& sh,
                                              uint32_t (&j)[kPartItems]) {
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t p0 = c * kPartTile;
  // runs r0 .. r1: r0 holds p0, r1 holds p0 + 4096 (or is the sentinel starting at n); run r0 is run 0 of the chunk
  const uint32_t r0 = chunk_first[c], r1 = chunk_first[c + 1];
  for (uint32_t i = tid; i <= r1 - r0; i += kPartThreads) {
    const uint2 run = runs[r0 + i];
    sh.src[i] = run.y;
    const uint32_t at = run.x - p0;  // wraps for run 0 when it starts before p0
    if (at < (uint32_t)kPartTile) sh.run[at] = static_cast<uint16_t>(i);
  }
  __syncthreads();
  // inclusive max-scan of the marks: thread t owns positions 16t .. 16t + 15
  {
    uint4 m4[2] = {reinterpret_cast<const uint4*>(sh.run)[2 * tid], reinterpret_cast<const uint4*>(sh.run)[2 * tid + 1]};
    uint32_t* m = reinterpret_cast<uint32_t*>(m4);  // 8 words of two uint16 each
    uint32_t run = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      const uint32_t lo = max(run, m[w] & 0xffffu), hi = max(lo, m[w] >> 16);
      m[w] = lo | hi << 16;
      run = hi;
    }
    uint32_t incl = run;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) incl = max(incl, __shfl_up_sync(0xffffffffu, incl, o));
    if (lane == 31) sh.warp_max[warp] = incl;
    uint32_t excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 0;
    __syncthreads();
#pragma unroll
    for (int w = 0; w < kPartWarps; ++w)
      if (w < (int)warp) excl = max(excl, sh.warp_max[w]);
#pragma unroll
    for (int w = 0; w < 8; ++w) m[w] = max(excl, m[w] & 0xffffu) | max(excl, m[w] >> 16) << 16;
    reinterpret_cast<uint4*>(sh.run)[2 * tid] = m4[0];
    reinterpret_cast<uint4*>(sh.run)[2 * tid + 1] = m4[1];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kPartItems; ++k) {
    const uint32_t p = p0 + k * kPartThreads + tid;
    j[k] = p < n ? __ldcs(part + (sh.src[sh.run[k * kPartThreads + tid]] + p)) : 0u;
  }
}

// gathers values[j] and its validity bit
template <typename VT, typename OT>
__global__ void __launch_bounds__(kPartThreads) part_gather_kernel(PartTakeArgs a, const uint32_t* __restrict__ part,
                                                                   const uint2* __restrict__ runs,
                                                                   const uint32_t* __restrict__ chunk_first, OT* g,
                                                                   uint32_t* __restrict__ gvalid, uint32_t* ticket) {
  __shared__ ChunkShared sh;
  if (threadIdx.x == 0) sh.claimed = atomicAdd(ticket, 1u);
  clear_marks(sh);
  __syncthreads();
  const uint32_t p0 = sh.claimed * kPartTile;
  uint32_t j[kPartItems];
  chunk_indices(a.n, part, runs, chunk_first, sh.claimed, sh, j);
  const VT* __restrict__ vals = static_cast<const VT*>(a.values);
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

// ---- fold under the gather ------------------------------------------------------------------------------------------
// With pass F, B's launch also does the folding (F3): its queue holds fold items (4096 values each) and gather chunks,
// one per CTA, claimed in order through the ticket.  The gathers are bound by the rate of random L2 requests and leave
// most of the DRAM bandwidth idle; the fold is pure streaming, so it runs under them, and a band is gathered while
// what the fold just stored is still in L2.
//
// Fold group of row j = j >> max(shift, 12): a band, or 4096 values when the bands are smaller; at most 256.  The
// queue is: the fold items of groups 0 .. kFoldLead - 1; then for g = 0, 1, ...: the fold items of group g + kFoldLead
// and the gather chunks whose last position reads group g, alternating in proportion.  Bucket order is sorted by band,
// so a chunk of step g reads the groups of its first position up to g and no other.  A fold CTA, after its stores,
// fences and adds one to its group's counter; a gather CTA, once it holds its indices, waits until each group it
// reads has counted all its items, then gathers through L2 (ld_l2_before_stores).
//
// Invariant (part_sched_kernel's gather_end and queue_step below are the only code that orders the queue): the last
// group a gather chunk reads is at most the highest group whose fold items all have smaller tickets than the chunk.
// So the wait cannot deadlock: every fold item a chunk waits on has a smaller ticket, a ticket is only ever claimed by
// a CTA that is already running, and a fold item waits on nothing.  Whatever a waiting CTA waits on is in the hands
// of running CTAs that finish unconditionally, however many CTAs are resident and in whatever order they start.
// The wait is bounded all the same: after kFoldWaitNs it sets *a.stalled and carries on, and the call fails.
constexpr int kFoldLead = 2;
constexpr unsigned long long kFoldWaitNs = 4000000000ull;  // a real wait is microseconds

// fold items in groups 0 .. g; g = -1 gives 0
__device__ __forceinline__ uint32_t fold_items_through(const FoldArgs& f, int g) {
  const uint64_t e = static_cast<uint64_t>(g + 1) << (f.group_shift - 12);
  return e < f.n_items ? static_cast<uint32_t>(e) : f.n_items;
}

// S4: gather_end[g] for every group, from the first position of each bucket (pass S2 leaves the rows before bucket b
// in grp_rows[b * n_scan_groups]).  A chunk's last position is 4096c + 4095, or n - 1 for the last chunk.
__global__ void __launch_bounds__(kBuckets) part_sched_kernel(const uint32_t* __restrict__ grp_rows, uint32_t n_scan_groups,
                                                              uint32_t n, uint32_t n_tiles, int buckets_per_group_log2,
                                                              uint32_t* __restrict__ gather_end) {
  const uint32_t b = (threadIdx.x + 1) << buckets_per_group_log2;  // the first bucket after group threadIdx.x
  const uint32_t p = b < (uint32_t)kBuckets ? grp_rows[(size_t)b * n_scan_groups] : n;
  gather_end[threadIdx.x] = p == n ? n_tiles : p / kPartTile;
}

__device__ __forceinline__ void wait_folded(const uint32_t* done, uint32_t want, unsigned long long* stalled) {
  unsigned long long t0 = 0;
  for (;;) {
    uint32_t seen;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(done) : "memory");
    if (seen >= want) return;
    unsigned long long now;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
    if (!t0) t0 = now;
    if (now - t0 > kFoldWaitNs || *reinterpret_cast<volatile unsigned long long*>(stalled)) {
      *stalled = 1ull;
      return;
    }
    __nanosleep(100);
  }
}

template <typename VT>
__global__ void __launch_bounds__(kPartThreads) part_fold_gather_kernel(PartTakeArgs a, const uint32_t* __restrict__ part,
                                                                        const uint2* __restrict__ runs,
                                                                        const uint32_t* __restrict__ chunk_first, float* g,
                                                                        uint32_t* __restrict__ gvalid, FoldArgs f) {
  __shared__ ChunkShared sh;
  __shared__ uint32_t s_band_base[kBuckets];
  __shared__ uint32_t s_gather_begin[kBuckets];  // per step: the gather chunks of earlier steps
  __shared__ uint32_t s_first_group;
  const unsigned tid = threadIdx.x;
  if (tid == 0) sh.claimed = atomicAdd(f.ticket, 1u);
  s_band_base[tid] = f.band_base[tid];
  const uint32_t gather_begin = tid ? f.gather_end[tid - 1] : 0u;
  s_gather_begin[tid] = gather_begin;
  clear_marks(sh);
  __syncthreads();
  // the step of ticket t: the last one that begins at or before t (step tid begins at its fold items); none: the lead
  const uint32_t t = sh.claimed;
  const int last = static_cast<int>(f.n_groups) - 1;
  const int step = __syncthreads_count(tid < f.n_groups &&
                                       fold_items_through(f, min((int)tid + kFoldLead - 1, last)) + gather_begin <= t) - 1;
  bool is_fold = true;
  uint32_t item = t;
  if (step >= 0) {
    const uint32_t f0 = fold_items_through(f, min(step + kFoldLead - 1, last));
    const uint32_t nf = fold_items_through(f, min(step + kFoldLead, last)) - f0;
    const uint32_t ng = (step < last ? s_gather_begin[step + 1] : gridDim.x - f.n_items) - s_gather_begin[step];
    const uint32_t r = t - f0 - s_gather_begin[step];
    // of the step's nf + ng items, item r is a fold item when the fold share of r + 1 items exceeds that of r
    const uint32_t before = static_cast<uint32_t>((uint64_t)r * nf / (nf + ng));
    is_fold = static_cast<uint32_t>((uint64_t)(r + 1) * nf / (nf + ng)) > before;
    item = is_fold ? f0 + before : s_gather_begin[step] + r - before;
  }
  if (is_fold) {
    fold_item(static_cast<const VT*>(a.values), a.values_valid, a.shift, f, item, reinterpret_cast<uint64_t*>(sh.src),
              sh.src + 2 * (kPartTile / 64));
    __threadfence();
    __syncthreads();
    if (tid == 0) atomicAdd(f.fold_done + (static_cast<uint64_t>(item) * kPartTile >> f.group_shift), 1u);
    return;
  }
  const uint32_t p0 = item * kPartTile;
  uint32_t j[kPartItems];
  chunk_indices(a.n, part, runs, chunk_first, item, sh, j);
  if (tid == 0) s_first_group = j[0] >> f.group_shift;
  __syncthreads();
  {
    const int grp = static_cast<int>(s_first_group + tid);
    if (grp <= step) wait_folded(f.fold_done + grp, fold_items_through(f, grp) - fold_items_through(f, grp - 1), a.stalled);
  }
  __syncthreads();
  // one request per row in one batch; a sentinel (a null row) sends a second one to `side`
  uint32_t x[kPartItems];
#pragma unroll
  for (int k = 0; k < kPartItems; ++k) x[k] = ld_l2_before_stores(f.folded + j[k]);
  uint32_t valid = 0;
#pragma unroll
  for (int k = 0; k < kPartItems; ++k) {
    if (is_fold_sentinel(x[k]))
      x[k] = ld_l2_before_stores(reinterpret_cast<const uint32_t*>(f.side) +
                                 min(s_band_base[j[k] >> a.shift] + fold_rank(x[k]), f.side_cap - 1));
    else
      valid |= 1u << k;
  }
#pragma unroll
  for (int k = 0; k < kPartItems; ++k) {
    const int64_t p = p0 + k * kPartThreads + threadIdx.x;
    if (p < a.n) __stcs(g + p, __uint_as_float(x[k]));
    const unsigned w = __ballot_sync(0xffffffffu, p < a.n && ((valid >> k) & 1u));
    if (lane_id() == 0 && p < a.n) gvalid[p >> 5] = w;
  }
}

// ---- pass C ---------------------------------------------------------------------------------------------------------
// OP: B2_ADD / B2_SUBTRACT / B2_MULTIPLY for b2_take_cast_arith, -1 for a plain take.
template <typename OT, int OP>
__global__ void __launch_bounds__(kPartThreads) part_restore_kernel(PartTakeArgs a, const uint16_t* __restrict__ pos,
                                                                    const uint32_t* __restrict__ cells,
                                                                    const uint32_t* __restrict__ gbase,
                                                                    const OT* __restrict__ g,
                                                                    const uint32_t* __restrict__ gvalid) {
  constexpr bool kFused = OP >= 0;
  __shared__ OT s_val[kPartTile];
  __shared__ __align__(16) uint16_t s_lp[kPartTile];  // each row's tile-local position (pass A)
  __shared__ uint8_t s_bkt[kPartTile];                // the bucket of each tile-local position
  __shared__ uint32_t s_gv[kPartTile / 32];           // gathered validity by tile-local position
  __shared__ uint64_t s_iv[kPartTile / 64], s_ov[kPartTile / 64];  // index / `other` validity by row
  __shared__ uint32_t s_gbase[kBuckets];
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t tile = blockIdx.x;
  const uint32_t base = tile * kPartTile;
  const uint32_t tile_n = static_cast<uint32_t>(a.n - base) < (uint32_t)kPartTile ? static_cast<uint32_t>(a.n - base) : (uint32_t)kPartTile;
  const uint4* pos4 = reinterpret_cast<const uint4*>(pos + base);
  const uint4 q0 = __ldcs(pos4 + tid), q1 = __ldcs(pos4 + kPartThreads + tid);
  const uint32_t cell = cells[(size_t)tile * kBuckets + tid];
  const uint32_t gb = gbase[(size_t)tile * kBuckets + tid];
  uint64_t bits = 0;
  if (tid < kPartTile / 64) bits = a.idx_valid.word((base >> 6) + tid);
  else if (kFused && tid < kPartTile / 32) bits = a.other_valid.word((base >> 6) + tid - kPartTile / 64);
  reinterpret_cast<uint4*>(s_lp)[tid] = q0;
  reinterpret_cast<uint4*>(s_lp)[kPartThreads + tid] = q1;
  if (tid < kPartTile / 64) s_iv[tid] = bits;
  else if (kFused && tid < kPartTile / 32) s_ov[tid - kPartTile / 64] = bits;
  // thread b owns bucket b: its run is [bin_off, bin_off + count) of the tile and starts at gathered element
  // gb + bin_off
  const uint32_t count = cell & kCellCount, bin_off = cell >> 16;
  s_gbase[tid] = gb;
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
static void launch_restore(const PartTakeArgs& a, uint32_t n_tiles, const uint16_t* pos, const uint32_t* cells,
                           const uint32_t* gbase, const OT* gathered, const uint32_t* gv, cudaStream_t s) {
  part_restore_kernel<OT, OP><<<n_tiles, kPartThreads, 0, s>>>(a, pos, cells, gbase, gathered, gv);
}

template <typename Idx, typename VT, typename OT, bool FUSED>
static int run_passes(B2Context* ctx, const PartTakeArgs& a, cudaStream_t s, bool* ran) {
  *ran = false;
  const int64_t n = a.n;
  const uint32_t n_tiles = static_cast<uint32_t>((n + kPartTile - 1) / kPartTile);
  const uint32_t n_groups = (n_tiles + kScanGroup - 1) / kScanGroup;
  const size_t n_cells = (size_t)n_tiles * kBuckets, n_sums = (size_t)n_groups * kBuckets;
  // cells, gbase, the two group-sum arrays, chunk_first (n_tiles + 1), the ticket of pass B and, for its fold items,
  // a counter and a gather_end per fold group
  const size_t meta_words = 2 * n_cells + 2 * n_sums + n_tiles + 2 + 2 * kBuckets;
  const size_t slots = (size_t)n_tiles * kPartTile;  // part, pos and g hold whole tiles
  // 4-byte results share part's block: 8 bytes a row, the size of the gathered block of a take of 8-byte values, so
  // a b2_take_cast_arith after such a take (as in a take, cast, add pipeline run both ways) reuses its cached blocks
  constexpr bool kShareBlock = sizeof(OT) == sizeof(uint32_t);
  Temp part(ctx, s), pos(ctx, s), g(ctx, s), gvalid(ctx, s), meta(ctx, s), runs(ctx, s);
  if (part.alloc((sizeof(uint32_t) + (kShareBlock ? sizeof(OT) : 0)) * slots) != B2_OK ||
      pos.alloc(sizeof(uint16_t) * slots) != B2_OK || (!kShareBlock && g.alloc(sizeof(OT) * slots) != B2_OK) ||
      meta.alloc(sizeof(uint32_t) * meta_words) != B2_OK || runs.alloc(sizeof(uint2) * (n_cells + 1)) != B2_OK ||
      ((a.values_valid.base != nullptr) && gvalid.alloc(bitmap_alloc_bytes(n)) != B2_OK))
    return B2_OK;  // the direct kernels run instead
  *ran = true;
  // the folded gather when the caller planned it and its temporaries can be had, else B reads the values
  constexpr bool kCanFold = FUSED && std::is_same<OT, float>::value && sizeof(VT) == 8;
  Temp folded(ctx, s), side(ctx, s), fold_meta(ctx, s);
  const int tb = a.shift < 12 ? a.shift : 12;  // count tiles of pass F: 2^tb values
  const uint32_t n_ct = static_cast<uint32_t>((a.values_length + (1ll << tb) - 1) >> tb);
  const bool fold = kCanFold && a.fold && a.values_valid.base != nullptr && a.value_nulls > 0 &&
                    a.shift >= kFoldMinShift && a.shift <= kFoldMaxShift &&
                    folded.alloc(sizeof(float) * a.values_length) == B2_OK &&
                    side.alloc(sizeof(float) * a.value_nulls) == B2_OK &&
                    fold_meta.alloc(sizeof(uint32_t) * (n_ct + 1 + kBuckets)) == B2_OK;
  uint32_t* cells = meta.as<uint32_t>();
  uint32_t* gbase = cells + n_cells;
  uint32_t* grp_rows = gbase + n_cells;  // n_cells and n_sums are multiples of 256: 16-byte aligned for pass S2
  uint32_t* grp_runs = grp_rows + n_sums;
  uint32_t* chunk_first = grp_runs + n_sums;
  uint32_t* ticket = chunk_first + n_tiles + 1;
  uint2* run_list = runs.as<uint2>();
  uint32_t* fold_done = ticket + 1;
  uint32_t* gather_end = fold_done + kBuckets;
  B2_CUDA(cudaMemsetAsync(ticket, 0, sizeof(uint32_t) * (1 + kBuckets), s));
  FoldArgs fa{};
  if constexpr (kCanFold) if (fold) {  // passes F1 and F2; instantiated for 8-byte values only
    uint32_t* tile_base = fold_meta.as<uint32_t>();
    uint32_t* band_base = tile_base + n_ct + 1;
    fold_count_kernel<<<(n_ct + kPartWarps - 1) / kPartWarps, kPartThreads, 0, s>>>(a.values_valid, n_ct, tb, tile_base);
    B2_LAUNCHED();
    fold_scan_kernel<<<1, kScanThreads, 0, s>>>(tile_base, n_ct, a.shift - tb, band_base);
    B2_LAUNCHED();
    fa.tile_base = tile_base;
    fa.band_base = band_base;
    fa.folded = folded.as<uint32_t>();
    fa.side = side.as<float>();
    fa.side_cap = static_cast<uint32_t>(a.value_nulls);
    fa.tb = tb;
    fa.group_shift = a.shift < 12 ? 12 : a.shift;
    fa.n_groups = static_cast<uint32_t>((a.values_length + (1ll << fa.group_shift) - 1) >> fa.group_shift);
    fa.n_items = static_cast<uint32_t>((a.values_length + kPartTile - 1) / kPartTile);
    fa.ticket = ticket;
    fa.fold_done = fold_done;
    fa.gather_end = gather_end;
  }
  part_tile_kernel<Idx><<<n_tiles, kPartThreads, 0, s>>>(a, part.as<uint32_t>(), pos.as<uint16_t>(), cells);
  B2_LAUNCHED();
  part_colsum_kernel<<<n_groups, kBuckets, 0, s>>>(cells, n_tiles, grp_rows, grp_runs);
  B2_LAUNCHED();
  part_scan_kernel<<<1, kScanThreads, 0, s>>>(grp_rows, grp_runs, static_cast<uint32_t>(n_sums), n_tiles,
                                              static_cast<uint32_t>(n), chunk_first, run_list);
  B2_LAUNCHED();
  part_runs_kernel<<<n_groups, kBuckets, 0, s>>>(cells, n_tiles, grp_rows, grp_runs, gbase, run_list, chunk_first);
  B2_LAUNCHED();
  uint32_t* gv = (a.values_valid.base != nullptr) ? gvalid.as<uint32_t>() : nullptr;
  OT* gathered = kShareBlock ? reinterpret_cast<OT*>(part.as<uint32_t>() + slots) : g.as<OT>();
  if constexpr (kCanFold) if (fold) {
    part_sched_kernel<<<1, kBuckets, 0, s>>>(grp_rows, n_groups, static_cast<uint32_t>(n), n_tiles,
                                             fa.group_shift - a.shift, gather_end);
    B2_LAUNCHED();
    part_fold_gather_kernel<VT><<<fa.n_items + n_tiles, kPartThreads, 0, s>>>(a, part.as<uint32_t>(), run_list, chunk_first,
                                                                             gathered, gv, fa);
  }
  if (!fold)
    part_gather_kernel<VT, OT><<<n_tiles, kPartThreads, 0, s>>>(a, part.as<uint32_t>(), run_list, chunk_first, gathered, gv,
                                                                ticket);
  B2_LAUNCHED();
  const uint16_t* ps = pos.as<uint16_t>();
  if constexpr (!FUSED) launch_restore<OT, -1>(a, n_tiles, ps, cells, gbase, gathered, gv, s);
  else if (a.op == B2_ADD) launch_restore<OT, B2_ADD>(a, n_tiles, ps, cells, gbase, gathered, gv, s);
  else if (a.op == B2_SUBTRACT) launch_restore<OT, B2_SUBTRACT>(a, n_tiles, ps, cells, gbase, gathered, gv, s);
  else launch_restore<OT, B2_MULTIPLY>(a, n_tiles, ps, cells, gbase, gathered, gv, s);
  B2_LAUNCHED();
  return B2_OK;
}

template <typename VT, typename OT, bool FUSED>
static int run_idx(B2Context* ctx, const PartTakeArgs& a, int idx_type, cudaStream_t s, bool* ran) {
  return visit_type(WideIndexTypes{}, idx_type, [&](auto it) { return run_passes<decltype(it), VT, OT, FUSED>(ctx, a, s, ran); },
                    [&] {
                      *ran = false;
                      return B2_OK;
                    });
}

template <typename OT>
static int run_fused(B2Context* ctx, const PartTakeArgs& a, int value_type, int idx_type, cudaStream_t s, bool* ran) {
  return visit_type(FusedTakeValueTypes{}, value_type, [&](auto vt) { return run_idx<decltype(vt), OT, true>(ctx, a, idx_type, s, ran); },
                    [&] {
                      *ran = false;
                      return B2_OK;
                    });
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
