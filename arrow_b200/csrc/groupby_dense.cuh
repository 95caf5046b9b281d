// groupby_dense.cuh -- the direct-addressed path of the fused group-by (hash_sum + hash_count).
//
// When the keys of a batch are DENSE -- the measured range R = kmax - kmin + 1 is at most a few times the number of
// groups, as for surrogate / dictionary / date keys -- no hashing and no partitioning is needed at all: the group's
// state lives at table[key - kmin] (what DuckDB calls a perfect hash aggregate; the reference's own analogue is the
// counting sorter it switches to for narrow ranges, kernels/vector_array_sort.cc:277-446).  The whole batch is then
// ONE streaming pass whose only cost beyond reading the two columns is one fire-and-forget 64-bit reduction per row:
//
//     table[key - kmin] += (1 << sb) | (value - vbase)        count in the high bits, sum of offsets in the low bits
//
// The packed state (R x 8 bytes, R <= 16M) is applied in key-range bands small enough to stay resident in L2
// (B2_DENSE_BAND_MB), so the reductions resolve in L2 instead of being 32-byte DRAM read-modify-writes.
// Field widths: a sub-batch of 2^m rows cannot overflow a count of m + 1 bits nor a sum of vb + m bits (vb = bits of
// the verified value window), so m = floor((63 - vb) / 2); after every sub-batch a drain pass folds the packed words
// into 64-bit sum / count arrays (traffic 24 R bytes per 2^m rows).  Rows with a null value only mark the group as
// existing (a bit in `exists`); rows with a null key go to the null group's accumulator, as in groupby_compact.cuh.
// The value window of 64-bit columns comes from a sample and is VERIFIED on every row: a violation raises the
// overflow flag and the host redoes the batch on the partitioned path -- nothing has reached the global table yet.
// One host driver, dense_accumulate in groupby_fused.cu, runs a batch: over keys for the fused group-by, and over group
// ids for hash_sum (dense_sum_count_by_id).
// At the end of the batch the dense state is flushed into the global 32-byte-slot table of groupby_fused.cu (one
// insert per group), which stays the single source of truth across batches and paths.
#pragma once
#include "groupby_compact.cuh"

namespace b2 {

constexpr unsigned long long kDenseMaxRange = 1ull << 24;  // 16M keys = 128 MB of packed state, applied in L2-sized bands

struct DenseArgs {
  const uint8_t* keys;  // advanced to the first row of the sub-batch
  const uint8_t* vals;
  int kw, vw;
  bool vsigned;
  BitmapReader key_valid, val_valid;  // addressed with row0 + i
  int64_t row0, n;
  unsigned long long kmin, kflip, range;  // idx = (key bits ^ kflip) - kmin < range (exact: from the stats pass)
  unsigned long long vbase;
  int vb, sb;                         // v' = value bits - vbase < 2^vb ; packed increment = (1 << sb) | v'
  unsigned long long* table;          // [range] packed, zero between sub-batches
  uint32_t* exists;                   // [range / 32 + 1]
  unsigned long long band_lo, band_hi;  // this launch applies rows with band_lo <= idx < band_hi
  unsigned long long* null_acc;       // [0] sum bits, [1] count, [2] rows
  unsigned int* overflow;
};

// min / max of <= 65536 evenly spaced valid keys (order-preserving encoding) and valid 64-bit values: sizes the dense table
// and the value window; both are verified on every row by dense_consume_kernel
template <int KW>
__global__ void __launch_bounds__(kBlock) dense_sample_kernel(const void* __restrict__ keys, BitmapReader key_valid,
                                                              const unsigned long long* __restrict__ vals, BitmapReader val_valid,
                                                              int64_t row0, int64_t n, int64_t step, unsigned long long kflip,
                                                              bool sample_values, bool vsigned, CompactStats* stats) {
  const unsigned long long vflip = vsigned ? 0x8000000000000000ull : 0ull;
  for (int64_t s = blockIdx.x * (int64_t)kBlock + threadIdx.x; s * step < n; s += (int64_t)gridDim.x * kBlock) {
    const int64_t i = row0 + s * step;
    if (key_valid.bit(i)) {
      const unsigned long long e = load_key_bits(keys, KW, i) ^ kflip;
      atomicMin(&stats->kmin, e);
      atomicMax(&stats->kmax, e);
    } else {
      atomicAdd(&stats->null_keys, 1ull);
    }
    if (sample_values && val_valid.bit(i)) {
      const unsigned long long v = vals[i] ^ vflip;
      atomicMin(&stats->vmin, v);
      atomicMax(&stats->vmax, v);
      atomicAdd(&stats->sampled, 1ull);
    }
  }
}

// zero-extended element `i` of a column of `width` bytes, loaded with an L2 cache policy
__device__ __forceinline__ unsigned long long load_bits_hint(const void* p, int width, int64_t i, uint64_t pol) {
  switch (width) {
    case 1: return ld_hint<uint8_t>(static_cast<const uint8_t*>(p) + i, pol);
    case 2: return ld_hint<uint16_t>(static_cast<const uint16_t*>(p) + i, pol);
    case 4: return ld_hint<uint32_t>(static_cast<const uint32_t*>(p) + i, pol);
    default: return ld_hint<uint64_t>(static_cast<const uint64_t*>(p) + i, pol);
  }
}
__device__ __forceinline__ unsigned long long sign_extend_bits(unsigned long long v, int width) {
  const int sh = 64 - 8 * width;
  return static_cast<unsigned long long>(static_cast<long long>(v << sh) >> sh);
}
// fire-and-forget 64-bit reduction that asks L2 to keep the line (the packed table is the hot working set)
__device__ __forceinline__ void red_add_u64_keep(unsigned long long* p, unsigned long long v, uint64_t pol) {
  asm volatile("red.relaxed.gpu.global.add.L2::cache_hint.u64 [%0], %1, %2;" ::"l"(p), "l"(v), "l"(pol) : "memory");
}

template <int KW, int VW>
__global__ void __launch_bounds__(kBlock) dense_consume_kernel(DenseArgs a) {
  const int kw = KW ? KW : a.kw, vw = VW ? VW : a.vw;
  // the two columns stream through once (evict-first); the packed table is hit by every row (evict-last): without the
  // hints the streamed input evicts the table and every reduction turns into dirty write-backs
  const uint64_t pol_stream = l2_policy_evict_first();
  const uint64_t pol_table = l2_policy_evict_last();
  const unsigned long long vmask = (1ull << a.vb) - 1ull;
  const unsigned long long one = 1ull << a.sb;
  unsigned long long null_sum = 0, null_cnt = 0, null_rows = 0;
  constexpr int U = 4;
  const int64_t stride = (int64_t)gridDim.x * kBlock * U;
  for (int64_t base = (int64_t)blockIdx.x * kBlock * U; base < a.n; base += stride) {
    unsigned long long k[U], v[U];
    bool ok[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = base + u * kBlock + threadIdx.x;
      ok[u] = i < a.n;
      k[u] = ok[u] ? load_bits_hint(a.keys, kw, i, pol_stream) : 0ull;
      v[u] = ok[u] ? load_bits_hint(a.vals, vw, i, pol_stream) : 0ull;
      if (a.vsigned && vw < 8) v[u] = sign_extend_bits(v[u], vw);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (!ok[u]) continue;
      const int64_t i = base + u * kBlock + threadIdx.x;
      const bool vv = a.val_valid.bit(a.row0 + i);
      if (!a.key_valid.bit(a.row0 + i)) {
        if (a.band_lo == 0) {  // counted by the first band only
          ++null_rows;
          if (vv) {
            null_sum += v[u];
            ++null_cnt;
          }
        }
        continue;
      }
      const unsigned long long idx = (k[u] ^ a.kflip) - a.kmin;  // wraps to a huge value for keys below kmin
      if (idx >= a.range) {  // outside the sampled key window: the host redoes the batch on the partitioned path
        atomicOr(a.overflow, 1u);
        continue;
      }
      if (idx < a.band_lo || idx >= a.band_hi) continue;
      if (vv) {
        const unsigned long long vp = v[u] - a.vbase;
        if (vp & ~vmask) {
          atomicOr(a.overflow, 1u);
          continue;
        }
        red_add_u64_keep(&a.table[idx], one | vp, pol_table);
      } else {
        atomicOr(&a.exists[idx >> 5], 1u << (idx & 31));
      }
    }
  }
  null_sum = static_cast<unsigned long long>(block_sum<kBlock>(static_cast<int64_t>(null_sum)));
  __syncthreads();
  null_cnt = static_cast<unsigned long long>(block_sum<kBlock>(static_cast<int64_t>(null_cnt)));
  __syncthreads();
  null_rows = static_cast<unsigned long long>(block_sum<kBlock>(static_cast<int64_t>(null_rows)));
  if (threadIdx.x == 0 && null_rows) {
    atomicAdd(&a.null_acc[0], null_sum);
    atomicAdd(&a.null_acc[1], null_cnt);
    atomicAdd(&a.null_acc[2], null_rows);
  }
}

// largest count field in the packed table: the drain after a sub-batch is only NEEDED when the next sub-batch could push
// a count past its m + 1 bits, i.e. when max_count + rows_of_next_sub_batch >= 2^(m+1) (for keys spread over many groups it never is)
__global__ void __launch_bounds__(kBlock) dense_maxcount_kernel(const unsigned long long* __restrict__ table, unsigned long long range, int sb,
                                                                unsigned long long* max_count) {
  unsigned long long m = 0;
  for (unsigned long long i = blockIdx.x * (unsigned long long)kBlock + threadIdx.x; i < range; i += (unsigned long long)gridDim.x * kBlock) {
    const unsigned long long c = table[i] >> sb;
    m = c > m ? c : m;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long v = __shfl_down_sync(0xffffffffu, m, o);
    m = v > m ? v : m;
  }
  if (lane_id() == 0 && m) atomicMax(max_count, m);
}

// packed words accumulated so far -> 64-bit sums (of the real values) and counts; the packed table is zeroed again.
// `guard` != NULL: skip the whole pass unless *guard + next_rows could overflow a count field (see dense_maxcount_kernel).
__global__ void __launch_bounds__(kBlock) dense_drain_kernel(unsigned long long* table, unsigned long long range, int sb,
                                                             unsigned long long vbase, unsigned long long* sums,
                                                             unsigned long long* counts, const unsigned long long* guard,
                                                             unsigned long long next_rows, unsigned long long limit) {
  if (guard && *guard + next_rows < limit) return;
  const unsigned long long smask = (1ull << sb) - 1ull;
  for (unsigned long long i = blockIdx.x * (unsigned long long)kBlock + threadIdx.x; i < range; i += (unsigned long long)gridDim.x * kBlock) {
    const unsigned long long p = table[i];
    if (!p) continue;
    const unsigned long long c = p >> sb;
    sums[i] += (p & smask) + c * vbase;  // sum of the values = sum of the offsets + count x base (mod 2^64)
    counts[i] += c;
    table[i] = 0;
  }
}

// dense state -> the global table (one insert per existing group)
__global__ void __launch_bounds__(kBlock) dense_flush_kernel(const unsigned long long* sums, const unsigned long long* counts,
                                                             const uint32_t* exists, unsigned long long range, unsigned long long kmin,
                                                             unsigned long long kflip, FusedTableRef table, unsigned long long* counters) {
  for (unsigned long long i = blockIdx.x * (unsigned long long)kBlock + threadIdx.x; i < range; i += (unsigned long long)gridDim.x * kBlock) {
    const unsigned long long c = counts[i];
    if (c == 0 && !((exists[i >> 5] >> (i & 31)) & 1u)) continue;
    // counts above 2^32 - 1 per group and batch are added in two steps (global_accumulate takes a 32-bit count)
    unsigned long long rest = c;
    bool first = true;
    do {
      const unsigned step = rest > 0xffffffffull ? 0xffffffffu : static_cast<unsigned>(rest);
      global_accumulate<false>(table, (i + kmin) ^ kflip, false, first ? sums[i] : 0ull, step, counters);
      rest -= step;
      first = false;
    } while (rest);
  }
}

// chunk state -> the object's persistent dense state (same window): element-wise add / or
__global__ void __launch_bounds__(kBlock) dense_merge_kernel(unsigned long long* sums, unsigned long long* counts, uint32_t* exists,
                                                             const unsigned long long* add_sums, const unsigned long long* add_counts,
                                                             const uint32_t* add_exists, unsigned long long range) {
  for (unsigned long long i = blockIdx.x * (unsigned long long)kBlock + threadIdx.x; i < range; i += (unsigned long long)gridDim.x * kBlock) {
    const unsigned long long c = add_counts[i];
    if (c) {
      sums[i] += add_sums[i];
      counts[i] += c;
    }
    if ((i & 31) == 0) {
      const uint32_t e = add_exists[i >> 5];
      if (e) exists[i >> 5] |= e;
    }
  }
}

// out[0] = existing groups, out[1] = groups whose count is 0 (their sum is null)
__global__ void __launch_bounds__(kBlock) dense_count_kernel(const unsigned long long* counts, const uint32_t* exists, unsigned long long range,
                                                             int64_t* out) {
  int64_t groups = 0, empty = 0;
  for (unsigned long long i = blockIdx.x * (unsigned long long)kBlock + threadIdx.x; i < range; i += (unsigned long long)gridDim.x * kBlock) {
    const bool has = counts[i] != 0;
    const bool ex = has || ((exists[i >> 5] >> (i & 31)) & 1u);
    groups += ex;
    empty += ex && !has;
  }
  groups = block_sum<kBlock>(groups);
  __syncthreads();
  empty = block_sum<kBlock>(empty);
  if (threadIdx.x == 0) {
    if (groups) atomicAdd(reinterpret_cast<unsigned long long*>(out), (unsigned long long)groups);
    if (empty) atomicAdd(reinterpret_cast<unsigned long long*>(out + 1), (unsigned long long)empty);
  }
}

// dense state -> output columns directly (no hash table involved): existing slots are compacted with one atomic
// ticket per warp; the null-key group, if any, is appended by thread 0 of block 0 at row `n_dense`
__global__ void __launch_bounds__(kBlock) dense_emit_kernel(const unsigned long long* sums, const unsigned long long* counts,
                                                            const uint32_t* exists, unsigned long long range, unsigned long long kmin,
                                                            unsigned long long kflip, int key_width, void* out_keys, uint32_t* key_validity,
                                                            unsigned long long* out_sums, uint32_t* sum_validity, long long* out_counts,
                                                            unsigned long long* ticket, int has_null, unsigned long long null_sum,
                                                            unsigned long long null_cnt, unsigned long long n_dense) {
  auto put_key = [&](unsigned long long g, unsigned long long kv) {
    switch (key_width) {
      case 1: static_cast<uint8_t*>(out_keys)[g] = static_cast<uint8_t>(kv); break;
      case 2: static_cast<uint16_t*>(out_keys)[g] = static_cast<uint16_t>(kv); break;
      case 4: static_cast<uint32_t*>(out_keys)[g] = static_cast<uint32_t>(kv); break;
      default: static_cast<uint64_t*>(out_keys)[g] = kv; break;
    }
  };
  if (has_null && blockIdx.x == 0 && threadIdx.x == 0) {
    put_key(n_dense, 0ull);
    out_sums[n_dense] = null_sum;
    out_counts[n_dense] = static_cast<long long>(null_cnt);
    atomicAnd(&key_validity[n_dense >> 5], ~(1u << (n_dense & 31)));
    if (null_cnt == 0) atomicAnd(&sum_validity[n_dense >> 5], ~(1u << (n_dense & 31)));
  }
  for (unsigned long long base = (blockIdx.x * (unsigned long long)kBlock + threadIdx.x) & ~31ull; base < range;
       base += (unsigned long long)gridDim.x * kBlock) {
    const unsigned long long i = base + lane_id();
    unsigned long long c = 0;
    bool ex = false;
    if (i < range) {
      c = counts[i];
      ex = c != 0 || ((exists[i >> 5] >> (i & 31)) & 1u);
    }
    const unsigned m = __ballot_sync(0xffffffffu, ex);
    if (m == 0) continue;
    unsigned long long start = 0;
    if (lane_id() == 0) start = atomicAdd(ticket, (unsigned long long)__popc(m));
    start = __shfl_sync(0xffffffffu, start, 0);
    if (ex) {
      const unsigned long long g = start + __popc(m & lanemask_lt());
      put_key(g, (i + kmin) ^ kflip);
      out_sums[g] = c ? sums[i] : 0ull;
      out_counts[g] = static_cast<long long>(c);
      if (c == 0) atomicAnd(&sum_validity[g >> 5], ~(1u << (g & 31)));
    }
  }
}

// the null-key group's partial state (host values) -> the global table
__global__ void dense_null_flush_kernel(FusedTableRef table, unsigned long long null_sum, unsigned long long null_cnt, unsigned long long* counters) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    unsigned long long rest = null_cnt;
    bool first = true;
    do {
      const unsigned step = rest > 0xffffffffull ? 0xffffffffu : static_cast<unsigned>(rest);
      global_accumulate<false>(table, 0ull, true, first ? null_sum : 0ull, step, counters);
      rest -= step;
      first = false;
    } while (rest);
  }
}

}  // namespace b2
