// hash_join.cu -- equi-join of two key column sets: the matching (left row, right row) pairs.
//
// Replaces the match / materialize core of HashJoinNode (acero/hash_join_node.cc, acero/swiss_join.cc: build a SwissTable
// over the build side's row-encoded keys, probe it with the other side, emit row-id pairs that the node then uses to Take
// the payload columns) for INNER / LEFT OUTER / FULL OUTER / LEFT SEMI / LEFT ANTI joins with equality keys (JoinKeyCmp::EQ,
// acero/options.h:384-392: a null key matches nothing); the RIGHT variants are the same joins with the sides swapped.
//
// Design: the join is the Grouper plus three streaming passes -- no second hash table and no per-row chains.
//   build : Grouper::Consume on the RIGHT keys gives every right row a dense group id; a per-id COUNT (only rows whose
//           keys are all valid) and its exclusive scan lay out one contiguous run per id, and a stable radix sort of the
//           ids (b2_sort_indices) is the right rows in run order;
//   probe : Grouper::Lookup on the LEFT keys gives each left row its id or "unknown"; its match count is the run length;
//   emit  : an exclusive scan of the per-row output counts (tile sums + one scan block + tile-local scans) places every
//           left row's pairs; one thread per left row writes them -- left rows in row order, their right matches in row
//           order, so the result is deterministic (the reference's order depends on thread scheduling).
// Keys are whatever the Grouper takes: numeric, utf8 / binary, any number of columns and total width.
// JoinKeyCmp::IS (b2_hash_join_ex): the Grouper already gives a null key its own group, so an IS column only drops out of
// the key validity that excludes rows from matching.
// Residual filter (b2_join_residual): the caller evaluates the filter on the INNER pairs; one pass over the pairs counts the
// survivors per left row (and marks matched right rows for FULL OUTER), b2_filter compacts the surviving pairs, and for the
// outer joins two scans of the counts (max(count, 1) and count) place each survivor and each null-extended row.
#include <vector>

#include "bitmap.h"
#include "common.cuh"
#include "context.h"

namespace b2 {
namespace {

constexpr int kScanTile = 4096;
constexpr uint32_t kNoMatch = 0xffffffffu;

// per-row MATCH count of the probe side -> counts[i] (uint32; 0 = no partner) and the OUTPUT rows per 4096-row tile
// (an outer join emits one null-extended row for an unmatched probe row).  cnt32 is 4 bytes per group: 40 MB at 10M groups,
// L2-resident, where the 64-bit counts were not.
__global__ void __launch_bounds__(kBlock) probe_counts_kernel(const uint32_t* __restrict__ ids, BitmapReader ids_valid, BitmapReader keys_valid,
                                                              const uint32_t* __restrict__ cnt32, int64_t n, bool outer,
                                                              uint32_t* __restrict__ counts, int64_t* __restrict__ tile_sums) {
  const int64_t tile = blockIdx.x;
  int64_t local = 0;
  for (int r = threadIdx.x; r < kScanTile; r += kBlock) {
    const int64_t i = tile * kScanTile + r;
    if (i >= n) break;
    uint32_t c = 0;
    if (ids_valid.bit(i) && keys_valid.bit(i)) c = cnt32[ids[i]];
    counts[i] = c;
    local += (c == 0 && outer) ? 1 : static_cast<int64_t>(c);
  }
  const int64_t s = block_sum<kBlock>(local);
  if (threadIdx.x == 0) tile_sums[tile] = s;
}

// per group: cnt32[g] = its build rows (saturated), where32[g] = the build row itself when there is exactly one (the
// dimension-table case: the emit pass then needs ONE random access per probe row), else the start of its run in build_rows
__global__ void __launch_bounds__(kBlock) group_records_kernel(const unsigned long long* __restrict__ cnt, const int64_t* __restrict__ run_start,
                                                               const uint32_t* __restrict__ build_rows, int64_t groups,
                                                               uint32_t* __restrict__ cnt32, uint32_t* __restrict__ where32) {
  for (int64_t g = blockIdx.x * (int64_t)kBlock + threadIdx.x; g < groups; g += (int64_t)gridDim.x * kBlock) {
    const unsigned long long c = cnt[g];
    cnt32[g] = c > 0xffffffffull ? 0xffffffffu : static_cast<uint32_t>(c);
    if (where32) where32[g] = c == 0 ? 0u : (c == 1 ? build_rows[run_start[g]] : static_cast<uint32_t>(run_start[g]));
  }
}

// per-tile sums for the two-level exclusive scan: of the per-id counts (uint64, run_start[g]) and of the residual step's
// per-left-row survivor counts (uint32)
//   min_one: a zero counts as one (the null-extended row of an outer join)
template <typename In>
__global__ void __launch_bounds__(kBlock) tile_sums_kernel(const In* __restrict__ v, int64_t n, bool min_one, int64_t* __restrict__ tile_sums) {
  const int64_t tile = blockIdx.x;
  int64_t local = 0;
  for (int r = threadIdx.x; r < kScanTile; r += kBlock) {
    const int64_t i = tile * kScanTile + r;
    if (i < n) local += (min_one && v[i] == 0) ? 1 : static_cast<int64_t>(v[i]);
  }
  const int64_t s = block_sum<kBlock>(local);
  if (threadIdx.x == 0) tile_sums[tile] = s;
}

// tile-local exclusive scan (one thread block per tile, 16 consecutive elements per thread) + the tile's offset
//   min_one: a zero counts as one (the null-extended row of an outer join)
template <typename In>
__global__ void __launch_bounds__(kBlock) tile_scan_kernel(const In* __restrict__ v, int64_t n, const int64_t* __restrict__ tile_offsets,
                                                           int64_t* __restrict__ out, bool min_one) {
  __shared__ int64_t warp_tot[kBlock / 32];
  constexpr int kPer = kScanTile / kBlock;
  const int64_t tile = blockIdx.x;
  const int64_t i0 = tile * kScanTile + static_cast<int64_t>(threadIdx.x) * kPer;
  int64_t vals[kPer], sum = 0;
#pragma unroll
  for (int k = 0; k < kPer; ++k) {
    vals[k] = i0 + k < n ? static_cast<int64_t>(v[i0 + k]) : 0;
    if (min_one && i0 + k < n && vals[k] == 0) vals[k] = 1;
    sum += vals[k];
  }
  int64_t incl = sum;
  const unsigned lane = lane_id();
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t x = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += x;
  }
  if (lane == 31) warp_tot[threadIdx.x >> 5] = incl;
  __syncthreads();
  int64_t base = tile_offsets[tile];
  for (int w = 0; w < static_cast<int>(threadIdx.x >> 5); ++w) base += warp_tot[w];
  int64_t run = base + incl - sum;
#pragma unroll
  for (int k = 0; k < kPer; ++k) {
    if (i0 + k < n) out[i0 + k] = run;
    run += vals[k];
  }
}

// one thread per probe row: its pairs go to [row_off[i], row_off[i] + max(counts[i], outer)); the match count comes from the
// streamed counts[], so the only random accesses are where32[g] and -- for groups with several build rows -- their run
__global__ void __launch_bounds__(kBlock) emit_pairs_kernel(const uint32_t* __restrict__ ids, const uint32_t* __restrict__ counts,
                                                            const uint32_t* __restrict__ where32, const uint32_t* __restrict__ build_rows,
                                                            const int64_t* __restrict__ row_off, int64_t n, uint32_t* __restrict__ out_left,
                                                            uint32_t* __restrict__ out_right, bool outer) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const uint32_t c = counts[i];
    if (c == 0) {
      if (outer) {  // the null-extended row, marked for the validity pass (no row number reaches 2^32 - 16)
        const int64_t base = row_off[i];
        out_left[base] = static_cast<uint32_t>(i);
        out_right[base] = kNoMatch;
      }
      continue;
    }
    const int64_t base = row_off[i];
    const uint32_t w = where32[ids[i]];
    if (c == 1) {
      out_left[base] = static_cast<uint32_t>(i);
      out_right[base] = w;
      continue;
    }
    for (uint32_t k = 0; k < c; ++k) {
      out_left[base + k] = static_cast<uint32_t>(i);
      out_right[base + k] = build_rows[static_cast<int64_t>(w) + k];
    }
  }
}

// LEFT OUTER: validity of the right indices = "not the marker"; the marker is replaced by 0; one ballot per 32 pairs
__global__ void __launch_bounds__(kBlock) right_validity_kernel(uint32_t* __restrict__ out_right, int64_t n, uint32_t* __restrict__ validity,
                                                                int64_t* valid_count) {
  const int64_t nw = (n + 31) >> 5;
  int64_t local = 0;
  for (int64_t w = (blockIdx.x * (int64_t)kBlock + threadIdx.x) >> 5; w < nw; w += ((int64_t)gridDim.x * kBlock) >> 5) {
    const int64_t i = (w << 5) + lane_id();
    bool ok = false;
    if (i < n) {
      ok = out_right[i] != kNoMatch;
      if (!ok) out_right[i] = 0;
    }
    const unsigned word = __ballot_sync(0xffffffffu, ok);
    if (lane_id() == 0) {
      validity[w] = word;
      local += __popc(word);
    }
  }
  const int64_t s = block_sum<kBlock>(local);
  if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(valid_count), (unsigned long long)s);
}

// bit i = probe row i has (SEMI) / has no (ANTI) match
__global__ void __launch_bounds__(kBlock) semi_mask_kernel(const uint32_t* __restrict__ ids, BitmapReader ids_valid, BitmapReader keys_valid,
                                                           const unsigned long long* __restrict__ cnt, int64_t n, bool anti, uint32_t* __restrict__ mask) {
  const int64_t nw = (n + 31) >> 5;
  for (int64_t w = (blockIdx.x * (int64_t)kBlock + threadIdx.x) >> 5; w < nw; w += ((int64_t)gridDim.x * kBlock) >> 5) {
    const int64_t i = (w << 5) + lane_id();
    bool hit = false;
    if (i < n) {
      const bool m = ids_valid.bit(i) && keys_valid.bit(i) && cnt[ids[i]] > 0;
      hit = anti ? !m : m;
    }
    const unsigned word = __ballot_sync(0xffffffffu, hit);
    if (lane_id() == 0) mask[w] = word;
  }
}

// FULL OUTER: matched[g] = 1 for every group some probe row hits (idempotent byte stores, no atomics)
__global__ void __launch_bounds__(kBlock) mark_matched_kernel(const uint32_t* __restrict__ ids, BitmapReader ids_valid, BitmapReader keys_valid,
                                                              int64_t n, uint8_t* matched) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock)
    if (ids_valid.bit(i) && keys_valid.bit(i)) matched[ids[i]] = 1;
}

// FULL OUTER: bit r = build row r found no partner (its key has a null, or no probe row hit its group)
__global__ void __launch_bounds__(kBlock) unmatched_build_kernel(const uint32_t* __restrict__ ids, BitmapReader keys_valid, const uint8_t* __restrict__ matched,
                                                                 int64_t n, uint32_t* __restrict__ mask) {
  const int64_t nw = (n + 31) >> 5;
  for (int64_t w = (blockIdx.x * (int64_t)kBlock + threadIdx.x) >> 5; w < nw; w += ((int64_t)gridDim.x * kBlock) >> 5) {
    const int64_t i = (w << 5) + lane_id();
    const bool lonely = i < n && !(keys_valid.bit(i) && matched[ids[i]]);
    const unsigned word = __ballot_sync(0xffffffffu, lonely);
    if (lane_id() == 0) mask[w] = word;
  }
}

// FULL OUTER: the tail of the result = (null, unmatched build row); validity of both index columns over the whole result
__global__ void __launch_bounds__(kBlock) full_outer_finish_kernel(uint32_t* __restrict__ out_left, uint32_t* __restrict__ out_right,
                                                                   const uint32_t* __restrict__ lonely_rows, int64_t head, int64_t n,
                                                                   uint32_t* __restrict__ left_validity, uint32_t* __restrict__ right_validity,
                                                                   int64_t* right_valid_count) {
  const int64_t nw = (n + 31) >> 5;
  int64_t local = 0;
  for (int64_t w = (blockIdx.x * (int64_t)kBlock + threadIdx.x) >> 5; w < nw; w += ((int64_t)gridDim.x * kBlock) >> 5) {
    const int64_t i = (w << 5) + lane_id();
    bool lv = false, rv = false;
    if (i < n) {
      if (i < head) {
        lv = true;
        rv = out_right[i] != kNoMatch;
        if (!rv) out_right[i] = 0;
      } else {
        out_left[i] = 0;
        out_right[i] = lonely_rows[i - head];
        rv = true;
      }
    }
    const unsigned lw = __ballot_sync(0xffffffffu, lv), rw = __ballot_sync(0xffffffffu, rv);
    if (lane_id() == 0) {
      left_validity[w] = lw;
      right_validity[w] = rw;
      local += __popc(rw);
    }
  }
  const int64_t s = block_sum<kBlock>(local);
  if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(right_valid_count), (unsigned long long)s);
}

// ---- residual step (b2_join_residual): the caller's candidate pairs and its keep flags -> the join's result ----
constexpr unsigned long long kBadLeft = 1, kBadRight = 2, kBadOrder = 4;

// one warp per 32 candidate pairs: the survivor word (keep AND its validity), the survivors per left row (pairs come sorted
// by left row, so one atomic per run of equal left rows in the word), FULL OUTER's mark per right row, the survivor total
// (stats[0]) and the checks of the caller's pairs: an index out of range or a left row below the one before sets a bit of
// stats[1], and such an index is never used as an address
__global__ void __launch_bounds__(kBlock) residual_count_kernel(const uint32_t* __restrict__ cl, const uint32_t* __restrict__ cr, BitmapReader keep,
                                                                BitmapReader keep_valid, int64_t m, int64_t n_left, int64_t n_right,
                                                                uint32_t* __restrict__ survivors, uint32_t* __restrict__ counts,
                                                                uint8_t* __restrict__ matched, int64_t* stats) {
  const int64_t nw = (m + 31) >> 5;
  const unsigned lane = lane_id();
  int64_t local = 0;
  unsigned long long bad = 0;
  for (int64_t w = (blockIdx.x * (int64_t)kBlock + threadIdx.x) >> 5; w < nw; w += ((int64_t)gridDim.x * kBlock) >> 5) {
    const int64_t i = (w << 5) + lane;
    const bool in = i < m;
    const uint32_t l = in ? cl[i] : 0xffffffffu, r = in ? cr[i] : 0u;
    uint32_t prev = __shfl_up_sync(0xffffffffu, l, 1);
    if (lane == 0) prev = (in && i > 0) ? cl[i - 1] : 0u;
    const bool l_ok = in && l < n_left, r_ok = in && r < n_right;
    if (in && !l_ok) bad |= kBadLeft;
    if (in && !r_ok) bad |= kBadRight;
    if (in && prev > l) bad |= kBadOrder;
    const uint32_t word = keep.word32(w) & keep_valid.word32(w);  // bits at or past m read as 0
    const unsigned heads = __ballot_sync(0xffffffffu, in && (lane == 0 || l != prev));
    if ((heads >> lane) & 1) {  // the first lane of a run of equal left rows counts the run's survivors
      const unsigned later = lane == 31 ? 0u : heads & ~((2u << lane) - 1u);
      const unsigned upto = later ? (1u << (__ffs(later) - 1)) - 1u : 0xffffffffu;
      const int c = __popc(word & upto & ~((1u << lane) - 1u));
      if (c && l_ok) atomicAdd(counts + l, static_cast<uint32_t>(c));
    }
    if (matched && r_ok && ((word >> lane) & 1)) matched[r] = 1;
    if (lane == 0) {
      survivors[w] = word;
      local += __popc(word);
    }
  }
  bad = __reduce_or_sync(0xffffffffu, static_cast<unsigned>(bad));
  if (lane == 0 && bad) atomicOr(reinterpret_cast<unsigned long long*>(stats + 1), bad);
  const int64_t s = block_sum<kBlock>(local);
  if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(stats), (unsigned long long)s);
}

// bit i = v[i] is zero (want_zero) / non-zero: SEMI / ANTI from the survivor counts, FULL OUTER's lonely right rows
template <typename T>
__global__ void __launch_bounds__(kBlock) zero_mask_kernel(const T* __restrict__ v, int64_t n, bool want_zero, uint32_t* __restrict__ mask) {
  const int64_t nw = (n + 31) >> 5;
  for (int64_t w = (blockIdx.x * (int64_t)kBlock + threadIdx.x) >> 5; w < nw; w += ((int64_t)gridDim.x * kBlock) >> 5) {
    const int64_t i = (w << 5) + lane_id();
    const unsigned word = __ballot_sync(0xffffffffu, i < n && (v[i] == 0) == want_zero);
    if (lane_id() == 0) mask[w] = word;
  }
}

// LEFT / FULL OUTER emit: compacted survivor j of left row l goes to row_off[l] + (j - first[l]); a left row without a
// survivor gets its null-extended row at row_off[l].  Items [0, k) are the survivors, [k, k + n_left) the left rows.
__global__ void __launch_bounds__(kBlock) residual_emit_kernel(const uint32_t* __restrict__ kept_left, const uint32_t* __restrict__ kept_right, int64_t k,
                                                               const uint32_t* __restrict__ counts, const int64_t* __restrict__ first,
                                                               const int64_t* __restrict__ row_off, int64_t n_left, uint32_t* __restrict__ out_left,
                                                               uint32_t* __restrict__ out_right) {
  for (int64_t t = blockIdx.x * (int64_t)kBlock + threadIdx.x; t < k + n_left; t += (int64_t)gridDim.x * kBlock) {
    if (t < k) {
      const uint32_t l = kept_left[t];
      const int64_t pos = row_off[l] + (t - first[l]);
      out_left[pos] = l;
      out_right[pos] = kept_right[t];
    } else {
      const int64_t l = t - k;
      if (counts[l] == 0) {
        out_left[row_off[l]] = static_cast<uint32_t>(l);
        out_right[row_off[l]] = kNoMatch;
      }
    }
  }
}

// AND of the validity bitmaps of the key columns whose nulls match nothing (JoinKeyCmp::EQ; null_equal[j] != 0 marks an
// IS column, where a null equals a null and the Grouper's own null group does the matching), re-based to bit 0;
// *out = NULL when none of those columns has nulls
int keys_validity(B2Context* ctx, const B2Array* keys, int n_keys, const uint8_t* null_equal, int64_t n, Temp* bits, const void** out,
                  cudaStream_t s) {
  *out = nullptr;
  auto counts = [&](int j) { return keys[j].null_count != 0 && keys[j].validity && !(null_equal && null_equal[j]); };
  bool any = false;
  for (int j = 0; j < n_keys; ++j) any = any || counts(j);
  if (!any || n == 0) return B2_OK;
  B2_RETURN_NOT_OK(bits->alloc(bitmap_alloc_bytes(n)));
  B2_CUDA(cudaMemsetAsync(bits->ptr, 0xff, bitmap_alloc_bytes(n), s));
  for (int j = 0; j < n_keys; ++j) {
    if (!counts(j)) continue;
    B2_RETURN_NOT_OK(launch_bitmap_and(bits->ptr, 0, keys[j].validity, keys[j].offset, n, bits->ptr, nullptr, s));
  }
  *out = bits->ptr;
  return B2_OK;
}

// the set rows of an n-bit mask as uint32 row numbers (b2_filter_indices returns uint16 for short masks)
int mask_rows_u32(B2Context* ctx, const void* bits, int64_t n, PoolArray* out, cudaStream_t s) {
  B2Array m{};
  m.type = B2_BOOL;
  m.data = bits;
  m.length = n;
  PoolArray rows(ctx, s);
  B2_RETURN_NOT_OK(b2_filter_indices(ctx, &m, 0, &rows.a, s));
  if (rows.a.type == B2_UINT32 || rows.a.length == 0) {
    out->take_from(rows);
    out->a.type = B2_UINT32;
    return B2_OK;
  }
  B2CastOptions wide{B2_UINT32, 1, 1, 0};
  out->reset();
  return b2_cast_numeric(ctx, &rows.a, &wide, &out->a, s);
}

// outer joins: the validity of the index columns (the unmatched marker becomes a null slot; FULL OUTER also appends the
// lonely right rows after the first `head` pairs), then the result arrays
int finish_outer(B2Context* ctx, Temp* ol, Temp* orr, const PoolArray& lonely, int64_t head, int64_t total, bool full, B2Array* out_left,
                 B2Array* out_right, cudaStream_t s) {
  Temp obits(ctx, s), lbits(ctx, s);
  B2_RETURN_NOT_OK(obits.alloc(bitmap_alloc_bytes(total)));
  B2_CUDA(cudaMemsetAsync(obits.ptr, 0, bitmap_alloc_bytes(total), s));
  if (full) {
    B2_RETURN_NOT_OK(lbits.alloc(bitmap_alloc_bytes(total)));
    B2_CUDA(cudaMemsetAsync(lbits.ptr, 0, bitmap_alloc_bytes(total), s));
  }
  int64_t right_nulls = 0;
  if (total > 0) {
    ScalarSlot vs(ctx);
    B2_RETURN_NOT_OK(vs.zero(s));
    if (full) {
      full_outer_finish_kernel<<<grid_for(total, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(
          ol->as<uint32_t>(), orr->as<uint32_t>(), static_cast<const uint32_t*>(lonely.a.data), head, total, lbits.as<uint32_t>(),
          obits.as<uint32_t>(), vs.dev());
    } else {
      right_validity_kernel<<<grid_for(total, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(orr->as<uint32_t>(), total, obits.as<uint32_t>(), vs.dev());
    }
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(vs.fetch(s));
    right_nulls = total - vs.host()[0];
  }
  const int64_t left_nulls = full ? total - head : 0;
  fill_out(out_left, B2_UINT32, total, left_nulls, left_nulls ? lbits.release() : nullptr, ol->release());
  fill_out(out_right, B2_UINT32, total, right_nulls, right_nulls ? obits.release() : nullptr, orr->release());
  return B2_OK;
}

struct GrouperGuard {
  B2Grouper* g = nullptr;
  ~GrouperGuard() {
    if (g) b2_grouper_destroy(g);
  }
};
struct AggGuard {
  B2HashAgg* a = nullptr;
  ~AggGuard() {
    if (a) b2_hashagg_destroy(a);
  }
};

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" int b2_hash_join(B2Context* ctx, const B2Array* left_keys, const B2Array* right_keys, int n_keys, int join_type,
                            B2Array* out_left, B2Array* out_right, void* stream) {
  return b2_hash_join_ex(ctx, left_keys, right_keys, n_keys, nullptr, join_type, out_left, out_right, stream);
}

extern "C" int b2_hash_join_ex(B2Context* ctx, const B2Array* left_keys, const B2Array* right_keys, int n_keys, const uint8_t* null_equal,
                               int join_type, B2Array* out_left, B2Array* out_right, void* stream) {
  if (!ctx || !left_keys || !right_keys || !out_left) return set_error(B2_INVALID, "b2_hash_join: null argument");
  if (join_type < B2_JOIN_INNER || join_type > B2_JOIN_FULL_OUTER) return set_error(B2_NOT_IMPLEMENTED, "b2_hash_join: join type %d", join_type);
  const bool full = join_type == B2_JOIN_FULL_OUTER;
  const bool pairs = join_type == B2_JOIN_INNER || join_type == B2_JOIN_LEFT_OUTER || full;
  if (pairs && !out_right) return set_error(B2_INVALID, "b2_hash_join: this join type returns right indices too");
  if (n_keys < 1) return set_error(B2_INVALID, "b2_hash_join: at least one key column");
  const int64_t nl = left_keys[0].length, nr = right_keys[0].length;
  for (int j = 0; j < n_keys; ++j) {
    if (left_keys[j].type != right_keys[j].type)
      return set_error(B2_TYPE_ERROR, "b2_hash_join: key %d has type id %d on the left and %d on the right", j, left_keys[j].type, right_keys[j].type);
    if (left_keys[j].length != nl || right_keys[j].length != nr) return set_error(B2_INVALID, "b2_hash_join: key columns differ in length");
  }
  if (nl > 0xfffffff0ll || nr > 0xfffffff0ll) return set_error(B2_NOT_IMPLEMENTED, "b2_hash_join: sides of 2^32 rows or more must be split");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));

  // ---- build: ids, per-id counts of the rows with fully valid keys, run starts, rows in run order ----
  std::vector<int32_t> types(n_keys);
  for (int j = 0; j < n_keys; ++j) types[j] = right_keys[j].type;
  GrouperGuard gg;
  B2_RETURN_NOT_OK(b2_grouper_create(ctx, types.data(), n_keys, &gg.g));
  PoolArray rids(ctx, s), lids(ctx, s);
  B2_RETURN_NOT_OK(b2_grouper_consume(gg.g, right_keys, &rids.a, s));
  uint32_t groups = 0;
  B2_RETURN_NOT_OK(b2_grouper_num_groups(gg.g, &groups));
  Temp rvalid_bits(ctx, s), lvalid_bits(ctx, s);
  const void *rvalid = nullptr, *lvalid = nullptr;
  B2_RETURN_NOT_OK(keys_validity(ctx, right_keys, n_keys, null_equal, nr, &rvalid_bits, &rvalid, s));
  B2_RETURN_NOT_OK(keys_validity(ctx, left_keys, n_keys, null_equal, nl, &lvalid_bits, &lvalid, s));

  // counts per id: hash_count over "values" that carry only the key validity
  AggGuard counter;
  B2HashAggOptions co{1, 0, /*ONLY_VALID=*/0, 0};
  B2_RETURN_NOT_OK(b2_hashagg_create(ctx, B2_HASH_COUNT, B2_BOOL, &co, &counter.a));
  B2_RETURN_NOT_OK(b2_hashagg_resize(counter.a, groups, s));
  B2Array marker{};
  marker.type = B2_BOOL;
  marker.length = nr;
  marker.validity = rvalid;
  marker.null_count = rvalid ? -1 : 0;
  marker.data = rids.a.data;  // never read: hash_count of a non-numeric column looks at the validity only
  if (nr > 0) B2_RETURN_NOT_OK(b2_hashagg_consume(counter.a, &marker, &rids.a, s));
  PoolArray cnt(ctx, s);
  B2_RETURN_NOT_OK(b2_hashagg_finalize(counter.a, &cnt.a, s));  // int64 counts, one per id
  const unsigned long long* d_cnt = static_cast<const unsigned long long*>(cnt.a.data);

  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  Temp run_start(ctx, s), build_rows(ctx, s), cnt32(ctx, s), where32(ctx, s);
  if (pairs) {
    const int64_t g_tiles = (static_cast<int64_t>(groups) + kScanTile - 1) / kScanTile;
    Temp g_sums(ctx, s), g_offs(ctx, s);
    B2_RETURN_NOT_OK(run_start.alloc(sizeof(int64_t) * (size_t)(groups ? groups : 1)));
    B2_RETURN_NOT_OK(g_sums.alloc(sizeof(int64_t) * (size_t)(g_tiles ? g_tiles : 1)));
    B2_RETURN_NOT_OK(g_offs.alloc(sizeof(int64_t) * (size_t)(g_tiles ? g_tiles : 1)));
    if (groups) {
      tile_sums_kernel<unsigned long long><<<(unsigned)g_tiles, kBlock, 0, s>>>(d_cnt, groups, false, g_sums.as<int64_t>());
      B2_LAUNCHED();
      B2_RETURN_NOT_OK(launch_exclusive_scan_i64(g_sums.as<int64_t>(), g_tiles, g_offs.as<int64_t>(), nullptr, s));
      tile_scan_kernel<unsigned long long><<<(unsigned)g_tiles, kBlock, 0, s>>>(d_cnt, groups, g_offs.as<int64_t>(), run_start.as<int64_t>(), false);
      B2_LAUNCHED();
    }
    // right rows grouped by id (stable), rows with a null key last: the radix sort of the ids with the key validity as theirs
    B2Array sortable = rids.a;
    sortable.validity = rvalid;
    sortable.null_count = rvalid ? -1 : 0;
    PoolArray order(ctx, s);
    B2_RETURN_NOT_OK(b2_sort_indices(ctx, &sortable, 0, /*AtEnd=*/1, &order.a, s));
    B2CastOptions narrow{B2_UINT32, 1, 1, 0};
    PoolArray order32(ctx, s);
    B2_RETURN_NOT_OK(b2_cast_numeric(ctx, &order.a, &narrow, &order32.a, s));
    build_rows.ptr = const_cast<void*>(order32.a.data);
    order32.a.data = nullptr;
    B2_RETURN_NOT_OK(cnt32.alloc(sizeof(uint32_t) * (size_t)(groups ? groups : 1)));
    B2_RETURN_NOT_OK(where32.alloc(sizeof(uint32_t) * (size_t)(groups ? groups : 1)));
    if (groups) {
      group_records_kernel<<<grid_for(groups, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(d_cnt, run_start.as<int64_t>(), build_rows.as<uint32_t>(), groups,
                                                                               cnt32.as<uint32_t>(), where32.as<uint32_t>());
      B2_LAUNCHED();
    }
  }

  // ---- probe ----
  B2_RETURN_NOT_OK(b2_grouper_lookup(gg.g, left_keys, &lids.a, s));
  const uint32_t* d_lids = static_cast<const uint32_t*>(lids.a.data);
  const BitmapReader lid_valid(lids.a.null_count == 0 ? nullptr : lids.a.validity, 0, nl);
  const BitmapReader lkey_valid(lvalid, 0, nl);

  if (!pairs) {  // SEMI / ANTI: a mask over the left rows, then their row numbers
    Temp mask(ctx, s);
    B2_RETURN_NOT_OK(mask.alloc(bitmap_alloc_bytes(nl)));
    B2_CUDA(cudaMemsetAsync(mask.ptr, 0, bitmap_alloc_bytes(nl), s));
    if (nl > 0) {
      semi_mask_kernel<<<grid_for(nl, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(d_lids, lid_valid, lkey_valid, d_cnt, nl,
                                                                            join_type == B2_JOIN_LEFT_ANTI, mask.as<uint32_t>());
      B2_LAUNCHED();
    }
    PoolArray rows(ctx, s);
    B2_RETURN_NOT_OK(mask_rows_u32(ctx, mask.ptr, nl, &rows, s));
    rows.give(out_left);
    return B2_OK;
  }

  // ---- emit ----
  const bool outer = join_type == B2_JOIN_LEFT_OUTER || full;
  const int64_t l_tiles = (nl + kScanTile - 1) / kScanTile;
  Temp counts(ctx, s), l_sums(ctx, s), l_offs(ctx, s), row_off(ctx, s);
  B2_RETURN_NOT_OK(counts.alloc(sizeof(uint32_t) * (size_t)(nl ? nl : 1)));
  B2_RETURN_NOT_OK(l_sums.alloc(sizeof(int64_t) * (size_t)(l_tiles ? l_tiles : 1)));
  B2_RETURN_NOT_OK(l_offs.alloc(sizeof(int64_t) * (size_t)(l_tiles ? l_tiles : 1)));
  B2_RETURN_NOT_OK(row_off.alloc(sizeof(int64_t) * (size_t)(nl ? nl : 1)));
  int64_t total = 0;
  if (nl > 0) {
    probe_counts_kernel<<<(unsigned)l_tiles, kBlock, 0, s>>>(d_lids, lid_valid, lkey_valid, cnt32.as<uint32_t>(), nl, outer, counts.as<uint32_t>(),
                                                            l_sums.as<int64_t>());
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(launch_exclusive_scan_i64(l_sums.as<int64_t>(), l_tiles, l_offs.as<int64_t>(), slot.dev(), s));
    tile_scan_kernel<uint32_t><<<(unsigned)l_tiles, kBlock, 0, s>>>(counts.as<uint32_t>(), nl, l_offs.as<int64_t>(), row_off.as<int64_t>(), outer);
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(slot.fetch(s));
    total = slot.host()[0];
  }
  if (total > 0xfffffff0ll * 16) return set_error(B2_CAPACITY_ERROR, "b2_hash_join: %lld result pairs; join the sides in chunks", (long long)total);
  // FULL OUTER: the build rows nobody matched follow the probe side's pairs
  PoolArray lonely(ctx, s);
  int64_t n_lonely = 0;
  if (full && nr > 0) {
    Temp matched(ctx, s), lmask(ctx, s);
    B2_RETURN_NOT_OK(matched.alloc(groups ? groups : 1));
    B2_CUDA(cudaMemsetAsync(matched.ptr, 0, groups ? groups : 1, s));
    if (nl > 0) {
      mark_matched_kernel<<<grid_for(nl, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(d_lids, lid_valid, lkey_valid, nl, matched.as<uint8_t>());
      B2_LAUNCHED();
    }
    B2_RETURN_NOT_OK(lmask.alloc(bitmap_alloc_bytes(nr)));
    B2_CUDA(cudaMemsetAsync(lmask.ptr, 0, bitmap_alloc_bytes(nr), s));
    unmatched_build_kernel<<<grid_for(nr, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(static_cast<const uint32_t*>(rids.a.data), BitmapReader(rvalid, 0, nr),
                                                                            matched.as<uint8_t>(), nr, lmask.as<uint32_t>());
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(mask_rows_u32(ctx, lmask.ptr, nr, &lonely, s));
    n_lonely = lonely.a.length;
  }
  const int64_t head = total;
  total += n_lonely;
  Temp ol(ctx, s), orr(ctx, s);
  B2_RETURN_NOT_OK(ol.alloc(sizeof(uint32_t) * (size_t)(total ? total : 1)));
  B2_RETURN_NOT_OK(orr.alloc(sizeof(uint32_t) * (size_t)(total ? total : 1)));
  if (head > 0) {
    emit_pairs_kernel<<<grid_for(nl, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(d_lids, counts.as<uint32_t>(), where32.as<uint32_t>(),
                                                                          build_rows.as<uint32_t>(), row_off.as<int64_t>(), nl,
                                                                          ol.as<uint32_t>(), orr.as<uint32_t>(), outer);
    B2_LAUNCHED();
  }
  if (outer) return finish_outer(ctx, &ol, &orr, lonely, head, total, full, out_left, out_right, s);
  fill_out(out_left, B2_UINT32, total, 0, nullptr, ol.release());
  fill_out(out_right, B2_UINT32, total, 0, nullptr, orr.release());
  return B2_OK;
}

extern "C" int b2_join_residual(B2Context* ctx, const B2Array* cand_left, const B2Array* cand_right, const B2Array* keep, int64_t n_left,
                                int64_t n_right, int join_type, B2Array* out_left, B2Array* out_right, void* stream) {
  if (!ctx || !cand_left || !cand_right || !keep || !out_left) return set_error(B2_INVALID, "b2_join_residual: null argument");
  if (join_type < B2_JOIN_INNER || join_type > B2_JOIN_FULL_OUTER) return set_error(B2_NOT_IMPLEMENTED, "b2_join_residual: join type %d", join_type);
  const bool full = join_type == B2_JOIN_FULL_OUTER;
  const bool outer = join_type == B2_JOIN_LEFT_OUTER || full;
  if ((outer || join_type == B2_JOIN_INNER) && !out_right) return set_error(B2_INVALID, "b2_join_residual: this join type returns right indices too");
  if (cand_left->type != B2_UINT32 || cand_right->type != B2_UINT32) return set_error(B2_TYPE_ERROR, "b2_join_residual: candidate rows must be uint32");
  if (keep->type != B2_BOOL) return set_error(B2_TYPE_ERROR, "b2_join_residual: keep must be boolean, got type id %d", keep->type);
  const int64_t m = cand_left->length;
  if (cand_right->length != m || keep->length != m)
    return set_error(B2_INVALID, "b2_join_residual: %lld left rows, %lld right rows and %lld keep flags per candidate pair", (long long)m,
                     (long long)cand_right->length, (long long)keep->length);
  if ((cand_left->validity && cand_left->null_count != 0) || (cand_right->validity && cand_right->null_count != 0))
    return set_error(B2_INVALID, "b2_join_residual: candidate rows must not be null");
  if (n_left < 0 || n_right < 0) return set_error(B2_INVALID, "b2_join_residual: negative side length");
  if (n_left > 0xfffffff0ll || n_right > 0xfffffff0ll) return set_error(B2_NOT_IMPLEMENTED, "b2_join_residual: sides of 2^32 rows or more must be split");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));

  // ---- survivors, their count per left row, FULL OUTER's matched right rows; the pairs are checked before any use ----
  Temp survivors(ctx, s), counts(ctx, s), matched(ctx, s);
  B2_RETURN_NOT_OK(survivors.alloc(bitmap_alloc_bytes(m)));
  B2_RETURN_NOT_OK(counts.alloc(sizeof(uint32_t) * (size_t)(n_left ? n_left : 1)));
  B2_CUDA(cudaMemsetAsync(counts.ptr, 0, sizeof(uint32_t) * (size_t)(n_left ? n_left : 1), s));
  if (full) {
    B2_RETURN_NOT_OK(matched.alloc(n_right ? n_right : 1));
    B2_CUDA(cudaMemsetAsync(matched.ptr, 0, n_right ? n_right : 1, s));
  }
  ScalarSlot stats(ctx);
  B2_RETURN_NOT_OK(stats.zero(s));
  if (m > 0) {
    const uint32_t* cl = static_cast<const uint32_t*>(cand_left->data) + cand_left->offset;
    const uint32_t* cr = static_cast<const uint32_t*>(cand_right->data) + cand_right->offset;
    residual_count_kernel<<<grid_for(m, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(
        cl, cr, BitmapReader(keep->data, keep->offset, m), BitmapReader(keep->null_count == 0 ? nullptr : keep->validity, keep->offset, m), m,
        n_left, n_right, survivors.as<uint32_t>(), counts.as<uint32_t>(), full ? matched.as<uint8_t>() : nullptr, stats.dev());
    B2_LAUNCHED();
  }
  B2_RETURN_NOT_OK(stats.fetch(s));
  const int64_t k = stats.host()[0];
  const int64_t bad = stats.host()[1];
  if (bad & kBadLeft) return set_error(B2_INVALID, "b2_join_residual: a candidate left row is not below n_left = %lld", (long long)n_left);
  if (bad & kBadRight) return set_error(B2_INVALID, "b2_join_residual: a candidate right row is not below n_right = %lld", (long long)n_right);
  if (bad & kBadOrder) return set_error(B2_INVALID, "b2_join_residual: candidate left rows must be non-decreasing");
  B2Array mask{};
  mask.type = B2_BOOL;
  mask.data = survivors.ptr;
  mask.length = m;

  if (join_type == B2_JOIN_INNER) {  // the surviving pairs, compacted
    if (k > 0xfffffff0ll * 16) return set_error(B2_CAPACITY_ERROR, "b2_join_residual: %lld result pairs; join the sides in chunks", (long long)k);
    PoolArray l(ctx, s), r(ctx, s);
    B2_RETURN_NOT_OK(b2_filter(ctx, cand_left, &mask, 0, &l.a, s));
    B2_RETURN_NOT_OK(b2_filter(ctx, cand_right, &mask, 0, &r.a, s));
    l.give(out_left);
    r.give(out_right);
    return B2_OK;
  }
  if (!outer) {  // SEMI / ANTI: the left rows with / without a survivor
    Temp lmask(ctx, s);
    B2_RETURN_NOT_OK(lmask.alloc(bitmap_alloc_bytes(n_left)));
    if (n_left > 0) {
      zero_mask_kernel<uint32_t><<<grid_for(n_left, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(counts.as<uint32_t>(), n_left,
                                                                                          join_type == B2_JOIN_LEFT_ANTI, lmask.as<uint32_t>());
      B2_LAUNCHED();
    }
    PoolArray rows(ctx, s);
    B2_RETURN_NOT_OK(mask_rows_u32(ctx, lmask.ptr, n_left, &rows, s));
    rows.give(out_left);
    return B2_OK;
  }

  // ---- LEFT / FULL OUTER: row_off = exclusive scan of max(count, 1), first = exclusive scan of the counts ----
  const int64_t l_tiles = (n_left + kScanTile - 1) / kScanTile;
  Temp sums(ctx, s), offs(ctx, s), row_off(ctx, s), first(ctx, s);
  B2_RETURN_NOT_OK(sums.alloc(sizeof(int64_t) * (size_t)(l_tiles ? l_tiles : 1)));
  B2_RETURN_NOT_OK(offs.alloc(sizeof(int64_t) * (size_t)(l_tiles ? l_tiles : 1)));
  B2_RETURN_NOT_OK(row_off.alloc(sizeof(int64_t) * (size_t)(n_left ? n_left : 1)));
  B2_RETURN_NOT_OK(first.alloc(sizeof(int64_t) * (size_t)(n_left ? n_left : 1)));
  int64_t head = 0;
  if (n_left > 0) {
    ScalarSlot tot(ctx);
    B2_RETURN_NOT_OK(tot.zero(s));
    for (const bool min_one : {true, false}) {
      tile_sums_kernel<uint32_t><<<(unsigned)l_tiles, kBlock, 0, s>>>(counts.as<uint32_t>(), n_left, min_one, sums.as<int64_t>());
      B2_LAUNCHED();
      B2_RETURN_NOT_OK(launch_exclusive_scan_i64(sums.as<int64_t>(), l_tiles, offs.as<int64_t>(), min_one ? tot.dev() : nullptr, s));
      tile_scan_kernel<uint32_t><<<(unsigned)l_tiles, kBlock, 0, s>>>(counts.as<uint32_t>(), n_left, offs.as<int64_t>(),
                                                                       (min_one ? row_off : first).as<int64_t>(), min_one);
      B2_LAUNCHED();
    }
    B2_RETURN_NOT_OK(tot.fetch(s));
    head = tot.host()[0];
  }
  if (head > 0xfffffff0ll * 16) return set_error(B2_CAPACITY_ERROR, "b2_join_residual: %lld result pairs; join the sides in chunks", (long long)head);
  PoolArray lonely(ctx, s);
  if (full && n_right > 0) {  // the right rows no surviving pair reached follow the left rows' pairs
    Temp rmask(ctx, s);
    B2_RETURN_NOT_OK(rmask.alloc(bitmap_alloc_bytes(n_right)));
    zero_mask_kernel<uint8_t><<<grid_for(n_right, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(matched.as<uint8_t>(), n_right, true, rmask.as<uint32_t>());
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(mask_rows_u32(ctx, rmask.ptr, n_right, &lonely, s));
  }
  const int64_t total = head + lonely.a.length;
  PoolArray kept_left(ctx, s), kept_right(ctx, s);
  if (k > 0) {
    B2_RETURN_NOT_OK(b2_filter(ctx, cand_left, &mask, 0, &kept_left.a, s));
    B2_RETURN_NOT_OK(b2_filter(ctx, cand_right, &mask, 0, &kept_right.a, s));
  }
  Temp ol(ctx, s), orr(ctx, s);
  B2_RETURN_NOT_OK(ol.alloc(sizeof(uint32_t) * (size_t)(total ? total : 1)));
  B2_RETURN_NOT_OK(orr.alloc(sizeof(uint32_t) * (size_t)(total ? total : 1)));
  if (head > 0) {
    residual_emit_kernel<<<grid_for(k + n_left, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(
        static_cast<const uint32_t*>(kept_left.a.data), static_cast<const uint32_t*>(kept_right.a.data), k, counts.as<uint32_t>(),
        first.as<int64_t>(), row_off.as<int64_t>(), n_left, ol.as<uint32_t>(), orr.as<uint32_t>());
    B2_LAUNCHED();
  }
  return finish_outer(ctx, &ol, &orr, lonely, head, total, full, out_left, out_right, s);
}
