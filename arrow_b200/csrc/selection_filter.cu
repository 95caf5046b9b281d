// selection_filter.cu -- Filter for fixed-width (and dictionary-index) columns, the
// filter-output-size pre-pass, and mask -> take-indices.
//
// Replaces:
//   GetFilterOutputSize / GetBitmapFilterOutputSize   kernels/vector_selection_filter_internal.cc:62-114
//   PrimitiveFilterExec + PrimitiveFilterImpl<W>      :158-510
//   DictionaryFilterExec (filters the index column)   :871-881
//   GetTakeIndices (bitmap filter -> uint16/uint32 indices)
//                                                     kernels/vector_selection_take_internal.cc:62-305
// Semantics kept (FilterOptions, compute/api_vector.h:37-51): DROP keeps rows whose mask
// slot is valid and true; EMIT_NULL additionally keeps rows whose mask slot is null and
// emits a null there; output validity = values validity AND mask validity compacted
// alongside; the output carries a validity bitmap iff values or mask may have nulls.
//
// Design (two launches, HBM streaming):
//   1. filter_count_scan_kernel : one warp per 4096-row tile popcounts the selection words
//      (mask data &/| mask validity), publishes the count and resolves its exclusive prefix
//      with a chained scan (decoupled look-back over atomic-ticket ordered tiles); also emits
//      the survivors-before-chunk table (uint16 per 512 rows).      reads bitmaps only
//   2. filter_compact_kernel<W> : one WARP per 512-row chunk, no shared memory, no barrier.
//      Dense chunks issue all their 16-byte coalesced value loads first (they need every
//      sector anyway) so the loads overlap the bitmap round trip; lanes 0..15 rebuild the
//      chunk's 32-bit selection words and prefix popcounts in registers and every lane
//      stores its survivors at base + prefix + popc(lower bits): ranks are dense and
//      monotonic across a warp, so each store instruction writes one contiguous span.
//      Sparse chunks load only lanes holding a survivor.  Validity bits are compacted with
//      a software PEXT and OR-ed into the zeroed output bitmap (2 RED per 32 rows).
// Algorithmic bytes/row (int64, values nullable, mask non-null, s=0.5): 12.3125
// (SURVEY section 8d); pass 1 re-reads only the bitmaps (+0.25 B/row).
#include "selection.cuh"

namespace b2 {

// ---- passes 1+2 fused: per-tile counts with a chained scan (decoupled look-back) ----
// One warp owns a SPAN of kSpanTiles consecutive tiles; a CTA claims 8 consecutive spans with one
// atomic ticket, so the owners of all earlier spans are running or done (no residency
// assumption) and the single ticket address sees n_tiles/32 atomics, not n_tiles.  A span
// publishes its survivor count, then looks back over up to 32 predecessor cells per step (one
// per lane) until it meets one that already carries an inclusive prefix.
// cell = flag(2 bits) << 62 | value.
constexpr unsigned long long kCellAgg = 1ull << 62, kCellIncl = 2ull << 62, kCellMask = (1ull << 62) - 1ull;
constexpr int kSpanTiles = 4;

__global__ void __launch_bounds__(kBlock) filter_count_scan_kernel(FilterBitmaps fb, int64_t n_tiles,
                                                                   unsigned long long* cells, int64_t* offsets,
                                                                   uint16_t* chunk_rel, int64_t* totals, bool want_valid) {
  __shared__ unsigned long long s_ticket;
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  const int64_t n_spans = (n_tiles + kSpanTiles - 1) / kSpanTiles;
  int64_t valid_local = 0;
  volatile unsigned long long* vc = cells;
  unsigned long long* ticket = cells + n_spans;  // zero-initialised with the cells
  while (true) {
    __syncthreads();  // previous round's readers of s_ticket are done
    if (threadIdx.x == 0) s_ticket = atomicAdd(ticket, 1ull);
    __syncthreads();
    const int64_t span = static_cast<int64_t>(s_ticket) * kWarpsPerBlock + warp;
    if (static_cast<int64_t>(s_ticket) * kWarpsPerBlock >= n_spans) break;  // uniform across the CTA
    if (span >= n_spans) continue;
    const int64_t tile0 = span * kSpanTiles;
    int c[kSpanTiles];
    uint64_t w[kSpanTiles][2];
#pragma unroll
    for (int k = 0; k < kSpanTiles; ++k) {
      const int64_t w0 = (tile0 + k) * kTileWords + 2 * lane;
      const bool in = tile0 + k < n_tiles;
      w[k][0] = in ? fb.sel(w0) : 0ull;
      w[k][1] = in ? fb.sel(w0 + 1) : 0ull;
      c[k] = __popcll(w[k][0]) + __popcll(w[k][1]);
    }
    if (want_valid) {
#pragma unroll
      for (int k = 0; k < kSpanTiles; ++k) {
        if (tile0 + k >= n_tiles) break;
        const int64_t w0 = (tile0 + k) * kTileWords + 2 * lane;
        valid_local += __popcll(w[k][0] & fb.out_valid(w0)) + __popcll(w[k][1] & fb.out_valid(w0 + 1));
      }
    }
    unsigned tile_count[kSpanTiles];
    unsigned long long count = 0;
#pragma unroll
    for (int k = 0; k < kSpanTiles; ++k) {
      tile_count[k] = __reduce_add_sync(0xffffffffu, static_cast<unsigned>(c[k]));
      count += tile_count[k];
    }
    if (lane == 0) vc[span] = (span == 0 ? kCellIncl : kCellAgg) | count;
    if (chunk_rel) {
      // survivors before each 512-row chunk of a tile (lane 4j owns the first word of chunk j)
#pragma unroll
      for (int k = 0; k < kSpanTiles; ++k) {
        int incl = c[k];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          int v = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += v;
        }
        if ((lane & 3) == 0 && tile0 + k < n_tiles)
          chunk_rel[(tile0 + k) * 8 + (lane >> 2)] = static_cast<uint16_t>(incl - c[k]);
      }
    }
    unsigned long long excl = 0;
    if (span > 0) {
      int64_t back = span - 1;  // newest cell not yet folded in
      while (true) {
        const int64_t t = back - lane;
        unsigned long long cell = 0;
        if (t >= 0) {
          do {
            cell = vc[t];
          } while ((cell >> 62) == 0);
        }
        const unsigned incl_mask = __ballot_sync(0xffffffffu, t >= 0 && (cell >> 62) == 2);
        // lanes up to (and including) the first inclusive cell contribute
        const int first = incl_mask ? __ffs(incl_mask) - 1 : 31;
        unsigned long long part = (t >= 0 && (int)lane <= first) ? (cell & kCellMask) : 0ull;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
        excl += part;
        if (incl_mask || back - 32 < 0) break;
        back -= 32;
      }
      if (lane == 0) vc[span] = kCellIncl | (excl + count);
    }
    if (lane == 0) {
      unsigned long long run = excl;
#pragma unroll
      for (int k = 0; k < kSpanTiles; ++k) {
        if (tile0 + k < n_tiles) offsets[tile0 + k] = static_cast<int64_t>(run);
        run += tile_count[k];
      }
      if (span == n_spans - 1) {
        offsets[n_tiles] = static_cast<int64_t>(excl + count);
        totals[0] = static_cast<int64_t>(excl + count);
      }
    }
  }
  if (want_valid) {
    int64_t s = block_sum<kBlock>(valid_local);
    if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(totals + 1), (unsigned long long)s);
  }
}

// ---- pass 3: compaction ----
template <int W>
struct RowBytes;
template <> struct RowBytes<1> { using type = uint8_t; };
template <> struct RowBytes<2> { using type = uint16_t; };
template <> struct RowBytes<4> { using type = uint32_t; };
template <> struct RowBytes<8> { using type = uint64_t; };
template <> struct RowBytes<16> { using type = uint4; };

template <typename T>
__device__ __forceinline__ T iota_value(int64_t x) {
  return static_cast<T>(x);
}
template <>
__device__ __forceinline__ uint4 iota_value<uint4>(int64_t x) {
  return make_uint4(static_cast<unsigned>(x), static_cast<unsigned>(x >> 32), 0u, 0u);
}

struct FilterArgs {
  FilterBitmaps fb;
  const void* values;  // already advanced by offset * W
  void* out;
  uint32_t* out_validity;  // zero-initialised, or NULL
  const int64_t* tile_offsets;
  const uint16_t* chunk_rel;  // survivors before each 512-row chunk, relative to its tile
  int64_t n;
  bool vec_ok;
};

// 32-bit software PEXT (Hacker's Delight 7-4): bits of x selected by m, packed to the right
__device__ __forceinline__ uint32_t pext32(uint32_t x, uint32_t m) {
  x &= m;
  uint32_t mk = ~m << 1;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    uint32_t mp = mk ^ (mk << 1);
    mp ^= mp << 2;
    mp ^= mp << 4;
    mp ^= mp << 8;
    mp ^= mp << 16;
    const uint32_t mv = mp & m;
    m = (m ^ mv) | (mv >> (1 << i));
    const uint32_t t = x & mv;
    x = (x ^ t) | (t >> (1 << i));
    mk &= ~mp;
  }
  return x;
}

constexpr int kChunkRows = 512;  // rows per warp: 16 selection words of 32 bits

// One WARP compacts one 512-row chunk (a CTA = 8 chunks = one 4096-row tile), fully
// autonomously: no shared memory, no barrier.
//   * lanes 0..15 each build one 32-bit selection word of the chunk (+ its output-validity
//     word) and an exclusive prefix popcount over the 16 words (one warp scan);
//   * per pass a lane fetches the word and prefix covering its R rows with two 32-bit
//     shuffles, ranks its survivors with a popcount and stores them -- ranks are dense and
//     ascending across the warp, so each store instruction writes one contiguous span;
//   * validity: the same 16 lanes compress their 32 validity bits with a software PEXT and
//     OR them into the (zeroed) output bitmap -- 2 RED.OR per 32 rows, off the data path.
// Dense chunks (>= 1/8 survivors) issue all 16-byte value loads before anything else.
// IOTA: the "value" of row r is r itself (GetTakeIndices); W = index width
// SPARSE: same code compiled for 5 CTAs/SM (48 registers); latency-bound low-selectivity calls gain
// 11 % from the extra warps, dense ones lose 5 % to the spills, so the host picks by out_length / n.
template <int W, bool HAS_VALID, bool IOTA, bool SPARSE>
__global__ void __launch_bounds__(kBlock, (W <= 8 ? (SPARSE ? 5 : 4) : 1)) filter_compact_kernel(FilterArgs a) {
  using T = typename RowBytes<W>::type;
  constexpr int R = 16 / W;                    // rows per lane per 16-byte load
  constexpr int kPasses = kChunkRows / (32 * R);  // W=8: 8, W=4: 4, W=1: 1, W=16: 16
  const unsigned lane = lane_id();
  const int64_t tile = blockIdx.x;
  const int64_t chunk = tile * (kTileRows / kChunkRows) + (threadIdx.x >> 5);
  const int64_t row0 = chunk * kChunkRows;
  if (row0 >= a.n) return;
  const int64_t tile_base = a.tile_offsets[tile];
  const unsigned rel = a.chunk_rel[chunk];
  const unsigned next_rel = ((threadIdx.x >> 5) == kTileRows / kChunkRows - 1)
                                ? static_cast<unsigned>(a.tile_offsets[tile + 1] - tile_base)
                                : a.chunk_rel[chunk + 1];
  const unsigned chunk_count = next_rel - rel;
  if (chunk_count == 0) return;
  const int64_t out_base = tile_base + rel;
  const T* vals = static_cast<const T*>(a.values);

  const bool dense = !IOTA && a.vec_ok && chunk_count >= kChunkRows / 8 && row0 + kChunkRows <= a.n;
  uint4 raw[kPasses];
  if (dense) {
#pragma unroll
    for (int p = 0; p < kPasses; ++p) raw[p] = __ldcs(reinterpret_cast<const uint4*>(vals + row0 + p * 32 * R + lane * R));
  }

  // selection / validity words of this chunk (lanes 0..15) and their exclusive prefix
  uint32_t sel = 0, ov = 0;
  if (lane < 16) {
    const int64_t w64 = (row0 >> 6) + (lane >> 1);
    const uint64_t s64 = a.fb.sel(w64);
    sel = static_cast<uint32_t>((lane & 1) ? (s64 >> 32) : s64);
    if (HAS_VALID) {
      const uint64_t o64 = a.fb.out_valid(w64);
      ov = static_cast<uint32_t>((lane & 1) ? (o64 >> 32) : o64);
    }
  }
  const int c = __popc(sel);
  int incl = c;
#pragma unroll
  for (int o = 1; o < 16; o <<= 1) {
    int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  const unsigned pre = incl - c;

  if (HAS_VALID && c) {
    const uint32_t bits = pext32(ov, sel);
    const uint64_t q = static_cast<uint64_t>(out_base) + pre;  // absolute output bit position
    uint32_t* w = a.out_validity + (q >> 5);
    const unsigned sh = static_cast<unsigned>(q & 31);
    if (bits << sh) atomicOr(w, bits << sh);
    if (sh + c > 32 && (bits >> (32 - sh))) atomicOr(w + 1, bits >> (32 - sh));
  }

  T* out = static_cast<T*>(a.out) + out_base;
#pragma unroll
  for (int p = 0; p < kPasses; ++p) {
    const int r = p * 32 * R + lane * R;  // row within chunk
    const uint32_t wsel = __shfl_sync(0xffffffffu, sel, r >> 5);
    const unsigned wpre = __shfl_sync(0xffffffffu, pre, r >> 5);
    const unsigned sh = r & 31;
    const unsigned bits = (wsel >> sh) & ((1u << R) - 1u);
    if (bits == 0) continue;
    const unsigned rank = wpre + __popc(wsel & ((1u << sh) - 1u));
    const int64_t grow = row0 + r;
    T v[R];
    if (IOTA) {
#pragma unroll
      for (int k = 0; k < R; ++k) v[k] = iota_value<T>(grow + k);
    } else if (dense) {
      memcpy(v, &raw[p], 16);
    } else if (a.vec_ok && grow + R <= a.n) {
      uint4 x = __ldcs(reinterpret_cast<const uint4*>(vals + grow));
      memcpy(v, &x, 16);
    } else {
#pragma unroll
      for (int k = 0; k < R; ++k)
        if ((bits >> k) & 1) v[k] = vals[grow + k];
    }
    unsigned j = 0;
#pragma unroll
    for (int k = 0; k < R; ++k) {
      if ((bits >> k) & 1) {
        out[rank + j] = v[k];
        ++j;
      }
    }
  }
}

// passes 1+2 (one kernel): device tile offsets (caller frees), output length, selected-valid count
int filter_plan(B2Context* ctx, const FilterBitmaps& fb, int64_t n, bool want_valid,
                Temp* offsets, int64_t* out_length, int64_t* out_valid, cudaStream_t s, Temp* chunk_rel) {
  int64_t n_tiles = tiles_for(n);
  Temp cells(ctx, s);
  B2_RETURN_NOT_OK(cells.alloc((n_tiles + 1) * sizeof(unsigned long long)));  // + the ticket
  B2_RETURN_NOT_OK(offsets->alloc((n_tiles + 1) * sizeof(int64_t)));
  B2_CUDA(cudaMemsetAsync(cells.ptr, 0, (n_tiles + 1) * sizeof(unsigned long long), s));
  if (chunk_rel) B2_RETURN_NOT_OK(chunk_rel->alloc(n_tiles * 8 * sizeof(uint16_t)));
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  int grid = grid_for(n_tiles, kWarpsPerBlock * kSpanTiles, ctx->sm_count * 8);
  filter_count_scan_kernel<<<grid, kBlock, 0, s>>>(fb, n_tiles, cells.as<unsigned long long>(),
                                                   offsets->as<int64_t>(), chunk_rel ? chunk_rel->as<uint16_t>() : nullptr,
                                                   slot.dev(), want_valid);
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(slot.fetch(s));
  *out_length = slot.host()[0];
  *out_valid = slot.host()[1];
  return B2_OK;
}

static int check_mask(const B2Array* mask) {
  if (!mask) return set_error(B2_INVALID, "filter: null mask");
  if (mask->type != B2_BOOL) return set_error(B2_TYPE_ERROR, "filter mask must be a boolean array");
  if (mask->length < 0 || mask->offset < 0) return set_error(B2_INVALID, "negative length/offset");
  return B2_OK;
}

FilterBitmaps make_filter_bitmaps(const B2Array* values, const B2Array* mask, int null_selection) {
  FilterBitmaps fb;
  fb.mask_data = BitmapReader(mask->data, mask->offset, mask->length);
  fb.mask_valid = BitmapReader(mask->null_count == 0 ? nullptr : mask->validity, mask->offset, mask->length);
  fb.values_valid = values ? BitmapReader(values->null_count == 0 ? nullptr : values->validity,
                                          values->offset, values->length)
                           : BitmapReader(nullptr, 0, mask->length);
  fb.emit_null = null_selection == 1;
  return fb;
}

template <bool IOTA>
static int launch_compact(int width, bool has_valid, bool sparse, const FilterArgs& a, int64_t n_tiles,
                          cudaStream_t s) {
  dim3 grid(static_cast<unsigned>(n_tiles));
  B2_RETURN_NOT_OK((visit_width<1, 2, 4, 8, 16>(
      width,
      [&](auto w) {
        if (sparse) {
          if (has_valid) filter_compact_kernel<w, true, IOTA, true><<<grid, kBlock, 0, s>>>(a);
          else filter_compact_kernel<w, false, IOTA, true><<<grid, kBlock, 0, s>>>(a);
        } else {
          if (has_valid) filter_compact_kernel<w, true, IOTA, false><<<grid, kBlock, 0, s>>>(a);
          else filter_compact_kernel<w, false, IOTA, false><<<grid, kBlock, 0, s>>>(a);
        }
        return B2_OK;
      },
      [&] { return set_error(B2_NOT_IMPLEMENTED, "filter: unsupported byte width %d", width); })));
  B2_LAUNCHED();
  return B2_OK;
}

int filter_binary(B2Context* ctx, const B2Array* values, const B2Array* mask, int null_selection,
                  B2Array* out, cudaStream_t s);  // selection_binary.cu
int filter_bool(B2Context* ctx, const B2Array* values, const B2Array* mask, int null_selection, B2Array* out,
                cudaStream_t s);  // selection_bool.cu

}  // namespace b2

using namespace b2;

extern "C" int b2_filter_output_size(B2Context* ctx, const B2Array* mask, int null_selection,
                                     int64_t* out_length, void* stream) {
  if (!ctx || !out_length) return set_error(B2_INVALID, "b2_filter_output_size: null argument");
  B2_RETURN_NOT_OK(check_mask(mask));
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  *out_length = 0;
  if (mask->length == 0) return B2_OK;
  FilterBitmaps fb = make_filter_bitmaps(nullptr, mask, null_selection);
  Temp offsets(ctx, s);
  int64_t valid;
  return filter_plan(ctx, fb, mask->length, false, &offsets, out_length, &valid, s);
}

extern "C" int b2_filter(B2Context* ctx, const B2Array* values, const B2Array* mask,
                         int null_selection, B2Array* out, void* stream) {
  if (!ctx || !values || !out) return set_error(B2_INVALID, "b2_filter: null argument");
  B2_RETURN_NOT_OK(check_mask(mask));
  if (values->length != mask->length)
    return set_error(B2_INVALID, "Filter inputs must all be the same length");
  if (null_selection != 0 && null_selection != 1) return set_error(B2_INVALID, "bad null_selection");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  if (type_is_binary_like(values->type)) return filter_binary(ctx, values, mask, null_selection, out, s);
  if (values->type == B2_BOOL) return filter_bool(ctx, values, mask, null_selection, out, s);
  int width = values->type == B2_FIXED_SIZE_BINARY ? values->byte_width : type_width(values->type);
  if (width != 1 && width != 2 && width != 4 && width != 8 && width != 16)
    return set_error(B2_NOT_IMPLEMENTED, "filter: unsupported value type id %d (width %d)", values->type, width);
  const int64_t n = values->length;
  const bool has_valid = (values->null_count != 0 && values->validity) ||
                         (mask->null_count != 0 && mask->validity);
  if (n == 0) {
    fill_out(out, values->type, 0, 0, nullptr, nullptr);
    out->byte_width = values->byte_width;
    return B2_OK;
  }
  FilterBitmaps fb = make_filter_bitmaps(values, mask, null_selection);
  Temp offsets(ctx, s);
  int64_t out_len = 0, out_valid = 0;
  Temp chunk_rel(ctx, s);
  B2_RETURN_NOT_OK(filter_plan(ctx, fb, n, has_valid, &offsets, &out_len, &out_valid, s, &chunk_rel));

  Temp data(ctx, s), bits(ctx, s);
  B2_RETURN_NOT_OK(data.alloc(static_cast<size_t>(out_len) * width));
  if (has_valid) {
    B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(out_len)));
    B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bitmap_alloc_bytes(out_len), s));
  }
  if (out_len > 0) {
    FilterArgs a;
    a.fb = fb;
    a.values = static_cast<const char*>(values->data) + values->offset * width;
    a.out = data.ptr;
    a.out_validity = bits.as<uint32_t>();
    a.tile_offsets = offsets.as<int64_t>();
    a.chunk_rel = chunk_rel.as<uint16_t>();
    a.n = n;
    a.vec_ok = aligned_to(a.values, 16);
    B2_RETURN_NOT_OK(launch_compact<false>(width, has_valid, out_len < n / 8, a, tiles_for(n), s));
  }
  int64_t null_count = has_valid ? out_len - out_valid : 0;
  fill_out(out, values->type, out_len, null_count, has_valid ? bits.release() : nullptr, data.release());
  out->byte_width = values->byte_width;
  return B2_OK;
}

extern "C" int b2_filter_indices(B2Context* ctx, const B2Array* mask, int null_selection,
                                 B2Array* out, void* stream) {
  if (!ctx || !out) return set_error(B2_INVALID, "b2_filter_indices: null argument");
  B2_RETURN_NOT_OK(check_mask(mask));
  // vector_selection_take_internal.cc:262-271
  if (mask->length > 0xffffffffll)
    return set_error(B2_NOT_IMPLEMENTED, "Filter length exceeds UINT32_MAX, consider a different strategy for selecting elements");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = mask->length;
  const int out_type = n <= 0xffff ? B2_UINT16 : B2_UINT32;  // :298-305
  const int width = n <= 0xffff ? 2 : 4;
  if (n == 0) {
    fill_out(out, out_type, 0, 0, nullptr, nullptr);
    return B2_OK;
  }
  const bool has_valid = null_selection == 1 && mask->null_count != 0 && mask->validity;
  FilterBitmaps fb = make_filter_bitmaps(nullptr, mask, null_selection);
  Temp offsets(ctx, s);
  int64_t out_len = 0, out_valid = 0;
  Temp chunk_rel(ctx, s);
  B2_RETURN_NOT_OK(filter_plan(ctx, fb, n, has_valid, &offsets, &out_len, &out_valid, s, &chunk_rel));
  Temp data(ctx, s), bits(ctx, s);
  B2_RETURN_NOT_OK(data.alloc(static_cast<size_t>(out_len) * width));
  if (has_valid) {
    B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(out_len)));
    B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bitmap_alloc_bytes(out_len), s));
  }
  if (out_len > 0) {
    FilterArgs a;
    a.fb = fb;
    a.values = nullptr;
    a.out = data.ptr;
    a.out_validity = bits.as<uint32_t>();
    a.tile_offsets = offsets.as<int64_t>();
    a.chunk_rel = chunk_rel.as<uint16_t>();
    a.n = n;
    a.vec_ok = false;
    B2_RETURN_NOT_OK(launch_compact<true>(width, has_valid, out_len < n / 8, a, tiles_for(n), s));
  }
  int64_t null_count = has_valid ? out_len - out_valid : 0;
  fill_out(out, out_type, out_len, null_count, (has_valid && null_count) ? bits.release() : nullptr,
           data.release());
  return B2_OK;
}
