// selection_binary.cu -- Filter and Take for (large_)utf8 / (large_)binary columns.
//
// Replaces:
//   BinaryFilterExec / BinaryFilterNonNullImpl / BinaryFilterImpl
//                                   kernels/vector_selection_filter_internal.cc:552-856
//   VarBinaryTakeExec -> VarBinarySelectionImpl::GenerateOutput
//                                   kernels/vector_selection_internal.cc:475-548,966
// Semantics kept: the output has fresh offsets starting at 0 (running sum of the kept
// lengths) and the concatenation of the kept bytes; null output slots have length 0;
// an int32-offset Take whose output would exceed 2^31-2 bytes fails like the reference
// (vector_selection_internal.cc:519-523); a Filter never does, since its output is at most its input.
//
// Design (per call): sizes pass -> tile scan -> copy pass.
//   sizes: one CTA per 4096-row tile; each warp walks 512 rows 32 at a time (coalesced
//          offset loads), sums the kept lengths -> bytes per tile.
//   scan : exclusive scan of the per-tile byte counts (single CTA, tiny).
//   copy : the same walk with a warp scan per step rebuilds per-row output offsets, stages
//          (output offset, source offset) of the tile's kept rows in shared memory and writes
//          the new offsets coalesced; then EVERY thread produces 16-byte chunks of the tile's
//          contiguous output range: a coarse index + short binary search finds the row a
//          chunk starts in, each overlapping row segment is fetched with aligned 8-byte loads
//          and funnel-shifted into place, and the chunk leaves with one aligned 16-byte
//          store -- writes are fully coalesced regardless of string length.
// Algorithmic bytes/row (offset width o, mean length L, selectivity s): o + L + bitmaps
// read, s*(o + L + 1/8) written (utf8 Filter o=8, L=16, s=0.5: 36.3 B/row, SURVEY 8d).
#include <type_traits>

#include "selection.cuh"

namespace b2 {

constexpr int kBinThreads = 256;
constexpr int kTakeTile = 2048;
constexpr int kTakeRowsPerThread = kTakeTile / kBinThreads;  // 8 consecutive indices

// exclusive block scan of one int64 per thread; total returned to all threads
__device__ __forceinline__ int64_t block_excl_scan(int64_t v, int64_t* total) {
  __shared__ int64_t s_w[kBinThreads / 32 + 1];
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  int64_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int64_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  __syncthreads();  // protect s_w reuse across calls
  if (lane == 31) s_w[warp] = incl;
  __syncthreads();
  int64_t woff = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kBinThreads / 32; ++w) {
    int64_t x = s_w[w];
    if (w < (int)warp) woff += x;
    tot += x;
  }
  *total = tot;
  return woff + incl - v;
}

// Copies the tile's output byte range [out_base, out_base + tile_bytes) from the staged
// rows: s_out[j] = output offset of kept row j relative to out_base (s_out[n_rows] =
// tile_bytes), s_src[j] = absolute source byte offset of row j.
template <typename SrcT>
__device__ __forceinline__ void copy_tile_bytes(const uint8_t* __restrict__ src, const uint8_t* data_base,
                                                uint8_t* __restrict__ dst, int64_t out_base, int64_t tile_bytes,
                                                const uint32_t* s_out, const SrcT* s_src, int n_rows) {
  if (tile_bytes == 0) return;
  uint8_t* d0 = dst + out_base;
  // split into an unaligned head, aligned 16-byte chunks and a tail
  int64_t head = static_cast<int64_t>((16 - (reinterpret_cast<uintptr_t>(d0) & 15)) & 15);
  if (head > tile_bytes) head = tile_bytes;
  const int64_t body_chunks = (tile_bytes - head) >> 4;
  const int64_t tail_start = head + (body_chunks << 4);
  // coarse index: s_coarse[k] = the row that covers output byte k << g (g >= 6 chosen so the
  // table has <= 512 entries), so a chunk's row is found by a binary search over the handful of
  // rows between two table entries instead of over the whole tile (12 dependent LDS steps)
  __shared__ uint16_t s_coarse[513];
  int g = 6;
  while ((tile_bytes >> g) >= 512) ++g;
  for (int j = threadIdx.x; j < n_rows; j += blockDim.x) {
    const uint32_t a = s_out[j], b = s_out[j + 1];
    for (uint32_t k = (a + (1u << g) - 1u) >> g; (static_cast<uint64_t>(k) << g) < b; ++k) s_coarse[k] = static_cast<uint16_t>(j);
  }
  __syncthreads();
  auto find_row = [&](uint32_t pos) {  // largest j with s_out[j] <= pos
    const uint32_t k = pos >> g;
    int lo = s_coarse[k];
    int hi = ((static_cast<int64_t>(k + 1) << g) < tile_bytes) ? s_coarse[k + 1] + 1 : n_rows;
    while (hi - lo > 1) {
      int mid = (lo + hi) >> 1;
      if (s_out[mid] <= pos) lo = mid;
      else hi = mid;
    }
    return lo;
  };
  // Word path: every row segment that overlaps the chunk is fetched with up to three aligned
  // 8-byte loads and funnel-shifted into place (a 16-byte string costs 2-3 LDG.64 instead of
  // 16 LDG.U8 -- the byte version was bound by L1 tag lookups).
  // Aligned words never start before an 8-byte-aligned data buffer; the word holding the last
  // byte may extend <= 7 bytes past the logical end, which stays inside the allocation
  // granule of any device allocation (Arrow buffers are padded to 8 bytes anyway).
  const bool word_ok = (reinterpret_cast<uintptr_t>(data_base) & 7) == 0;
  for (int64_t c = threadIdx.x; c < body_chunks; c += blockDim.x) {
    uint32_t pos = static_cast<uint32_t>(head + (c << 4));
    int j = find_row(pos);
    if (word_ok) {
      unsigned long long lo = 0, hi = 0;
      unsigned filled = 0;
      while (filled < 16) {
        // describe up to two row segments first (shared memory only), then issue the loads of
        // both, then merge: twice the loads in flight per thread on this latency-bound loop
        const unsigned long long* q[2];
        unsigned sh[2], len[2] = {0, 0}, at[2];
#pragma unroll
        for (int g = 0; g < 2; ++g) {
          if (filled < 16) {
            while (pos >= s_out[j + 1]) ++j;  // skips empty strings; sentinel s_out[n_rows] = tile_bytes > pos
            const unsigned avail = s_out[j + 1] - pos;
            len[g] = avail < 16u - filled ? avail : 16u - filled;
            const uint8_t* p = src + static_cast<int64_t>(s_src[j]) + (pos - s_out[j]);
            q[g] = reinterpret_cast<const unsigned long long*>(reinterpret_cast<uintptr_t>(p) & ~uintptr_t(7));
            sh[g] = static_cast<unsigned>(reinterpret_cast<uintptr_t>(p) & 7) * 8;
            at[g] = filled;
            filled += len[g];
            pos += len[g];
          }
        }
        unsigned long long w[2][3];
#pragma unroll
        for (int g = 0; g < 2; ++g) {
          w[g][0] = len[g] ? __ldg(q[g]) : 0ull;
          w[g][1] = (len[g] && sh[g] + len[g] * 8 > 64) ? __ldg(q[g] + 1) : 0ull;
          w[g][2] = (len[g] && sh[g] + len[g] * 8 > 128) ? __ldg(q[g] + 2) : 0ull;
        }
#pragma unroll
        for (int g = 0; g < 2; ++g) {
          if (!len[g]) continue;
          unsigned long long vlo = w[g][0], vhi = w[g][1];
          if (sh[g]) {
            vlo = (w[g][0] >> sh[g]) | (w[g][1] << (64 - sh[g]));
            vhi = (w[g][1] >> sh[g]) | (w[g][2] << (64 - sh[g]));
          }
          if (len[g] < 8) {
            vlo &= (1ull << (len[g] * 8)) - 1ull;
            vhi = 0;
          } else if (len[g] < 16) {
            vhi &= (1ull << ((len[g] - 8) * 8)) - 1ull;  // len == 8 -> 0
          }
          if (at[g] == 0) {
            lo = vlo;
            hi = vhi;
          } else if (at[g] < 8) {
            const unsigned s8 = at[g] * 8;
            lo |= vlo << s8;
            hi |= (vhi << s8) | (vlo >> (64 - s8));
          } else {
            hi |= vlo << ((at[g] - 8) * 8);  // at >= 8 -> len <= 8 -> vhi == 0
          }
        }
      }
      *reinterpret_cast<uint4*>(d0 + head + (c << 4)) =
          make_uint4(static_cast<uint32_t>(lo), static_cast<uint32_t>(lo >> 32), static_cast<uint32_t>(hi),
                     static_cast<uint32_t>(hi >> 32));
      continue;
    }
    uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
    for (int b = 0; b < 16; ++b) {
      while (pos >= s_out[j + 1]) ++j;
      uint32_t byte = src[static_cast<int64_t>(s_src[j]) + (pos - s_out[j])];
      w[b >> 2] |= byte << ((b & 3) * 8);
      ++pos;
    }
    *reinterpret_cast<uint4*>(d0 + head + (c << 4)) = make_uint4(w[0], w[1], w[2], w[3]);
  }
  // head + tail bytes (< 32 per tile)
  const int64_t edge = head + (tile_bytes - tail_start);
  for (int64_t e = threadIdx.x; e < edge; e += blockDim.x) {
    uint32_t pos = static_cast<uint32_t>(e < head ? e : tail_start + (e - head));
    int j = find_row(pos);
    while (pos >= s_out[j + 1]) ++j;
    d0[pos] = src[static_cast<int64_t>(s_src[j]) + (pos - s_out[j])];
  }
}

// ------------------------------------------------------------------------------------------
// Filter
// ------------------------------------------------------------------------------------------
template <typename OffT>
struct BinFilterArgs {
  FilterBitmaps fb;
  const OffT* offsets;  // advanced by values.offset
  const uint8_t* data;
  const int64_t* tile_rows;   // exclusive prefix of kept rows per tile  [n_tiles + 1]
  int64_t* tile_bytes;        // sizes pass: out ; copy pass: exclusive prefix [n_tiles]
  OffT* out_offsets;
  uint8_t* out_data;
  uint32_t* out_validity;  // zero-initialised or NULL
  int64_t n;
  int64_t* oversize;       // sizes pass, 64-bit offsets: set when a tile's source span does not fit the 32-bit staging
};

template <typename OffT, bool COPY, bool HAS_VALID>
__global__ void __launch_bounds__(kBinThreads, 1) filter_binary_kernel(BinFilterArgs<OffT> a) {
  __shared__ uint64_t s_sel[kTileWords];
  __shared__ uint64_t s_ov[kTileWords];
  __shared__ uint32_t s_prefix[kTileWords];
  __shared__ uint32_t s_out[COPY ? kTileRows + 1 : 1];
  __shared__ uint32_t s_src[COPY ? kTileRows : 1];
  __shared__ uint32_t s_bits[(COPY && HAS_VALID) ? kTileRows / 32 + 2 : 1];
  const int64_t tile = blockIdx.x;
  const int64_t row0 = tile * kTileRows;
  const unsigned lane = lane_id();
  if (threadIdx.x < 32) {
    int64_t w0 = tile * kTileWords + 2 * lane;
    uint64_t s0 = a.fb.sel(w0), s1 = a.fb.sel(w0 + 1);
    int c0 = __popcll(s0), c1 = __popcll(s1);
    int incl = c0 + c1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    int excl = incl - c0 - c1;
    s_sel[2 * lane] = s0;
    s_sel[2 * lane + 1] = s1;
    s_prefix[2 * lane] = excl;
    s_prefix[2 * lane + 1] = excl + c0;
    s_ov[2 * lane] = a.fb.out_valid(w0);
    s_ov[2 * lane + 1] = a.fb.out_valid(w0 + 1);
  }
  if (COPY && HAS_VALID)
    for (int i = threadIdx.x; i < kTileRows / 32 + 2; i += kBinThreads) s_bits[i] = 0;
  __syncthreads();

  // Every warp walks its 512 rows 32 at a time, so the offset loads are coalesced (a thread
  // owning 16 consecutive rows made every LDG touch 32 different lines: the L1 tag stage, not
  // HBM, bounded the kernel).  Per step: lengths of the kept rows, a warp scan for their
  // warp-relative output offsets, and -- in the copy pass -- (offset, source) staged at the
  // row's rank among the tile's kept rows.
  const unsigned warp = threadIdx.x >> 5;
  constexpr int kWarps = kBinThreads / 32;
  constexpr int kRowsPerWarp = kTileRows / kWarps;  // 512
  __shared__ int64_t s_wtot[kWarps];
  const int64_t out_row_base = COPY ? a.tile_rows[tile] : 0;
  const OffT tile_src0 = a.offsets[row0];
  int64_t wrun = 0;  // bytes of this warp's kept rows so far (uniform across the warp)
#pragma unroll 4
  for (int it = 0; it < kRowsPerWarp / 32; ++it) {
    const int r = warp * kRowsPerWarp + it * 32 + lane;
    const int64_t g = row0 + r;
    const uint64_t selw = s_sel[r >> 6];
    const bool sel = (selw >> (r & 63)) & 1;
    const bool ov = (s_ov[r >> 6] >> (r & 63)) & 1;
    OffT o0 = 0, o1 = 0;
    if (g < a.n) {
      o0 = a.offsets[g];
      o1 = a.offsets[g + 1];
    }
    const uint32_t len = (sel && ov) ? static_cast<uint32_t>(o1 - o0) : 0u;
    uint32_t incl = len;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (COPY && sel) {
      const unsigned j = s_prefix[r >> 6] + __popcll(selw & ((1ull << (r & 63)) - 1ull));
      s_out[j] = static_cast<uint32_t>(wrun) + incl - len;
      s_src[j] = static_cast<uint32_t>(o0 - tile_src0);
      if (HAS_VALID && ov) {
        const unsigned q = static_cast<unsigned>(out_row_base & 31) + j;
        atomicOr(&s_bits[q >> 5], 1u << (q & 31));
      }
    }
    wrun += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (lane == 0) s_wtot[warp] = wrun;
  __syncthreads();
  int64_t total = 0, wbase[kWarps];
#pragma unroll
  for (int w = 0; w < kWarps; ++w) {
    wbase[w] = total;
    total += s_wtot[w];
  }
  if (!COPY) {
    if (threadIdx.x == 0) {
      a.tile_bytes[tile] = total;
      // lengths, staged offsets and sources are 32-bit and tile-relative: with 64-bit offsets a tile whose SOURCE span reaches
      // 4 GiB (a single value that large, or 4096 huge ones) would wrap silently -- report it instead (ADVICE r1)
      if (sizeof(OffT) == 8 && a.oversize) {
        const int64_t end = row0 + kTileRows < a.n ? row0 + kTileRows : a.n;
        if (static_cast<int64_t>(a.offsets[end]) - static_cast<int64_t>(tile_src0) >= (1ll << 32)) *a.oversize = 1;
      }
    }
    return;
  }
  const int64_t byte_base = a.tile_bytes[tile];
  const int n_rows = static_cast<int>(a.tile_rows[tile + 1] - out_row_base);
  // second half: add the warp bases and write the new offsets, coalesced
  for (int j = threadIdx.x; j < n_rows; j += kBinThreads) {
    int64_t base = 0;
#pragma unroll
    for (int w = 1; w < kWarps; ++w)
      if (s_prefix[w * (kRowsPerWarp / 64)] <= static_cast<uint32_t>(j)) base = wbase[w];
    const uint32_t v = s_out[j] + static_cast<uint32_t>(base);
    s_out[j] = v;
    a.out_offsets[out_row_base + j] = static_cast<OffT>(byte_base + v);
  }
  if (threadIdx.x == 0) {
    s_out[n_rows] = static_cast<uint32_t>(total);
    if (tile == gridDim.x - 1) a.out_offsets[out_row_base + n_rows] = static_cast<OffT>(byte_base + total);
  }
  __syncthreads();
  copy_tile_bytes<uint32_t>(a.data + tile_src0, a.data, a.out_data, byte_base, total, s_out, s_src, n_rows);
  if (HAS_VALID) {
    const unsigned bit_base = static_cast<unsigned>(out_row_base & 31);
    const unsigned q_end = bit_base + n_rows;
    uint32_t* gw = a.out_validity + (out_row_base >> 5);
    for (unsigned i = threadIdx.x; i * 32 < q_end; i += kBinThreads) {
      uint32_t wv = s_bits[i];
      bool full = (i * 32 >= bit_base) && ((i + 1) * 32 <= q_end);
      if (full) gw[i] = wv;
      else if (wv) atomicOr(&gw[i], wv);
    }
  }
}

template <typename OffT>
static int filter_binary_typed(B2Context* ctx, const B2Array* values, const B2Array* mask, int null_selection,
                               B2Array* out, cudaStream_t s) {
  const int64_t n = values->length;
  const bool has_valid = (values->null_count != 0 && values->validity) || (mask->null_count != 0 && mask->validity);
  if (n == 0) {
    Temp offs(ctx, s);
    B2_RETURN_NOT_OK(offs.alloc(sizeof(OffT)));
    B2_CUDA(cudaMemsetAsync(offs.ptr, 0, sizeof(OffT), s));
    fill_out(out, values->type, 0, 0, nullptr, offs.release(), nullptr);
    return B2_OK;
  }
  FilterBitmaps fb = make_filter_bitmaps(values, mask, null_selection);
  Temp row_offsets(ctx, s);
  int64_t out_len = 0, out_valid = 0;
  B2_RETURN_NOT_OK(filter_plan(ctx, fb, n, has_valid, &row_offsets, &out_len, &out_valid, s));
  const int64_t n_tiles = tiles_for(n);
  Temp tile_bytes(ctx, s), byte_offsets(ctx, s);
  B2_RETURN_NOT_OK(tile_bytes.alloc(sizeof(int64_t) * n_tiles));
  B2_RETURN_NOT_OK(byte_offsets.alloc(sizeof(int64_t) * n_tiles));
  BinFilterArgs<OffT> a;
  a.fb = fb;
  a.offsets = static_cast<const OffT*>(values->data) + values->offset;
  a.data = static_cast<const uint8_t*>(values->data2);
  a.tile_rows = row_offsets.as<int64_t>();
  a.tile_bytes = tile_bytes.as<int64_t>();
  a.out_offsets = nullptr;
  a.out_data = nullptr;
  a.out_validity = nullptr;
  a.n = n;
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  a.oversize = slot.dev() + 3;
  filter_binary_kernel<OffT, false, false><<<(unsigned)n_tiles, kBinThreads, 0, s>>>(a);
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(launch_exclusive_scan_i64(tile_bytes.as<int64_t>(), n_tiles, byte_offsets.as<int64_t>(), slot.dev(), s));
  B2_RETURN_NOT_OK(slot.fetch(s));
  // no capacity check: the kept bytes are a subset of the input's, which its offsets already bound (the reference's
  // filter has none either, vector_selection_internal.cc:519-523 is Take only)
  const int64_t total_bytes = slot.host()[0];
  if (slot.host()[3] != 0)
    return set_error(B2_NOT_IMPLEMENTED, "filter: a 4096-row tile of this large_utf8 / large_binary array spans 4 GiB or more of value bytes");
  Temp offs(ctx, s), data(ctx, s), bits(ctx, s);
  B2_RETURN_NOT_OK(offs.alloc(sizeof(OffT) * (size_t)(out_len + 1)));
  B2_RETURN_NOT_OK(data.alloc((size_t)total_bytes + 16));
  if (has_valid) {
    B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(out_len)));
    B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bitmap_alloc_bytes(out_len), s));
  }
  if (out_len == 0) B2_CUDA(cudaMemsetAsync(offs.ptr, 0, sizeof(OffT), s));
  a.tile_bytes = byte_offsets.as<int64_t>();
  a.out_offsets = offs.as<OffT>();
  a.out_data = data.as<uint8_t>();
  a.out_validity = bits.as<uint32_t>();
  if (has_valid) filter_binary_kernel<OffT, true, true><<<(unsigned)n_tiles, kBinThreads, 0, s>>>(a);
  else filter_binary_kernel<OffT, true, false><<<(unsigned)n_tiles, kBinThreads, 0, s>>>(a);
  B2_LAUNCHED();
  int64_t null_count = has_valid ? out_len - out_valid : 0;
  fill_out(out, values->type, out_len, null_count, has_valid ? bits.release() : nullptr, offs.release(), data.release());
  return B2_OK;
}

int filter_binary(B2Context* ctx, const B2Array* values, const B2Array* mask, int null_selection, B2Array* out,
                  cudaStream_t s) {
  if (offset_width(values->type) == 8) return filter_binary_typed<int64_t>(ctx, values, mask, null_selection, out, s);
  return filter_binary_typed<int32_t>(ctx, values, mask, null_selection, out, s);
}

// ------------------------------------------------------------------------------------------
// Take
// ------------------------------------------------------------------------------------------
template <typename OffT>
struct BinTakeArgs {
  const OffT* offsets;  // advanced by values.offset
  const uint8_t* data;
  BitmapReader values_valid;
  int64_t values_length;
  const void* indices;  // advanced by indices.offset
  BitmapReader idx_valid;
  int64_t n;
  int64_t* tile_bytes;
  OffT* out_offsets;
  uint8_t* out_data;
  uint32_t* out_validity;
  int64_t* valid_count;
  unsigned long long* first_bad;
  int64_t* oversize;  // sizes pass, 64-bit offsets: a taken value or a tile's total does not fit the 32-bit staging
};

template <typename Idx>
__device__ __forceinline__ uint64_t index_value(const void* p, int64_t i) {
  Idx raw = static_cast<const Idx*>(p)[i];
  if (std::is_unsigned<Idx>::value) return static_cast<uint64_t>(raw);
  return static_cast<uint64_t>(static_cast<int64_t>(raw));
}

template <typename OffT, typename Idx, bool COPY>
__global__ void __launch_bounds__(kBinThreads) take_binary_kernel(BinTakeArgs<OffT> a) {
  __shared__ uint32_t s_out[COPY ? kTakeTile + 1 : 1];
  __shared__ int64_t s_src[COPY ? kTakeTile : 1];
  __shared__ uint32_t s_bits[COPY ? kTakeTile / 32 : 1];
  const int64_t tile = blockIdx.x;
  const int64_t row0 = tile * kTakeTile + threadIdx.x * kTakeRowsPerThread;
  if (COPY)
    for (int i = threadIdx.x; i < kTakeTile / 32; i += kBinThreads) s_bits[i] = 0;
  uint32_t len[kTakeRowsPerThread];
  int64_t src[kTakeRowsPerThread];
  unsigned vb = 0;
  int64_t local = 0;
#pragma unroll
  for (int k = 0; k < kTakeRowsPerThread; ++k) {
    len[k] = 0;
    src[k] = 0;
    const int64_t i = row0 + k;
    if (i < a.n && a.idx_valid.bit(i)) {
      const uint64_t j = index_value<Idx>(a.indices, i);
      if (j >= static_cast<uint64_t>(a.values_length)) {
        atomicMin(a.first_bad, static_cast<unsigned long long>(i));
      } else if (a.values_valid.bit(static_cast<int64_t>(j))) {
        const OffT o0 = a.offsets[j], o1 = a.offsets[j + 1];
        len[k] = static_cast<uint32_t>(o1 - o0);
        src[k] = static_cast<int64_t>(o0);
        vb |= 1u << k;
        local += static_cast<int64_t>(o1) - static_cast<int64_t>(o0);  // the true length: a wrapped one must not hide an oversize tile
      }
    }
  }
  int64_t total;
  const int64_t excl = block_excl_scan(local, &total);
  if (!COPY) {
    if (threadIdx.x == 0) {
      a.tile_bytes[tile] = total;
      if (sizeof(OffT) == 8 && a.oversize && total >= (1ll << 32)) *a.oversize = 1;  // covers a single value >= 4 GiB too
    }
    return;
  }
  const int64_t byte_base = a.tile_bytes[tile];
  const int64_t tile_left = a.n - tile * kTakeTile;
  const int tile_n = tile_left < kTakeTile ? static_cast<int>(tile_left) : kTakeTile;
  uint32_t run = static_cast<uint32_t>(excl);
#pragma unroll
  for (int k = 0; k < kTakeRowsPerThread; ++k) {
    const int lr = threadIdx.x * kTakeRowsPerThread + k;
    if (lr < tile_n) {
      s_out[lr] = run;
      s_src[lr] = src[k];
      a.out_offsets[row0 + k] = static_cast<OffT>(byte_base + run);
      run += len[k];
    }
  }
  if (a.out_validity && vb) atomicOr(&s_bits[(threadIdx.x * kTakeRowsPerThread) >> 5], vb << ((threadIdx.x * kTakeRowsPerThread) & 31));
  if (threadIdx.x == 0) {
    s_out[tile_n] = static_cast<uint32_t>(total);
    if (tile == gridDim.x - 1) a.out_offsets[a.n] = static_cast<OffT>(byte_base + total);
  }
  __syncthreads();
  copy_tile_bytes<int64_t>(a.data, a.data, a.out_data, byte_base, total, s_out, s_src, tile_n);
  if (a.out_validity) {
    int64_t cnt = 0;
    if (threadIdx.x < kTakeTile / 32 && (int)threadIdx.x * 32 < tile_n) {
      a.out_validity[tile * (kTakeTile / 32) + threadIdx.x] = s_bits[threadIdx.x];
      cnt = __popc(s_bits[threadIdx.x]);
    }
    int64_t sum = block_sum<kBinThreads>(cnt);
    if (threadIdx.x == 0 && sum) atomicAdd(reinterpret_cast<unsigned long long*>(a.valid_count), (unsigned long long)sum);
  }
}


template <typename OffT, typename Idx>
static int take_binary_typed(B2Context* ctx, const B2Array* values, const B2Array* indices, B2Array* out, cudaStream_t s) {
  const int64_t n = indices->length;
  const bool has_valid = (values->null_count != 0 && values->validity) || (indices->null_count != 0 && indices->validity);
  const int64_t n_tiles = (n + kTakeTile - 1) / kTakeTile;
  Temp tile_bytes(ctx, s), byte_offsets(ctx, s);
  B2_RETURN_NOT_OK(tile_bytes.alloc(sizeof(int64_t) * (n_tiles ? n_tiles : 1)));
  B2_RETURN_NOT_OK(byte_offsets.alloc(sizeof(int64_t) * (n_tiles ? n_tiles : 1)));
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  B2_CUDA(cudaMemsetAsync(slot.dev() + 2, 0xff, 8, s));
  BinTakeArgs<OffT> a;
  a.offsets = static_cast<const OffT*>(values->data) + values->offset;
  a.data = static_cast<const uint8_t*>(values->data2);
  a.values_valid = BitmapReader(values->null_count == 0 ? nullptr : values->validity, values->offset, values->length);
  a.values_length = values->length;
  a.indices = static_cast<const char*>(indices->data) + indices->offset * sizeof(Idx);
  a.idx_valid = BitmapReader(indices->null_count == 0 ? nullptr : indices->validity, indices->offset, n);
  a.n = n;
  a.tile_bytes = tile_bytes.as<int64_t>();
  a.out_offsets = nullptr;
  a.out_data = nullptr;
  a.out_validity = nullptr;
  a.valid_count = slot.dev() + 1;
  a.first_bad = reinterpret_cast<unsigned long long*>(slot.dev() + 2);
  a.oversize = slot.dev() + 3;
  if (n == 0) {
    Temp offs(ctx, s);
    B2_RETURN_NOT_OK(offs.alloc(sizeof(OffT)));
    B2_CUDA(cudaMemsetAsync(offs.ptr, 0, sizeof(OffT), s));
    fill_out(out, values->type, 0, 0, nullptr, offs.release(), nullptr);
    return B2_OK;
  }
  take_binary_kernel<OffT, Idx, false><<<(unsigned)n_tiles, kBinThreads, 0, s>>>(a);
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(launch_exclusive_scan_i64(tile_bytes.as<int64_t>(), n_tiles, byte_offsets.as<int64_t>(), slot.dev(), s));
  B2_RETURN_NOT_OK(slot.fetch(s));
  const uint64_t bad = static_cast<uint64_t>(slot.host()[2]);
  if (bad != ~0ull) return index_error(indices, bad, s);
  const int64_t total_bytes = slot.host()[0];
  if (sizeof(OffT) == 4 && total_bytes > 2147483646ll)
    return set_error(B2_INVALID, "Take operation overflowed binary array capacity");  // vector_selection_internal.cc:519-523
  if (slot.host()[3] != 0)
    return set_error(B2_NOT_IMPLEMENTED, "take: 2048 taken rows of this large_utf8 / large_binary array hold 4 GiB or more of value bytes");
  Temp offs(ctx, s), data(ctx, s), bits(ctx, s);
  B2_RETURN_NOT_OK(offs.alloc(sizeof(OffT) * (size_t)(n + 1)));
  B2_RETURN_NOT_OK(data.alloc((size_t)total_bytes + 16));
  if (has_valid) {
    B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(n) + kTakeTile / 8));
    B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bitmap_alloc_bytes(n) + kTakeTile / 8, s));
  }
  B2_CUDA(cudaMemsetAsync(slot.dev() + 1, 0, 8, s));
  a.tile_bytes = byte_offsets.as<int64_t>();
  a.out_offsets = offs.as<OffT>();
  a.out_data = data.as<uint8_t>();
  a.out_validity = has_valid ? bits.as<uint32_t>() : nullptr;
  // 40 % of the shared memory rounds up to the 100 KB carveout: three 26 KB tiles per SM, and the rest of the SM's
  // 256 KB stays L1 for the random reads of the taken rows.  By default the driver fits five tiles (48 registers allow
  // it) and leaves less L1: a 500M-row large_utf8 take of 0-32 B strings by random int64 indices took 94.4 ms that way
  // and 90.0 ms this way (H100 80GB HBM3, 700 W power limit).
  B2_CUDA(cudaFuncSetAttribute(take_binary_kernel<OffT, Idx, true>, cudaFuncAttributePreferredSharedMemoryCarveout, 40));
  take_binary_kernel<OffT, Idx, true><<<(unsigned)n_tiles, kBinThreads, 0, s>>>(a);
  B2_LAUNCHED();
  int64_t null_count = 0;
  if (has_valid) {
    B2_RETURN_NOT_OK(slot.fetch(s));
    null_count = n - slot.host()[1];
  }
  fill_out(out, values->type, n, null_count, (has_valid && null_count) ? bits.release() : nullptr, offs.release(),
           data.release());
  return B2_OK;
}

template <typename OffT>
static int take_binary_off(B2Context* ctx, const B2Array* values, const B2Array* indices, B2Array* out, cudaStream_t s) {
  return visit_type(IndexTypes{}, indices->type,
                    [&](auto it) { return take_binary_typed<OffT, decltype(it)>(ctx, values, indices, out, s); },
                    [&] { return index_type_error(indices->type); });
}

int take_binary(B2Context* ctx, const B2Array* values, const B2Array* indices, int boundscheck, B2Array* out,
                cudaStream_t s) {
  (void)boundscheck;
  if (offset_width(values->type) == 8) return take_binary_off<int64_t>(ctx, values, indices, out, s);
  return take_binary_off<int32_t>(ctx, values, indices, out, s);
}

}  // namespace b2
