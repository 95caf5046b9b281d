// selection_bool.cu -- Filter and Take for boolean (bit-packed) value columns.
//
// Replaces PrimitiveFilterImpl<1, /*kIsBoolean=*/true>
// (cpp/src/arrow/compute/kernels/vector_selection_filter_internal.cc:158-441,478-480) and the
// boolean case of FixedWidthTakeExec / Gather<1-bit> (vector_selection_take_internal.cc:405-468,
// gather_internal.h:172-251).  Values and validity are both bitmaps, so Filter is two bit
// compressions per 64-row word (software PEXT) staged in a shared-memory bitmap per tile and
// flushed with whole-word stores; Take gathers one bit per row and packs 32 rows per warp ballot.
#include <type_traits>

#include "selection.cuh"

namespace b2 {

// parallel-suffix bit compress (Hacker's Delight 7-4): bits of x selected by m, packed to the right
__device__ __forceinline__ uint64_t pext64(uint64_t x, uint64_t m) {
  x &= m;
  uint64_t mk = ~m << 1;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    uint64_t mp = mk ^ (mk << 1);
    mp ^= mp << 2;
    mp ^= mp << 4;
    mp ^= mp << 8;
    mp ^= mp << 16;
    mp ^= mp << 32;
    const uint64_t mv = mp & m;
    m = (m ^ mv) | (mv >> (1 << i));
    const uint64_t t = x & mv;
    x = (x ^ t) | (t >> (1 << i));
    mk &= ~mp;
  }
  return x;
}

struct BoolFilterArgs {
  FilterBitmaps fb;
  BitmapReader data;  // the boolean values
  const int64_t* tile_offsets;
  unsigned long long* out_data;      // zero-initialised, 64-bit words
  unsigned long long* out_validity;  // zero-initialised or NULL
};

__device__ __forceinline__ void or_bits(unsigned long long* words, unsigned q, uint64_t bits, int count) {
  if (!bits) return;
  atomicOr(&words[q >> 6], (unsigned long long)(bits << (q & 63)));
  if ((q & 63) + count > 64) atomicOr(&words[(q >> 6) + 1], (unsigned long long)(bits >> (64 - (q & 63))));
}

__global__ void __launch_bounds__(64) filter_bool_kernel(BoolFilterArgs a) {
  __shared__ unsigned long long s_data[kTileRows / 64 + 2];
  __shared__ unsigned long long s_valid[kTileRows / 64 + 2];
  __shared__ int s_warp_total;
  const int64_t tile = blockIdx.x;
  const int t = threadIdx.x;  // one selection word per thread
  for (int i = t; i < kTileRows / 64 + 2; i += 64) {
    s_data[i] = 0;
    s_valid[i] = 0;
  }
  const int64_t w = tile * kTileWords + t;
  const uint64_t sel = a.fb.sel(w);
  const int c = __popcll(sel);
  // exclusive prefix of c over the 64 threads (2 warps)
  int incl = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int v = __shfl_up_sync(0xffffffffu, incl, o);
    if ((t & 31) >= o) incl += v;
  }
  if (t == 31) s_warp_total = incl;
  __syncthreads();
  const int excl = incl - c + (t >= 32 ? s_warp_total : 0);
  const int64_t out_base = a.tile_offsets[tile];
  const unsigned bit_base = static_cast<unsigned>(out_base & 63);
  if (c) {
    or_bits(s_data, bit_base + excl, pext64(a.data.word(w), sel), c);
    if (a.out_validity) or_bits(s_valid, bit_base + excl, pext64(a.fb.out_valid(w), sel), c);
  }
  __syncthreads();
  const unsigned count = static_cast<unsigned>(a.tile_offsets[tile + 1] - out_base);
  const unsigned q_end = bit_base + count;
  for (unsigned i = t; i * 64 < q_end; i += 64) {
    const bool full = (i * 64 >= bit_base) && ((i + 1) * 64 <= q_end);
    unsigned long long* gd = a.out_data + (out_base >> 6) + i;
    if (full) *gd = s_data[i];
    else if (s_data[i]) atomicOr(gd, s_data[i]);
    if (a.out_validity) {
      unsigned long long* gv = a.out_validity + (out_base >> 6) + i;
      if (full) *gv = s_valid[i];
      else if (s_valid[i]) atomicOr(gv, s_valid[i]);
    }
  }
}

int filter_bool(B2Context* ctx, const B2Array* values, const B2Array* mask, int null_selection, B2Array* out,
                cudaStream_t s) {
  const int64_t n = values->length;
  const bool has_valid = (values->null_count != 0 && values->validity) || (mask->null_count != 0 && mask->validity);
  if (n == 0) {
    fill_out(out, B2_BOOL, 0, 0, nullptr, nullptr);
    return B2_OK;
  }
  FilterBitmaps fb = make_filter_bitmaps(values, mask, null_selection);
  Temp offsets(ctx, s);
  int64_t out_len = 0, out_valid = 0;
  B2_RETURN_NOT_OK(filter_plan(ctx, fb, n, has_valid, &offsets, &out_len, &out_valid, s));
  Temp data(ctx, s), bits(ctx, s);
  const size_t bb = bitmap_alloc_bytes(out_len) + 8;
  B2_RETURN_NOT_OK(data.alloc(bb));
  B2_CUDA(cudaMemsetAsync(data.ptr, 0, bb, s));
  if (has_valid) {
    B2_RETURN_NOT_OK(bits.alloc(bb));
    B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bb, s));
  }
  if (out_len > 0) {
    BoolFilterArgs a;
    a.fb = fb;
    a.data = BitmapReader(values->data, values->offset, n);
    a.tile_offsets = offsets.as<int64_t>();
    a.out_data = data.as<unsigned long long>();
    a.out_validity = has_valid ? bits.as<unsigned long long>() : nullptr;
    filter_bool_kernel<<<(unsigned)tiles_for(n), 64, 0, s>>>(a);
    B2_LAUNCHED();
  }
  const int64_t null_count = has_valid ? out_len - out_valid : 0;
  fill_out(out, B2_BOOL, out_len, null_count, has_valid ? bits.release() : nullptr, data.release());
  return B2_OK;
}

// ---- take ----
template <typename Idx>
__global__ void __launch_bounds__(kBlock) take_bool_kernel(BitmapReader data, BitmapReader values_valid, int64_t values_length,
                                                           const Idx* __restrict__ idx, BitmapReader idx_valid, int64_t n,
                                                           uint32_t* out_data, uint32_t* out_validity, int64_t* valid_count,
                                                           unsigned long long* first_bad) {
  const int64_t nw = (n + 31) >> 5;
  int64_t local = 0;
  for (int64_t w = (blockIdx.x * (int64_t)kBlock + threadIdx.x) >> 5; w < nw; w += ((int64_t)gridDim.x * kBlock) >> 5) {
    const int64_t i = (w << 5) + lane_id();
    bool bit = false, ok = false;
    if (i < n && idx_valid.bit(i)) {
      const Idx raw = idx[i];
      const uint64_t j = std::is_unsigned<Idx>::value ? static_cast<uint64_t>(raw)
                                                      : static_cast<uint64_t>(static_cast<int64_t>(raw));
      if (j >= static_cast<uint64_t>(values_length)) {
        atomicMin(first_bad, static_cast<unsigned long long>(i));
      } else {
        ok = values_valid.bit(static_cast<int64_t>(j));
        bit = ok && data.bit(static_cast<int64_t>(j));
      }
    }
    const unsigned dw = __ballot_sync(0xffffffffu, bit), vw = __ballot_sync(0xffffffffu, ok);
    if (lane_id() == 0) {
      out_data[w] = dw;
      if (out_validity) out_validity[w] = vw;
      local += __popc(vw);
    }
  }
  int64_t sum = block_sum<kBlock>(local);
  if (threadIdx.x == 0 && sum) atomicAdd(reinterpret_cast<unsigned long long*>(valid_count), (unsigned long long)sum);
}

int take_bool(B2Context* ctx, const B2Array* values, const B2Array* indices, B2Array* out, cudaStream_t s) {
  const int64_t n = indices->length;
  if (n == 0) {
    fill_out(out, B2_BOOL, 0, 0, nullptr, nullptr);
    return B2_OK;
  }
  const bool has_valid = (values->null_count != 0 && values->validity) || (indices->null_count != 0 && indices->validity);
  Temp data(ctx, s), bits(ctx, s);
  const size_t bb = bitmap_alloc_bytes(n);
  B2_RETURN_NOT_OK(data.alloc(bb));
  B2_CUDA(cudaMemsetAsync(data.ptr, 0, bb, s));
  if (has_valid) {
    B2_RETURN_NOT_OK(bits.alloc(bb));
    B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bb, s));
  }
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  B2_CUDA(cudaMemsetAsync(slot.dev() + 1, 0xff, 8, s));
  BitmapReader dr(values->data, values->offset, values->length);
  BitmapReader vr(values->null_count == 0 ? nullptr : values->validity, values->offset, values->length);
  BitmapReader ir(indices->null_count == 0 ? nullptr : indices->validity, indices->offset, n);
  const int iw = type_width(indices->type);
  const void* ip = static_cast<const char*>(indices->data) + indices->offset * iw;
  const int grid = grid_for(n, kBlock * 4, kSMs * 16);
  B2_RETURN_NOT_OK(visit_type(
      IndexTypes{}, indices->type,
      [&](auto it) {
        using T = decltype(it);
        take_bool_kernel<T><<<grid, kBlock, 0, s>>>(dr, vr, values->length, static_cast<const T*>(ip), ir, n, data.as<uint32_t>(),
                                                    has_valid ? bits.as<uint32_t>() : nullptr, slot.dev(),
                                                    reinterpret_cast<unsigned long long*>(slot.dev() + 1));
        return B2_OK;
      },
      [&] { return index_type_error(indices->type); }));
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(slot.fetch(s));
  const uint64_t bad = static_cast<uint64_t>(slot.host()[1]);
  if (bad != ~0ull) return index_error(indices, bad, s);
  const int64_t null_count = has_valid ? n - slot.host()[0] : 0;
  fill_out(out, B2_BOOL, n, null_count, (has_valid && null_count) ? bits.release() : nullptr, data.release());
  return B2_OK;
}

}  // namespace b2
