// bitmap.cu -- validity-bitmap primitives.
//
// Replaces internal::CopyBitmap / BitmapAnd / CountSetBits
// (cpp/src/arrow/util/bitmap_ops.cc:40-330) as used by the executor's NullPropagator
// (cpp/src/arrow/compute/exec.cc:527-686, PropagateNullsSpans :1222-1281): output
// validity of a scalar kernel = AND of the input validities, re-based to offset 0.
//
// One thread produces one aligned 64-bit output word from funnel-shifted input
// words, so arbitrary (non byte-aligned) slice offsets cost one extra load.
// Algorithmic bytes: 1/8 B per row per bitmap read or written.
#include "bitmap.h"

namespace b2 {

__global__ void __launch_bounds__(kBlock) bitmap_and_kernel(BitmapReader a, BitmapReader b,
                                                            int64_t nwords, uint64_t* dst,
                                                            int64_t* count) {
  int64_t local = 0;
  for (int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; w < nwords;
       w += (int64_t)gridDim.x * blockDim.x) {
    uint64_t v = a.word(w) & b.word(w);
    if (dst) dst[w] = v;
    local += __popcll(v);
  }
  if (count) {
    int64_t s = block_sum<kBlock>(local);
    if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(count), (unsigned long long)s);
  }
}

int launch_bitmap_and(const void* a, int64_t a_off, const void* b, int64_t b_off, int64_t length,
                      void* dst, int64_t* d_count, cudaStream_t s) {
  if (length <= 0) return B2_OK;
  int64_t nwords = bitmap_words64(length);
  BitmapReader ra(a, a_off, length), rb(b, b_off, length);
  int grid = grid_for(nwords, kBlock, kSMs * 8);
  bitmap_and_kernel<<<grid, kBlock, 0, s>>>(ra, rb, nwords, static_cast<uint64_t*>(dst), d_count);
  B2_LAUNCHED();
  return B2_OK;
}

// single block: 1024 threads, each scans a contiguous span of in[], then one warp scans the 32 warp totals
__global__ void __launch_bounds__(1024) exclusive_scan_i64_kernel(const int64_t* __restrict__ in, int64_t n, int64_t* __restrict__ out,
                                                                  int64_t* total) {
  __shared__ int64_t warp_tot[32];
  const int t = threadIdx.x;
  const int64_t per = (n + 1023) / 1024;
  const int64_t lo = t * per, hi = lo + per < n ? lo + per : n;
  int64_t sum = 0;
  for (int64_t i = lo; i < hi; ++i) sum += in[i];
  int64_t incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if ((t & 31) >= o) incl += v;
  }
  if ((t & 31) == 31) warp_tot[t >> 5] = incl;
  __syncthreads();
  if (t < 32) {
    const int64_t w = warp_tot[t];
    int64_t wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t v = __shfl_up_sync(0xffffffffu, wi, o);
      if (t >= o) wi += v;
    }
    warp_tot[t] = wi - w;
    if (t == 31 && total) *total = wi;
  }
  __syncthreads();
  int64_t run = warp_tot[t >> 5] + incl - sum;
  for (int64_t i = lo; i < hi; ++i) {
    out[i] = run;
    run += in[i];
  }
}

int launch_exclusive_scan_i64(const int64_t* in, int64_t n, int64_t* out, int64_t* total, cudaStream_t s) {
  exclusive_scan_i64_kernel<<<1, 1024, 0, s>>>(in, n, out, total);
  B2_LAUNCHED();
  return B2_OK;
}

int make_validity(B2Context* ctx, const B2Array* a, const B2Array* b, int64_t length,
                  void** out_validity, int64_t* out_null_count, cudaStream_t s) {
  *out_validity = nullptr;
  *out_null_count = 0;
  const void* va = (a && a->validity && a->null_count != 0) ? a->validity : nullptr;
  const void* vb = (b && b->validity && b->null_count != 0) ? b->validity : nullptr;
  if ((!va && !vb) || length == 0) return B2_OK;
  Temp bits(ctx, s);
  B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(length)));
  // single known-null-count input: plain re-based copy, no read-back needed
  bool need_count = !((va && !vb && a->null_count >= 0) || (vb && !va && b->null_count >= 0));
  if (need_count) {
    ScalarSlot slot(ctx);
    B2_RETURN_NOT_OK(slot.zero(s));
    B2_RETURN_NOT_OK(launch_bitmap_and(va, a ? a->offset : 0, vb, b ? b->offset : 0, length,
                                       bits.ptr, slot.dev(), s));
    B2_RETURN_NOT_OK(slot.fetch(s));
    *out_null_count = length - slot.host()[0];
  } else {
    B2_RETURN_NOT_OK(launch_bitmap_and(va, a ? a->offset : 0, vb, b ? b->offset : 0, length,
                                       bits.ptr, nullptr, s));
    *out_null_count = va ? a->null_count : b->null_count;
  }
  if (*out_null_count == 0) return B2_OK;  // all valid: drop the bitmap like the reference
  *out_validity = bits.release();
  return B2_OK;
}

}  // namespace b2

using namespace b2;

extern "C" {

int b2_bitmap_count(B2Context* ctx, const void* bits, int64_t offset, int64_t length,
                    int64_t* out_count, void* stream) {
  if (!ctx || !out_count) return set_error(B2_INVALID, "b2_bitmap_count: null argument");
  if (length < 0 || offset < 0) return set_error(B2_INVALID, "negative length/offset");
  if (length == 0) {
    *out_count = 0;
    return B2_OK;
  }
  if (!bits) {
    *out_count = length;
    return B2_OK;
  }
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  B2_RETURN_NOT_OK(launch_bitmap_and(bits, offset, nullptr, 0, length, nullptr, slot.dev(), s));
  B2_RETURN_NOT_OK(slot.fetch(s));
  *out_count = slot.host()[0];
  return B2_OK;
}

int b2_bitmap_copy(B2Context* ctx, const void* src, int64_t src_offset, int64_t length, void* dst,
                   void* stream) {
  if (!ctx || !dst) return set_error(B2_INVALID, "b2_bitmap_copy: null argument");
  if (length < 0 || src_offset < 0) return set_error(B2_INVALID, "negative length/offset");
  B2_CUDA(cudaSetDevice(ctx->device));
  return launch_bitmap_and(src, src_offset, nullptr, 0, length, dst, nullptr, ctx->pick(stream));
}

int b2_bitmap_and(B2Context* ctx, const void* a, int64_t a_offset, const void* b, int64_t b_offset,
                  int64_t length, void* dst, int64_t* out_count, void* stream) {
  if (!ctx || !dst) return set_error(B2_INVALID, "b2_bitmap_and: null argument");
  if (length < 0 || a_offset < 0 || b_offset < 0) return set_error(B2_INVALID, "negative length/offset");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  if (!out_count) return launch_bitmap_and(a, a_offset, b, b_offset, length, dst, nullptr, s);
  if (length == 0) {
    *out_count = 0;
    return B2_OK;
  }
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  B2_RETURN_NOT_OK(launch_bitmap_and(a, a_offset, b, b_offset, length, dst, slot.dev(), s));
  B2_RETURN_NOT_OK(slot.fetch(s));
  *out_count = slot.host()[0];
  return B2_OK;
}

}  // extern "C"
