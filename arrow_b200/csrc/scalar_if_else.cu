// scalar_if_else.cu -- if_else(cond, left, right) over fixed-width and boolean columns.
//
// Replaces (SURVEY.md section 8f rank 3) IfElseFunctor<Type>::Call and its AAA / ASA / AAS / ASS shapes
// (cpp/src/arrow/compute/kernels/scalar_if_else.cc:62-330 for the validity rules of PromoteNullsVisitor,
// :353-520 for the number and boolean functors):
//   out[i]       = cond[i] ? left[i] : right[i]
//   out valid[i] = cond valid[i] AND (cond[i] ? left valid[i] : right valid[i])
// cond is a boolean array or scalar; left / right are arrays or scalars of ONE type (the caller applies the
// reference's DispatchBest casts).  Bytes under a null output slot are unspecified, as in the reference.
//
// Design: two streaming passes that never meet.  The VALUE pass reads cond (1 bit / row) and both value
// columns with 16-byte loads and writes 16-byte stores -- a random cond touches every 32-byte sector of both
// inputs anyway, so predicating the loads would save nothing: (1/8 + 3 w) B per row, pure HBM streaming.  The
// VALIDITY pass runs only when some operand can be null and works on whole 64-bit words of the bitmaps
// (funnel-shifted, any bit offset): 5/8 B per row.  Boolean left / right are bitmaps themselves, so their value
// pass is the same word kernel.
#include <cstring>

#include "bitmap.h"
#include "elementwise.cuh"

namespace b2 {

struct BitOperand {  // a bitmap operand of the word kernels: an array's bitmap, or a broadcast scalar word
  BitmapReader bits;
  uint64_t scalar;
  bool is_scalar;
  __device__ __forceinline__ uint64_t word(int64_t w) const { return is_scalar ? scalar : bits.word(w); }
};

// out = (c & l) | (~c & r), optionally ANDed with `gate` (the cond validity); counts the set bits when asked
__global__ void __launch_bounds__(kBlock) if_else_words_kernel(BitOperand c, BitOperand l, BitOperand r, BitOperand gate,
                                                               bool gated, int64_t n, int64_t nwords, uint64_t* out,
                                                               int64_t* set_count) {
  int64_t local = 0;
  for (int64_t w = blockIdx.x * (int64_t)kBlock + threadIdx.x; w < nwords; w += (int64_t)gridDim.x * kBlock) {
    const int64_t rem = n - (w << 6);
    const uint64_t keep = rem >= 64 ? ~0ull : ((1ull << rem) - 1ull);
    const uint64_t cw = c.word(w);
    uint64_t o = (cw & l.word(w)) | (~cw & r.word(w));
    if (gated) o &= gate.word(w);
    o &= keep;
    out[w] = o;
    local += __popcll(o);
  }
  if (set_count) {
    int64_t s = block_sum<kBlock>(local);
    if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(set_count), (unsigned long long)s);
  }
}

template <int W>
struct IfElseBytes;
template <> struct IfElseBytes<1> { using type = uint8_t; };
template <> struct IfElseBytes<2> { using type = uint16_t; };
template <> struct IfElseBytes<4> { using type = uint32_t; };
template <> struct IfElseBytes<8> { using type = uint64_t; };

struct IfElseArgs {
  BitOperand cond;
  const void* left;   // NULL: broadcast left_scalar
  const void* right;  // NULL: broadcast right_scalar
  uint64_t left_scalar, right_scalar;
  void* out;
  int64_t n;
  bool vec_ok;
};

// One lane = V consecutive rows = one 16-byte store; the V cond bits of a lane never straddle a 64-bit word (V is a
// power of two <= 16 and the lane's first row is a multiple of V).
template <int W>
__global__ void __launch_bounds__(kBlock) if_else_values_kernel(IfElseArgs a) {
  using T = typename IfElseBytes<W>::type;
  constexpr int V = 16 / W;
  const T* __restrict__ L = static_cast<const T*>(a.left);
  const T* __restrict__ R = static_cast<const T*>(a.right);
  T* __restrict__ out = static_cast<T*>(a.out);
  const T ls = static_cast<T>(a.left_scalar), rs = static_cast<T>(a.right_scalar);
  const int64_t n_vec = a.vec_ok ? a.n / V : 0;
  constexpr int U = 4;
  const int64_t stride = (int64_t)gridDim.x * kBlock;
  for (int64_t j0 = blockIdx.x * (int64_t)kBlock + threadIdx.x; j0 < n_vec; j0 += stride * U) {
    uint4 lv[U], rv[U];
    unsigned cb[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t j = j0 + u * stride;
      if (j < n_vec) {
        if (L) lv[u] = __ldcs(reinterpret_cast<const uint4*>(L) + j);
        if (R) rv[u] = __ldcs(reinterpret_cast<const uint4*>(R) + j);
        const int64_t i0 = j * V;
        cb[u] = static_cast<unsigned>(a.cond.word(i0 >> 6) >> (i0 & 63));
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t j = j0 + u * stride;
      if (j >= n_vec) continue;
      uint4 o;
      T* ov = reinterpret_cast<T*>(&o);
      const T* lp = reinterpret_cast<const T*>(&lv[u]);
      const T* rp = reinterpret_cast<const T*>(&rv[u]);
#pragma unroll
      for (int e = 0; e < V; ++e) {
        const T x = L ? lp[e] : ls, y = R ? rp[e] : rs;
        ov[e] = ((cb[u] >> e) & 1u) ? x : y;
      }
      __stcs(reinterpret_cast<uint4*>(out) + j, o);
    }
  }
  // tail rows (and every row of an unaligned operand)
  for (int64_t i = n_vec * V + blockIdx.x * (int64_t)kBlock + threadIdx.x; i < a.n; i += stride) {
    const bool c = (a.cond.word(i >> 6) >> (i & 63)) & 1ull;
    const T x = L ? L[i] : ls, y = R ? R[i] : rs;
    out[i] = c ? x : y;
  }
}

// cond: boolean array or scalar.  `data` = its value bits (false under a null scalar), `valid` = its validity.
static int make_cond(const B2Value* v, int64_t* length, BitOperand* data, BitOperand* valid, bool* may_null) {
  memset(data, 0, sizeof(*data));
  memset(valid, 0, sizeof(*valid));
  if (v->array) {
    const B2Array* a = v->array;
    if (a->type != B2_BOOL) return set_error(B2_TYPE_ERROR, "if_else: cond must be boolean (type id %d)", a->type);
    if (a->length < 0 || a->offset < 0) return set_error(B2_INVALID, "negative length/offset");
    *length = a->length;
    data->bits = BitmapReader(a->data, a->offset, a->length);
    *may_null = a->validity && a->null_count != 0;
    valid->bits = BitmapReader(*may_null ? a->validity : nullptr, a->offset, a->length);
    valid->is_scalar = !*may_null;
    valid->scalar = ~0ull;
  } else if (v->scalar) {
    if (v->scalar->type != B2_BOOL) return set_error(B2_TYPE_ERROR, "if_else: cond must be boolean");
    data->is_scalar = valid->is_scalar = true;
    data->scalar = (v->scalar->is_valid && (v->scalar->bits & 1)) ? ~0ull : 0ull;
    valid->scalar = v->scalar->is_valid ? ~0ull : 0ull;
    *may_null = !v->scalar->is_valid;
  } else {
    return set_error(B2_INVALID, "if_else: empty cond");
  }
  return B2_OK;
}

struct Branch {  // left or right
  int32_t type = B2_NA;
  const B2Array* array = nullptr;
  uint64_t scalar_bits = 0;
  bool may_null = false;
  BitOperand valid{};
};

static int make_branch(const B2Value* v, int64_t* length, Branch* b, const char* side) {
  if (v->array) {
    const B2Array* a = v->array;
    if (a->length < 0 || a->offset < 0) return set_error(B2_INVALID, "negative length/offset");
    if (*length >= 0 && *length != a->length) return set_error(B2_INVALID, "Array arguments must all be the same length");
    *length = a->length;
    b->type = a->type;
    b->array = a;
    b->may_null = a->validity && a->null_count != 0;
    b->valid.bits = BitmapReader(b->may_null ? a->validity : nullptr, a->offset, a->length);
    b->valid.is_scalar = !b->may_null;
    b->valid.scalar = ~0ull;
  } else if (v->scalar) {
    b->type = v->scalar->type;
    b->scalar_bits = v->scalar->bits;
    b->may_null = !v->scalar->is_valid;
    b->valid.is_scalar = true;
    b->valid.scalar = v->scalar->is_valid ? ~0ull : 0ull;
  } else {
    return set_error(B2_INVALID, "if_else: empty %s operand", side);
  }
  return B2_OK;
}

template <int W>
static int launch_values(const IfElseArgs& a, int sm_count, cudaStream_t s) {
  constexpr int V = 16 / W;
  if_else_values_kernel<W><<<grid_for(a.n, (int64_t)kBlock * V * 4, sm_count * 8), kBlock, 0, s>>>(a);
  return B2_OK;
}

}  // namespace b2

using namespace b2;

extern "C" int b2_if_else(B2Context* ctx, const B2Value* cond, const B2Value* left, const B2Value* right, B2Array* out,
                          void* stream) {
  if (!ctx || !cond || !left || !right || !out) return set_error(B2_INVALID, "b2_if_else: null argument");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  int64_t n = -1;
  BitOperand cdata, cvalid;
  bool cond_may_null = false;
  B2_RETURN_NOT_OK(make_cond(cond, &n, &cdata, &cvalid, &cond_may_null));
  Branch l, r;
  B2_RETURN_NOT_OK(make_branch(left, &n, &l, "left"));
  B2_RETURN_NOT_OK(make_branch(right, &n, &r, "right"));
  if (n < 0) return set_error(B2_NOT_IMPLEMENTED, "if_else: at least one argument must be an array");
  if (l.type != r.type)
    return set_error(B2_TYPE_ERROR, "if_else: left and right must have the same type after dispatch (type ids %d, %d)", l.type, r.type);
  const int32_t t = l.type;
  const int w = type_width(t);
  if (t != B2_BOOL && w == 0) return set_error(B2_NOT_IMPLEMENTED, "if_else over type id %d", t);

  Temp data(ctx, s), bits(ctx, s);
  const int64_t nwords = bitmap_words64(n);
  B2_RETURN_NOT_OK(data.alloc(t == B2_BOOL ? bitmap_alloc_bytes(n) : (size_t)(n > 0 ? n : 1) * w));
  if (n == 0) {
    fill_out(out, t, 0, 0, nullptr, data.release());
    return B2_OK;
  }
  const int wgrid = grid_for(nwords, kBlock, kSMs * 8);
  if (t == B2_BOOL) {
    BitOperand ld{}, rd{};
    if (l.array) ld.bits = BitmapReader(l.array->data, l.array->offset, n);
    else { ld.is_scalar = true; ld.scalar = (l.scalar_bits & 1) ? ~0ull : 0ull; }
    if (r.array) rd.bits = BitmapReader(r.array->data, r.array->offset, n);
    else { rd.is_scalar = true; rd.scalar = (r.scalar_bits & 1) ? ~0ull : 0ull; }
    B2_CUDA(cudaMemsetAsync(static_cast<char*>(data.ptr) + nwords * 8, 0, 8, s));
    if_else_words_kernel<<<wgrid, kBlock, 0, s>>>(cdata, ld, rd, cvalid, false, n, nwords, data.as<uint64_t>(), nullptr);
    B2_LAUNCHED();
  } else {
    IfElseArgs a{};
    a.cond = cdata;
    a.left = l.array ? static_cast<const char*>(l.array->data) + l.array->offset * w : nullptr;
    a.right = r.array ? static_cast<const char*>(r.array->data) + r.array->offset * w : nullptr;
    a.left_scalar = l.scalar_bits;
    a.right_scalar = r.scalar_bits;
    a.out = data.ptr;
    a.n = n;
    a.vec_ok = (!a.left || aligned_to(a.left, 16)) && (!a.right || aligned_to(a.right, 16));
    B2_RETURN_NOT_OK((visit_width<1, 2, 4, 8>(w, [&](auto wc) { return launch_values<wc>(a, ctx->sm_count, s); })));
    B2_LAUNCHED();
  }
  int64_t nulls = 0;
  if (cond_may_null || l.may_null || r.may_null) {
    B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(n)));
    B2_CUDA(cudaMemsetAsync(static_cast<char*>(bits.ptr) + nwords * 8, 0, 8, s));
    ScalarSlot slot(ctx);
    B2_RETURN_NOT_OK(slot.zero(s));
    if_else_words_kernel<<<wgrid, kBlock, 0, s>>>(cdata, l.valid, r.valid, cvalid, true, n, nwords, bits.as<uint64_t>(), slot.dev());
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(slot.fetch(s));
    nulls = n - slot.host()[0];
  }
  fill_out(out, t, n, nulls, nulls ? bits.release() : nullptr, data.release());
  return B2_OK;
}
