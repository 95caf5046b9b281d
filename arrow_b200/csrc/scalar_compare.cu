// scalar_compare.cu -- equal / not_equal / greater / greater_equal / less / less_equal
// over numeric inputs, producing Arrow's bit-packed boolean layout.
//
// Replaces ComparePrimitive{ArrayArray,ArrayScalar,ScalarArray} + CompareKernel::Exec
// (cpp/src/arrow/compute/kernels/scalar_compare.cc:164-303) and the op functors
// Equal/NotEqual/Greater/GreaterEqual (:42-72); less/less_equal are greater/
// greater_equal with the operands swapped, as MakeFlippedCompare does (:910).
// The reference packs 32 results at a time with PackBits; here a warp's 32*V results
// of one coalesced 16-byte-per-lane load become V output words through V
// warp-wide OR reductions (redux.sync), so no shared memory and no atomics.
//
// Roofline: HBM-bound; algorithmic bytes/row = 2*sizeof(T) + 1/8 (+3/8 with validity).
#include <type_traits>

#include "bitmap.h"
#include "elementwise.cuh"

namespace b2 {

template <typename T, int OP>
__device__ __forceinline__ bool cmp(T l, T r) {
  if constexpr (OP == B2_EQUAL) return l == r;
  else if constexpr (OP == B2_NOT_EQUAL) return l != r;
  else if constexpr (OP == B2_GREATER) return l > r;
  else return l >= r;
}

template <typename T, int OP>
__global__ void __launch_bounds__(kBlock) compare_kernel(const T* __restrict__ a, T sa,
                                                         const T* __restrict__ b, T sb,
                                                         uint32_t* __restrict__ out, int64_t n,
                                                         bool vec_ok) {
  constexpr int V = 16 / sizeof(T);
  constexpr int UU = kUnroll;
  constexpr int64_t kWarpTile = 32 * V * UU;
  constexpr int64_t kTile = kWarpTile * kWarpsPerBlock;
  const unsigned lane = lane_id();
  for (int64_t tile = (int64_t)blockIdx.x * kTile; tile < n; tile += (int64_t)gridDim.x * kTile) {
    int64_t wb = tile + (int64_t)(threadIdx.x >> 5) * kWarpTile;
    if (wb >= n) continue;
    if (vec_ok && wb + kWarpTile <= n) {
      Vec<T, V> x[UU], y[UU];
#pragma unroll
      for (int u = 0; u < UU; ++u) {
        int64_t i0 = wb + u * 32 * V + lane * V;
        if (a) {
          x[u] = load_vec<T, V>(a + i0);
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) x[u].v[k] = sa;
        }
        if (b) {
          y[u] = load_vec<T, V>(b + i0);
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) y[u].v[k] = sb;
        }
      }
#pragma unroll
      for (int u = 0; u < UU; ++u) {
        unsigned m = 0;
#pragma unroll
        for (int k = 0; k < V; ++k) m |= (cmp<T, OP>(x[u].v[k], y[u].v[k]) ? 1u : 0u) << k;
        // lane's V bits sit at bit (lane*V) of the warp's V-word span
        const unsigned my_word = (lane * V) >> 5;
        const unsigned shifted = m << ((lane * V) & 31);
        unsigned mine = 0;
#pragma unroll
        for (int j = 0; j < V; ++j) {
          unsigned w = __reduce_or_sync(0xffffffffu, my_word == j ? shifted : 0u);
          if (lane == j) mine = w;
        }
        if (lane < V) out[((wb + u * 32 * V) >> 5) + lane] = mine;
      }
    } else {
      int64_t end = wb + kWarpTile < n ? wb + kWarpTile : n;
      for (int64_t base = wb; base < end; base += 32) {
        int64_t i = base + lane;
        bool bit = false;
        if (i < end) bit = cmp<T, OP>(a ? a[i] : sa, b ? b[i] : sb);
        unsigned w = __ballot_sync(0xffffffffu, bit);
        if (lane == 0) out[base >> 5] = w;
      }
    }
  }
}

template <typename T>
static int run_compare(int op, const T* a, T sa, const T* b, T sb, uint32_t* out, int64_t n,
                       cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  bool vec_ok = (!a || aligned_to(a, 16)) && (!b || aligned_to(b, 16));
  int grid = map_grid<T, T, V>(n);
  // less(a,b) = greater(b,a)
  if (op == B2_LESS || op == B2_LESS_EQUAL) {
    const T* tp = a; a = b; b = tp;
    T ts = sa; sa = sb; sb = ts;
    op = (op == B2_LESS) ? B2_GREATER : B2_GREATER_EQUAL;
  }
  switch (op) {
    case B2_EQUAL: compare_kernel<T, B2_EQUAL><<<grid, kBlock, 0, s>>>(a, sa, b, sb, out, n, vec_ok); break;
    case B2_NOT_EQUAL: compare_kernel<T, B2_NOT_EQUAL><<<grid, kBlock, 0, s>>>(a, sa, b, sb, out, n, vec_ok); break;
    case B2_GREATER: compare_kernel<T, B2_GREATER><<<grid, kBlock, 0, s>>>(a, sa, b, sb, out, n, vec_ok); break;
    case B2_GREATER_EQUAL: compare_kernel<T, B2_GREATER_EQUAL><<<grid, kBlock, 0, s>>>(a, sa, b, sb, out, n, vec_ok); break;
    default: return set_error(B2_INVALID, "unknown compare op %d", op);
  }
  B2_LAUNCHED();
  return B2_OK;
}

}  // namespace b2

using namespace b2;

extern "C" int b2_compare(B2Context* ctx, int op, const B2Value* left, const B2Value* right,
                          B2Array* out, void* stream) {
  if (!ctx || !out) return set_error(B2_INVALID, "b2_compare: null argument");
  int type;
  int64_t n;
  bool null_scalar;
  B2_RETURN_NOT_OK(unpack_operands(left, right, &type, &n, &null_scalar));
  if (!type_is_numeric(type)) return set_error(B2_NOT_IMPLEMENTED, "compare on type id %d", type);
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const B2Array* la = left->array;
  const B2Array* ra = right->array;

  Temp data(ctx, s);
  const size_t out_bytes = bitmap_alloc_bytes(n);
  B2_RETURN_NOT_OK(data.alloc(out_bytes));
  // zero the tail words so padding bits past `length` are clean
  {
    size_t tail = out_bytes >= 24 ? out_bytes - 24 : 0;
    B2_CUDA(cudaMemsetAsync(static_cast<char*>(data.ptr) + tail, 0, out_bytes - tail, s));
  }
  if (null_scalar) {
    Temp bits(ctx, s);
    B2_RETURN_NOT_OK(bits.alloc(out_bytes));
    B2_CUDA(cudaMemsetAsync(bits.ptr, 0, out_bytes, s));
    B2_CUDA(cudaMemsetAsync(data.ptr, 0, out_bytes, s));
    fill_out(out, B2_BOOL, n, n, n ? bits.release() : nullptr, data.release());
    return B2_OK;
  }
  void* validity = nullptr;
  int64_t null_count = 0;
  B2_RETURN_NOT_OK(make_validity(ctx, la, ra, n, &validity, &null_count, s));
  Temp vguard(ctx, s);
  vguard.ptr = validity;
  if (n > 0) {
    B2_RETURN_NOT_OK(visit_type(NumericTypes{}, type, [&](auto tag) {
      using T = decltype(tag);
      const T* a = la ? static_cast<const T*>(la->data) + la->offset : nullptr;
      const T* b = ra ? static_cast<const T*>(ra->data) + ra->offset : nullptr;
      return run_compare<T>(op, a, scalar_bits<T>(left->scalar), b, scalar_bits<T>(right->scalar),
                            static_cast<uint32_t*>(data.ptr), n, s);
    }));
  }
  fill_out(out, B2_BOOL, n, null_count, vguard.release(), data.release());
  return B2_OK;
}
