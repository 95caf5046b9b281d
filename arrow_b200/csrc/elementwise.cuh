// elementwise.cuh -- the streaming applicator shared by cast / arithmetic / compare.
//
// Plays the role of the reference's ScalarUnary / ScalarBinary applicators
// (cpp/src/arrow/compute/kernels/codegen_internal.h:590-976): run an op functor over
// every slot (including slots under nulls, like the reference) of one or two inputs.
//
// Mapping: a warp owns 32*V*U consecutive elements; each lane issues U
// independent 16-byte (or narrower, for the narrower side of a widening op) streaming
// accesses striped by lane, so every instruction touches one contiguous 512-byte span
// (fully coalesced 128 B lines) and U requests are in flight per lane before the first
// use.  No shared memory: each byte is touched once (guide: element-wise kernels).
#pragma once
#include "common.cuh"
#include "context.h"

namespace b2 {

template <int NB>
struct Bytes;
template <>
struct Bytes<1> { using type = uint8_t; };
template <>
struct Bytes<2> { using type = uint16_t; };
template <>
struct Bytes<4> { using type = uint32_t; };
template <>
struct Bytes<8> { using type = uint2; };
template <>
struct Bytes<16> { using type = uint4; };

template <typename T, int V>
struct alignas(sizeof(T) * V) Vec {
  T v[V];
};

template <typename T, int V>
__device__ __forceinline__ Vec<T, V> load_vec(const T* p) {
  using B = typename Bytes<sizeof(T) * V>::type;
  B raw = __ldcs(reinterpret_cast<const B*>(p));
  Vec<T, V> r;
  *reinterpret_cast<B*>(&r) = raw;
  return r;
}
template <typename T, int V>
__device__ __forceinline__ void store_vec(T* p, const Vec<T, V>& x) {
  using B = typename Bytes<sizeof(T) * V>::type;
  __stcs(reinterpret_cast<B*>(p), *reinterpret_cast<const B*>(&x));
}

template <typename A, typename B>
constexpr int vec_elems() {
  return 16 / (sizeof(A) > sizeof(B) ? sizeof(A) : sizeof(B));
}

constexpr int kUnroll = 4;

// out[i] = f(in[i], i); U accesses in flight per lane (an op heavy in 64-bit constant divisions takes fewer so that
// its registers do not spill)
template <typename In, typename Out, int V, typename F, int U = kUnroll>
__global__ void __launch_bounds__(kBlock) map1_kernel(const In* __restrict__ in,
                                                      Out* __restrict__ out, int64_t n,
                                                      bool vec_ok, F f) {
  constexpr int64_t kWarpTile = 32 * V * U;
  constexpr int64_t kTile = kWarpTile * kWarpsPerBlock;
  const unsigned lane = lane_id();
  for (int64_t tile = (int64_t)blockIdx.x * kTile; tile < n; tile += (int64_t)gridDim.x * kTile) {
    int64_t wb = tile + (int64_t)(threadIdx.x >> 5) * kWarpTile;
    if (wb >= n) continue;
    if (vec_ok && wb + kWarpTile <= n) {
      Vec<In, V> x[U];
#pragma unroll
      for (int u = 0; u < U; ++u) x[u] = load_vec<In, V>(in + wb + u * 32 * V + lane * V);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        Vec<Out, V> y;
        int64_t i0 = wb + u * 32 * V + lane * V;
#pragma unroll
        for (int k = 0; k < V; ++k) y.v[k] = f(x[u].v[k], i0 + k);
        store_vec<Out, V>(out + i0, y);
      }
    } else {
      int64_t end = wb + kWarpTile < n ? wb + kWarpTile : n;
      for (int64_t i = wb + lane; i < end; i += 32) out[i] = f(in[i], i);
    }
  }
}

// out[i] = f(a[i] or sa, b[i] or sb, i); a == nullptr means broadcast scalar sa.  The right operand has its own type
// In2 where the op takes one (round_binary's int32 digit count); V must then suit the wider of In and In2.  U as for
// map1_kernel.
template <typename In, typename Out, int V, typename F, typename In2 = In, int U = kUnroll>
__global__ void __launch_bounds__(kBlock) map2_kernel(const In* __restrict__ a, In sa,
                                                      const In2* __restrict__ b, In2 sb,
                                                      Out* __restrict__ out, int64_t n,
                                                      bool vec_ok, F f) {
  constexpr int64_t kWarpTile = 32 * V * U;
  constexpr int64_t kTile = kWarpTile * kWarpsPerBlock;
  const unsigned lane = lane_id();
  for (int64_t tile = (int64_t)blockIdx.x * kTile; tile < n; tile += (int64_t)gridDim.x * kTile) {
    int64_t wb = tile + (int64_t)(threadIdx.x >> 5) * kWarpTile;
    if (wb >= n) continue;
    if (vec_ok && wb + kWarpTile <= n) {
      Vec<In, V> x[U];
      Vec<In2, V> y[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        int64_t i0 = wb + u * 32 * V + lane * V;
        if (a) {
          x[u] = load_vec<In, V>(a + i0);
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) x[u].v[k] = sa;
        }
        if (b) {
          y[u] = load_vec<In2, V>(b + i0);
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) y[u].v[k] = sb;
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        Vec<Out, V> z;
        int64_t i0 = wb + u * 32 * V + lane * V;
#pragma unroll
        for (int k = 0; k < V; ++k) z.v[k] = f(x[u].v[k], y[u].v[k], i0 + k);
        store_vec<Out, V>(out + i0, z);
      }
    } else {
      int64_t end = wb + kWarpTile < n ? wb + kWarpTile : n;
      // not unrolled: the hoisted bounds of an unrolled tail would otherwise be spilled
#pragma unroll 1
      for (int64_t i = wb + lane; i < end; i += 32) out[i] = f(a ? a[i] : sa, b ? b[i] : sb, i);
    }
  }
}

template <typename In, typename Out, int V, int U = kUnroll>
inline int map_grid(int64_t n) {
  constexpr int64_t kTile = (int64_t)32 * V * U * kWarpsPerBlock;
  // up to 16 CTA-waves over the 132 SMs; beyond that CTAs loop (grid-stride)
  return grid_for(n, kTile, kSMs * 8 * 16);
}

// first-error cell of the checked casts: rows race with atomicMin so the
// reported element is the first offending row, as the reference's in-order scan finds.
struct ErrorCell {
  unsigned long long* first_row;  // device; initialised to ~0ull
  __device__ __forceinline__ void report(int64_t row) const {
    atomicMin(first_row, static_cast<unsigned long long>(row));
  }
};

// last-error cell of the checked arithmetic: the reference's applicator (ScalarBinaryNotNullStateful,
// codegen_internal.h:878-976) runs every row and each failing row overwrites the status, so the
// message ("divide by zero" or "overflow") is that of the LAST offending row.  Holds row + 1.
struct LastErrorCell {
  unsigned long long* last_row1;  // device; initialised to 0 (no error)
  __device__ __forceinline__ void report(int64_t row) const {
    atomicMax(last_row1, static_cast<unsigned long long>(row) + 1ull);
  }
};

// res = a * b wrapped to T, and whether the exact product leaves T (MultiplyWithOverflow, util/int_util_overflow.h)
template <typename T>
__device__ __forceinline__ bool mul_overflow(T a, T b, T* res) {
  if constexpr (sizeof(T) < 8) {
    using Wide = typename std::conditional<std::is_signed<T>::value, int64_t, uint64_t>::type;
    const Wide p = static_cast<Wide>(a) * static_cast<Wide>(b);
    *res = static_cast<T>(p);
    return static_cast<Wide>(*res) != p;
  } else if constexpr (std::is_signed<T>::value) {
    *res = static_cast<T>(static_cast<uint64_t>(a) * static_cast<uint64_t>(b));
    return __mul64hi(static_cast<long long>(a), static_cast<long long>(b)) != (static_cast<long long>(*res) >> 63);
  } else {
    *res = a * b;
    return __umul64hi(a, b) != 0;
  }
}

// the operands of a binary arithmetic or compare call: their common type, length, and whether a scalar is null
inline int unpack_operands(const B2Value* left, const B2Value* right, int* type, int64_t* length, bool* null_scalar) {
  if (!left || !right) return set_error(B2_INVALID, "null operand");
  const B2Array* la = left->array;
  const B2Array* ra = right->array;
  if (!la && !left->scalar) return set_error(B2_INVALID, "left operand has neither array nor scalar");
  if (!ra && !right->scalar) return set_error(B2_INVALID, "right operand has neither array nor scalar");
  if (!la && !ra) return set_error(B2_INVALID, "at least one operand must be an array");
  int lt = la ? la->type : left->scalar->type;
  int rt = ra ? ra->type : right->scalar->type;
  if (lt != rt)
    return set_error(B2_TYPE_ERROR, "operand types differ (%d vs %d); dispatch must cast first", lt, rt);
  if (la && ra && la->length != ra->length)
    return set_error(B2_INVALID, "Array arguments must all be the same length");
  *type = lt;
  *length = la ? la->length : ra->length;
  *null_scalar = (!la && !left->scalar->is_valid) || (!ra && !right->scalar->is_valid);
  return B2_OK;
}

// the bits of operand v at `row` (a scalar's own bits), zero-extended from `w` bytes: what a failing row's message is
// built from
inline int operand_bits(const B2Value* v, int64_t row, int w, uint64_t* bits, cudaStream_t s) {
  *bits = 0;
  if (v->array) {
    B2_CUDA(cudaMemcpyAsync(bits, static_cast<const char*>(v->array->data) + (v->array->offset + row) * w, w,
                            cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
  } else {
    memcpy(bits, &v->scalar->bits, w);
  }
  return B2_OK;
}

// the Arrow name of a type id ("int8", "double"; scalar_cast.cu)
const char* type_name(int t);

// a scalar operand's value (T{} for an array operand)
template <typename T>
T scalar_bits(const B2Scalar* s) {
  T v{};
  if (s) memcpy(&v, &s->bits, sizeof(T));
  return v;
}

}  // namespace b2
