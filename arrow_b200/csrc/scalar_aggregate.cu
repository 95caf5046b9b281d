// scalar_aggregate.cu -- ungrouped sum / mean / min_max / count of one numeric column.
//
// Replaces (SURVEY section 8f rank 2, the ungrouped half):
//   SumImpl / MeanImpl            kernels/aggregate_basic.inc.cc:49-107,227-290
//   MinMaxState / MinMaxImpl      kernels/aggregate_basic.inc.cc:657-701,776-860
//   CountImpl                     kernels/aggregate_basic.cc:98-130
//   SumArray (pairwise summation) kernels/aggregate_internal.h
// One pass computes everything those kernels keep as state -- valid count, sum in the
// reference's accumulator type (int64 / uint64 / double, FindAccumulatorType), min and max --
// and the host side applies ScalarAggregateOptions{skip_nulls, min_count} exactly like the
// reference's Finalize.  Integer sums wrap like the reference's unsigned accumulation; float
// sums are accumulated in double per thread and combined in a fixed tree order, so the result
// is deterministic but may differ from the reference's pairwise order in the last bits
// (tests use rtol 1e-12).  Float min/max ignore NaNs (std::fmin/fmax) and are NaN when every
// value is NaN, as MinMaxState's quiet_NaN identity gives.
//
// Design: HBM streaming, W + 1/8 bytes read per row, nothing written.
// Every lane loads 16 bytes per step (a warp covers 64..512 rows and 1..8 validity words), four
// steps in flight; block partials go to global memory and a single CTA folds them in a fixed
// order; the five result words come back through the call's pinned slot.
#include <cmath>
#include <limits>
#include <type_traits>

#include "bitmap.h"

namespace b2 {

template <typename T>
struct AccOf {
  using type = typename std::conditional<std::is_floating_point<T>::value, double,
                                         typename std::conditional<std::is_signed<T>::value, long long, unsigned long long>::type>::type;
};

template <typename T>
struct Partial {
  typename AccOf<T>::type sum;
  long long hi;  // integers: bits 64..127 of the exact sum (MeanImpl must not see the int64 wrap-around)
  long long count;
  T mn, mx;
};

template <typename T>
__device__ __forceinline__ void partial_init(Partial<T>& p) {
  p.sum = 0;
  p.hi = 0;
  p.count = 0;
  if (std::is_floating_point<T>::value) {
    p.mn = p.mx = static_cast<T>(nan(""));
  } else {
    p.mn = std::numeric_limits<T>::max();
    p.mx = std::numeric_limits<T>::lowest();
  }
}

template <typename T>
__device__ __forceinline__ T min_of(T a, T b) {
  if constexpr (std::is_floating_point<T>::value) return static_cast<T>(fmin(static_cast<double>(a), static_cast<double>(b)));
  else return a < b ? a : b;
}
template <typename T>
__device__ __forceinline__ T max_of(T a, T b) {
  if constexpr (std::is_floating_point<T>::value) return static_cast<T>(fmax(static_cast<double>(a), static_cast<double>(b)));
  else return a > b ? a : b;
}

template <typename T>
__device__ __forceinline__ void partial_merge(Partial<T>& a, const Partial<T>& b) {
  if constexpr (!std::is_floating_point<T>::value) {
    const unsigned long long old = static_cast<unsigned long long>(a.sum);
    a.hi += b.hi + ((old + static_cast<unsigned long long>(b.sum)) < old ? 1 : 0);
  }
  a.sum += b.sum;
  a.count += b.count;
  a.mn = min_of(a.mn, b.mn);
  a.mx = max_of(a.mx, b.mx);
}

template <typename T>
__device__ __forceinline__ Partial<T> partial_shfl_down(const Partial<T>& p, int delta) {
  Partial<T> o;
  o.sum = __shfl_down_sync(0xffffffffu, p.sum, delta);
  o.hi = __shfl_down_sync(0xffffffffu, p.hi, delta);
  o.count = __shfl_down_sync(0xffffffffu, p.count, delta);
  o.mn = __shfl_down_sync(0xffffffffu, p.mn, delta);
  o.mx = __shfl_down_sync(0xffffffffu, p.mx, delta);
  return o;
}

// block tree reduction in a fixed order; result valid in thread 0
template <typename T>
__device__ __forceinline__ Partial<T> block_reduce(Partial<T> p) {
  __shared__ Partial<T> s_w[kBlock / 32];
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    Partial<T> o = partial_shfl_down(p, d);
    partial_merge(p, o);
  }
  if (lane_id() == 0) s_w[threadIdx.x >> 5] = p;
  __syncthreads();
  if (threadIdx.x < 32) {
    Partial<T> q;
    partial_init(q);
    if (threadIdx.x < kBlock / 32) q = s_w[threadIdx.x];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      Partial<T> o = partial_shfl_down(q, d);
      partial_merge(q, o);
    }
    p = q;
  }
  return p;
}

// Per-thread accumulator of the streaming loop.  In a straightforward version the exact 128-bit sum (carry and sign tests
// per element), per-load bounds tests and 64-bit index arithmetic are the cost, not the bytes.  So:
//   * 64-bit integers accumulate their low and high 32-bit halves in two 64-bit counters (no carry logic; a thread sees
//     < 2^20 elements, so neither can overflow) and the 128-bit value is assembled once per thread;
//   * narrower integers cannot overflow a 64-bit accumulator at all (< 2^32 rows x 2^32);
//   * the main loop covers only steps that lie entirely inside the column (no guards), the few remaining steps take
//     the guarded path.
template <typename T>
struct LocalAcc {
  using Acc = typename AccOf<T>::type;
  static constexpr bool kSplit = std::is_integral<T>::value && sizeof(T) == 8;
  Acc sum;                 // !kSplit: the sum; kSplit: sum of the low halves (as unsigned)
  Acc hi;                  // kSplit: sum of the (sign-extended) high halves
  long long count;
  T mn, mx;
  __device__ __forceinline__ void init() {
    sum = 0;
    hi = 0;
    count = 0;
    if (std::is_floating_point<T>::value) {
      mn = mx = static_cast<T>(nan(""));
    } else {
      mn = std::numeric_limits<T>::max();
      mx = std::numeric_limits<T>::lowest();
    }
  }
  // branch-free: a null slot adds 0 and leaves min / max alone (a divergent branch per element cost more than the
  // arithmetic it skipped); the caller counts
  __device__ __forceinline__ void add(T v, bool ok) {
    const T x = ok ? v : T(0);
    if constexpr (kSplit) {
      sum += static_cast<Acc>(static_cast<uint32_t>(static_cast<unsigned long long>(x)));
      hi += static_cast<Acc>(x >> 32);  // arithmetic shift for signed T
    } else {
      sum += static_cast<Acc>(x);
    }
    mn = ok ? min_of(mn, v) : mn;
    mx = ok ? max_of(mx, v) : mx;
  }
  __device__ __forceinline__ Partial<T> partial() const {
    Partial<T> p;
    p.count = count;
    p.mn = mn;
    p.mx = mx;
    if constexpr (kSplit) {
      // value = hi * 2^32 + sum, as a 128-bit two's complement number {p.hi, p.sum}
      const unsigned long long lo = static_cast<unsigned long long>(sum);
      const unsigned long long shifted = static_cast<unsigned long long>(hi) << 32;
      const unsigned long long low = lo + shifted;
      p.sum = static_cast<Acc>(low);
      p.hi = static_cast<long long>(hi >> 32) + (low < lo ? 1 : 0);  // hi >> 32: arithmetic for signed, logical for unsigned
    } else if constexpr (std::is_floating_point<T>::value) {
      p.sum = sum;
      p.hi = 0;
    } else {
      p.sum = sum;
      p.hi = (std::is_signed<T>::value && sum < 0) ? -1 : 0;  // sign extension of an exact 64-bit sum
    }
    return p;
  }
};

// VEC: every lane loads 16 bytes (E = 16 / sizeof(T) consecutive rows), so a warp covers 32 * E rows
// per step and needs E validity bits per lane; four steps are in flight.  The scalar variant (one row
// per lane per step) serves columns whose first value is not 16-byte aligned.
template <typename T, bool VEC>
__global__ void __launch_bounds__(kBlock, 4) reduce_kernel(const T* __restrict__ values, BitmapReader valid, int64_t n,
                                                        Partial<T>* __restrict__ partials) {
  LocalAcc<T> acc;
  acc.init();
  const unsigned lane = lane_id();
  const int64_t warp0 = (blockIdx.x * (int64_t)kBlock + threadIdx.x) >> 5;
  const int64_t warps = ((int64_t)gridDim.x * kBlock) >> 5;
  if (VEC) {
    constexpr int E = 16 / sizeof(T);
    constexpr int kRows = 32 * E;  // rows per warp step: 64 .. 512 = 1 .. 8 validity words
    constexpr int kU = 4;
    constexpr int W = E / 2;  // 64-bit validity words per step
    constexpr unsigned kFull = E == 32 ? 0xffffffffu : ((1u << E) - 1u);
    const int64_t n_steps = (n + kRows - 1) / kRows;
    const int64_t n_full = n / kRows;  // steps that lie entirely inside the column
    const int wsrc = (lane * E) >> 6, wsh = (lane * E) & 63;  // this lane's word inside a step, bit inside the word
    const bool has_valid = valid.present();
    int64_t s0 = warp0;
    // ---- main loop: kU full steps per iteration, no guards ----
    const uint4* p = reinterpret_cast<const uint4*>(values + warp0 * kRows + lane * E);
    const int64_t stride_u = warps * (kRows / E);       // in uint4 units: the next step of this warp
    const int64_t stride_it = stride_u * kU;
    for (; s0 + (kU - 1) * warps < n_full; s0 += warps * kU, p += stride_it) {
      uint4 raw[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) raw[u] = __ldcs(p + u * stride_u);
      unsigned bits[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) bits[u] = kFull;
      // validity: the kU * W words of these steps are extracted ONCE, by lanes 0 .. kU*W-1, and handed
      // round with shuffles (every lane redoing the unaligned-word extraction cost more than the sums)
      if (has_valid) {
        unsigned long long mine = 0;
        if (lane < kU * W) mine = valid.word((s0 + (lane / W) * warps) * W + (lane % W));
#pragma unroll
        for (int u = 0; u < kU; ++u) {
          const unsigned long long w = __shfl_sync(0xffffffffu, mine, u * W + wsrc);
          bits[u] = static_cast<unsigned>(w >> wsh) & kFull;
        }
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const T* v = reinterpret_cast<const T*>(&raw[u]);
#pragma unroll
        for (int e = 0; e < E; ++e) acc.add(v[e], ((bits[u] >> e) & 1u) != 0);
        acc.count += __popc(bits[u]);
      }
    }
    // ---- the remaining (at most kU) steps of this warp, the last of which may be partial ----
    for (int64_t step = s0; step < n_steps; step += warps) {
      const int64_t i0 = step * kRows + lane * E;
      unsigned bits = 0;
      uint4 raw = make_uint4(0, 0, 0, 0);
      if (i0 < n) {
        const int64_t rem = n - i0;
        if (rem >= E) {
          raw = __ldcs(reinterpret_cast<const uint4*>(values + i0));
          bits = kFull;
        } else {  // last, partial vector of the column
          T tmp[E];
#pragma unroll
          for (int e = 0; e < E; ++e) tmp[e] = e < rem ? values[i0 + e] : T(0);
          raw = *reinterpret_cast<const uint4*>(tmp);
          bits = (1u << rem) - 1u;
        }
      }
      if (has_valid) {
        unsigned long long mine = 0;
        if (lane < W) mine = valid.word(step * W + lane);
        const unsigned long long w = __shfl_sync(0xffffffffu, mine, wsrc);
        bits &= static_cast<unsigned>(w >> wsh);
      }
      const T* v = reinterpret_cast<const T*>(&raw);
#pragma unroll
      for (int e = 0; e < E; ++e) acc.add(v[e], ((bits >> e) & 1u) != 0);
      acc.count += __popc(bits);
    }
  } else {
    const int64_t n_groups = (n + 31) >> 5;
    constexpr int kU = 4;  // 32-row groups in flight per warp
    for (int64_t g0 = warp0; g0 < n_groups; g0 += warps * kU) {
      T v[kU];
      bool ok[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int64_t g = g0 + u * warps;
        const int64_t i = (g << 5) + lane;
        ok[u] = false;
        v[u] = T(0);
        if (g < n_groups && i < n) {
          ok[u] = valid.present() ? ((valid.word32(g) >> lane) & 1u) != 0 : true;
          if (ok[u]) v[u] = __ldcs(values + i);
        }
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        acc.add(v[u], ok[u]);
        acc.count += ok[u] ? 1 : 0;
      }
    }
  }
  Partial<T> part = block_reduce(acc.partial());
  if (threadIdx.x == 0) partials[blockIdx.x] = part;
}

template <typename T>
__device__ __forceinline__ unsigned long long widen_bits(T v) {
  if constexpr (std::is_floating_point<T>::value) return static_cast<unsigned long long>(__double_as_longlong(static_cast<double>(v)));
  else if constexpr (std::is_signed<T>::value) return static_cast<unsigned long long>(static_cast<long long>(v));
  else return static_cast<unsigned long long>(v);
}

// single CTA: fold the block partials (fixed order) and publish {count, sum, min, max, double sum}
template <typename T>
__global__ void __launch_bounds__(kBlock) reduce_final_kernel(const Partial<T>* __restrict__ partials, int n_partials,
                                                              unsigned long long* out) {
  Partial<T> p;
  partial_init(p);
  for (int i = threadIdx.x; i < n_partials; i += kBlock) partial_merge(p, partials[i]);
  p = block_reduce(p);
  if (threadIdx.x == 0) {
    out[0] = static_cast<unsigned long long>(p.count);
    if constexpr (std::is_floating_point<T>::value) out[1] = static_cast<unsigned long long>(__double_as_longlong(p.sum));
    else out[1] = static_cast<unsigned long long>(p.sum);
    out[2] = widen_bits(p.mn);
    out[3] = widen_bits(p.mx);
    // the sum as a double (what MeanImpl divides): floats = the sum itself, integers = the exact 128-bit value rounded once
    double ds;
    if constexpr (std::is_floating_point<T>::value) ds = p.sum;
    else {
      // sign-magnitude first: hi * 2^64 + lo would cancel catastrophically for small negative sums
      unsigned long long lo = static_cast<unsigned long long>(p.sum);
      long long hi = p.hi;
      const bool neg = hi < 0;
      if (neg) {  // two's complement negate of the 128-bit value
        lo = ~lo + 1ull;
        hi = ~hi + (lo == 0 ? 1 : 0);
      }
      ds = ldexp(static_cast<double>(hi), 64) + static_cast<double>(lo);
      if (neg) ds = -ds;
    }
    out[4] = static_cast<unsigned long long>(__double_as_longlong(ds));
  }
}

template <typename T>
static int reduce_typed(B2Context* ctx, const B2Array* values, B2ReduceResult* out, cudaStream_t s) {
  const int64_t n = values->length;
  const T* v = static_cast<const T*>(values->data) + values->offset;
  BitmapReader valid(values->null_count == 0 ? nullptr : values->validity, values->offset, n);
  const int grid = grid_for(n, kBlock * 8, ctx->sm_count * 8);
  Temp partials(ctx, s);
  B2_RETURN_NOT_OK(partials.alloc(sizeof(Partial<T>) * (size_t)grid));
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  if (aligned_to(v, 16)) reduce_kernel<T, true><<<grid, kBlock, 0, s>>>(v, valid, n, partials.as<Partial<T>>());
  else reduce_kernel<T, false><<<grid, kBlock, 0, s>>>(v, valid, n, partials.as<Partial<T>>());
  B2_LAUNCHED();
  reduce_final_kernel<T><<<1, kBlock, 0, s>>>(partials.as<Partial<T>>(), grid, reinterpret_cast<unsigned long long*>(slot.dev()));
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(slot.fetch(s));
  out->count = slot.host()[0];
  out->null_count = n - out->count;
  out->sum_bits = static_cast<uint64_t>(slot.host()[1]);
  out->min_bits = static_cast<uint64_t>(slot.host()[2]);
  out->max_bits = static_cast<uint64_t>(slot.host()[3]);
  out->dsum_bits = static_cast<uint64_t>(slot.host()[4]);
  out->value_type = values->type;
  out->acc_type = sum_type_of(values->type);
  return B2_OK;
}

}  // namespace b2

using namespace b2;

extern "C" int b2_reduce(B2Context* ctx, const B2Array* values, B2ReduceResult* out, void* stream) {
  if (!ctx || !values || !out) return set_error(B2_INVALID, "b2_reduce: null argument");
  if (!type_is_numeric(values->type)) return set_error(B2_NOT_IMPLEMENTED, "sum/mean/min_max over type id %d", values->type);
  if (values->length < 0 || values->offset < 0) return set_error(B2_INVALID, "negative length/offset");
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->pick(stream);
  return visit_type(NumericTypes{}, values->type, [&](auto tag) { return reduce_typed<decltype(tag)>(ctx, values, out, s); });
}
