// hash_moments.cu -- variance / stddev / skew / kurtosis per group, and over one group without ids.
//
// Replaces
//   GroupedStatisticImpl (hash_variance / hash_stddev / hash_skew / hash_kurtosis)
//                                      kernels/hash_aggregate_numeric.cc:452-842
//   VarianceImpl / MomentsState (variance / stddev / skew / kurtosis)
//                                      kernels/aggregate_var_std.cc:40-235
//   IntegerVarStd, Moments             kernels/aggregate_var_std_internal.h:33-152
// Semantics kept: output float64; a group is null when count <= ddof, count < min_count, unbiased skew with count < 3,
// unbiased kurtosis with count < 4, or (skip_nulls = false) it saw a null; null slots hold 0.  The algorithm split is the
// reference's, chosen by value type and level only:
//
//   EXACT     int8..uint32 at level 2 (variance / stddev).  Per group the count, Sx and Sx^2 are kept exactly as
//             128-bit integers (two 64-bit limbs, the high limb bumped by the atomic that carried out of the low one), so
//             the state is exact for any number of rows, consumes and merges, and independent of atomic order.
//             Finalize forms N = n*Sx^2 - (Sx)^2 and D = n*(n - ddof) in 256-bit integers and rounds N/D to double once
//             (to nearest, ties to even); stddev = sqrt of that double.  The reference rounds twice (IntegerVarStd::m2
//             then / (n - ddof)), so this is at least as accurate, and bit-reproducible.
//   TWO-PASS  every other type and level.  Per consume call, pass 1 takes the batch count and sum per group (floats in
//             double; integers exactly in 128 bits, rounded to double once), pass 2 sums (x - mean_g)^k for k = 2..level in
//             double, and each group's batch moments are folded into the running state with Moments::Merge (Neumaier
//             sums, math_internal.h:44-60).  A merge of two states uses the same formula; it relies on the group id
//             mapping being injective and fails with B2_INVALID if a destination repeats.
//
// Regimes per pass, as the other aggregators (hash_aggregate.cu): <= 2048 groups keep a private copy of the pass's
// planes per CTA in shared memory; otherwise one global atomic per plane, and large batches whose planes outgrow
// B2_HASHAGG_BAND_MB go in bands of group ids.  Without ids (one group) every CTA reduces its rows in registers and a
// fixed tree into one slot, and a single thread folds the slots in order: no float atomics, so the ungrouped result is
// bitwise identical from run to run for a given input and batch split.
#include <cmath>
#include <type_traits>

#include "bitmap.h"
#include "hash_moments.h"
#include "hash_table.cuh"

namespace b2 {
namespace {

typedef unsigned long long u64;
typedef unsigned __int128 u128;

enum Pass { PASS_EXACT = 0, PASS_SUM = 1, PASS_MOM = 2 };

// State planes (5 x cap words).  EXACT: count, Sx lo, Sx hi, Sx^2 lo, Sx^2 hi.  TWO-PASS: count, mean, m2, m3, m4.
// Batch planes of a two-pass consume (7 x G words): count, sum lo (or the double sum), sum hi, mean, m2, m3, m4.
constexpr int kStatePlanes = 5, kBatchPlanes = 7, kBatchMean = 3, kBatchMom = 4;
constexpr int kMomentPrivateGroups = 2048;

template <typename T>
constexpr bool kNarrowInt = std::is_integral<T>::value && sizeof(T) <= 4;

__device__ __forceinline__ double as_f64(u64 b) { return __longlong_as_double(static_cast<long long>(b)); }
__device__ __forceinline__ u64 f64_bits(double d) { return static_cast<u64>(__double_as_longlong(d)); }

// word adds, atomic (shared or global memory) or plain (registers, one thread)
template <bool ATOMIC>
__device__ __forceinline__ void add_u64(u64* p, u64 v) {
  if (ATOMIC) atomicAdd(p, v);
  else *p += v;
}
template <bool ATOMIC>
__device__ __forceinline__ void add_f64(u64* p, double v) {
  if (ATOMIC) atomicAdd(reinterpret_cast<double*>(p), v);
  else *p = f64_bits(as_f64(*p) + v);
}
// (hi:lo) += (a_hi:a_lo) modulo 2^128: whoever carries out of the low limb adds the carry to the high one
template <bool ATOMIC>
__device__ __forceinline__ void add_i128(u64* lo, u64* hi, u64 a_lo, u64 a_hi) {
  if (ATOMIC) {
    const u64 old = atomicAdd(lo, a_lo);
    const u64 d = a_hi + ((old + a_lo) < old ? 1ull : 0ull);
    if (d) atomicAdd(hi, d);
  } else {
    const u64 old = *lo;
    *lo = old + a_lo;
    *hi += a_hi + (*lo < old ? 1ull : 0ull);
  }
}

template <typename T>
__device__ __forceinline__ u64 sign_word(T x) {
  if constexpr (std::is_signed<T>::value) return x < 0 ? ~0ull : 0ull;
  else return 0ull;
}

template <typename T, int PASS>
__host__ __device__ constexpr int planes_of(int level) {
  return PASS == PASS_EXACT ? 5 : PASS == PASS_SUM ? (std::is_floating_point<T>::value ? 2 : 3) : level - 1;
}

// one valid row into the pass's planes at w[k * stride]
template <typename T, int PASS, bool ATOMIC>
__device__ __forceinline__ void add_row(u64* w, int64_t stride, T x, double mean, int level) {
  if constexpr (PASS == PASS_EXACT) {
    const long long xs = static_cast<long long>(x);
    add_u64<ATOMIC>(w, 1ull);
    add_i128<ATOMIC>(w + stride, w + 2 * stride, static_cast<u64>(xs), sign_word(x));
    // |x| <= 2^32 - 1: x^2 fits 64 bits unsigned
    add_i128<ATOMIC>(w + 3 * stride, w + 4 * stride, static_cast<u64>(xs) * static_cast<u64>(xs), 0ull);
  } else if constexpr (PASS == PASS_SUM) {
    add_u64<ATOMIC>(w, 1ull);
    if constexpr (std::is_floating_point<T>::value) add_f64<ATOMIC>(w + stride, static_cast<double>(x));
    else add_i128<ATOMIC>(w + stride, w + 2 * stride, static_cast<u64>(x), sign_word(x));
  } else {
    // the reference's (v - mean)^k terms: d2, d2 * d, d2 * d2 (hash_aggregate_numeric.cc:587-602)
    const double d = static_cast<double>(x) - mean, d2 = d * d;
    add_f64<ATOMIC>(w, d2);
    if (level >= 3) add_f64<ATOMIC>(w + stride, d2 * d);
    if (level >= 4) add_f64<ATOMIC>(w + 2 * stride, d2 * d2);
  }
}

// dst planes += src planes
template <typename T, int PASS, bool ATOMIC>
__device__ __forceinline__ void add_planes(u64* dst, int64_t ds, const u64* src, int64_t ss, int level) {
  if constexpr (PASS == PASS_EXACT) {
    add_u64<ATOMIC>(dst, src[0]);
    add_i128<ATOMIC>(dst + ds, dst + 2 * ds, src[ss], src[2 * ss]);
    add_i128<ATOMIC>(dst + 3 * ds, dst + 4 * ds, src[3 * ss], src[4 * ss]);
  } else if constexpr (PASS == PASS_SUM) {
    add_u64<ATOMIC>(dst, src[0]);
    if constexpr (std::is_floating_point<T>::value) add_f64<ATOMIC>(dst + ds, as_f64(src[ss]));
    else add_i128<ATOMIC>(dst + ds, dst + 2 * ds, src[ss], src[2 * ss]);
  } else {
    for (int k = 0; k < level - 1; ++k) add_f64<ATOMIC>(dst + k * ds, as_f64(src[k * ss]));
  }
}

// ---- grouped: one atomic per plane and row, ids outside [g_lo, g_hi) belong to another band ----
template <typename T, int PASS>
__global__ void __launch_bounds__(kBlock) moments_rows_kernel(const T* __restrict__ values, BitmapReader valid,
                                                              const uint32_t* __restrict__ ids, int64_t n, u64* dst,
                                                              int64_t stride, const double* __restrict__ means,
                                                              uint8_t* flags, int level, uint32_t g_lo, uint32_t g_hi) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const uint32_t g = __ldcs(ids + i);
    if (g < g_lo || g >= g_hi) continue;
    if (!valid.bit(i)) {
      if (flags) flags[g] |= 1;  // benign race: only ever sets bit 0
      continue;
    }
    add_row<T, PASS, true>(dst + g, stride, __ldcs(values + i), PASS == PASS_MOM ? means[g] : 0.0, level);
  }
}

// ---- grouped, few groups: a private copy of the planes per CTA in shared memory, added to dst once ----
template <typename T, int PASS>
__global__ void __launch_bounds__(kBlock) moments_rows_private_kernel(const T* __restrict__ values, BitmapReader valid,
                                                                      const uint32_t* __restrict__ ids, int64_t n, u64* dst,
                                                                      int64_t stride, const double* __restrict__ means,
                                                                      uint8_t* flags, int level, int num_groups) {
  extern __shared__ u64 s_w[];  // planes_of<T, PASS>(level) x num_groups
  const int np = planes_of<T, PASS>(level);
  for (int i = threadIdx.x; i < np * num_groups; i += kBlock) s_w[i] = 0ull;
  __syncthreads();
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const uint32_t g = __ldcs(ids + i);
    if (!valid.bit(i)) {
      if (flags) flags[g] |= 1;
      continue;
    }
    add_row<T, PASS, true>(s_w + g, num_groups, __ldcs(values + i), PASS == PASS_MOM ? means[g] : 0.0, level);
  }
  __syncthreads();
  for (int g = threadIdx.x; g < num_groups; g += kBlock)
    if (s_w[g] != 0ull) add_planes<T, PASS, true>(dst + g, stride, s_w + g, num_groups, level);
}

// ---- one group, no ids: registers, then a fixed tree per CTA into slots[k * gridDim.x + blockIdx.x] ----
template <typename T, int PASS>
__global__ void __launch_bounds__(kBlock) moments_rows_single_kernel(const T* __restrict__ values, BitmapReader valid, int64_t n,
                                                                     u64* slots, const double* __restrict__ mean_p,
                                                                     uint8_t* flags, int level) {
  __shared__ u64 s_w[kStatePlanes * kBlock];
  u64 acc[kStatePlanes] = {0ull, 0ull, 0ull, 0ull, 0ull};
  const double mean = PASS == PASS_MOM ? *mean_p : 0.0;
  bool saw_null = false;
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    if (!valid.bit(i)) {
      saw_null = true;
      continue;
    }
    add_row<T, PASS, false>(acc, 1, __ldcs(values + i), mean, level);
  }
  if (__syncthreads_or(saw_null) && flags && threadIdx.x == 0) flags[0] |= 1;
#pragma unroll
  for (int k = 0; k < kStatePlanes; ++k) s_w[k * kBlock + threadIdx.x] = acc[k];
  __syncthreads();
  for (int h = kBlock / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) add_planes<T, PASS, false>(s_w + threadIdx.x, kBlock, s_w + threadIdx.x + h, kBlock, level);
    __syncthreads();
  }
  if (threadIdx.x == 0)
    for (int k = 0; k < kStatePlanes; ++k) slots[k * gridDim.x + blockIdx.x] = s_w[k * kBlock];
}

// one thread adds the slots into group 0 of dst in slot order
template <typename T, int PASS>
__global__ void moments_fold_kernel(const u64* slots, int nslots, u64* dst, int64_t stride, int level) {
  for (int b = 0; b < nslots; ++b) add_planes<T, PASS, false>(dst, stride, slots + b, nslots, level);
}

// the two's-complement 128-bit (hi:lo) as the nearest double, one rounding: the top 64 significant bits of |v| with every
// lower bit folded into bit 0 (a sticky bit far below the 53-bit rounding point) round exactly as |v| itself would
__device__ __forceinline__ double i128_to_double(u64 lo, u64 hi) {
  const bool neg = hi >> 63;
  u128 v = ((u128)hi << 64) | lo;
  if (neg) v = (u128)0 - v;
  const u64 vh = (u64)(v >> 64);
  double r;
  if (vh == 0) {
    r = static_cast<double>((u64)v);
  } else {
    const int lz = __clzll((long long)vh);
    const u128 top = v << lz;  // the leading one at bit 127
    const u64 m = (u64)(top >> 64) | ((u64)top != 0 ? 1ull : 0ull);
    r = ldexp(static_cast<double>(m), 64 - lz);
  }
  return neg ? -r : r;
}

// batch mean per group: sum / count (plane 3); integer sums are exact until this one conversion
__global__ void __launch_bounds__(kBlock) moments_means_kernel(u64* batch, int64_t g_n, int int_sum) {
  for (int64_t g = blockIdx.x * (int64_t)kBlock + threadIdx.x; g < g_n; g += (int64_t)gridDim.x * kBlock) {
    const u64 c = batch[g];
    const double sum = int_sum ? i128_to_double(batch[g_n + g], batch[2 * g_n + g]) : as_f64(batch[g_n + g]);
    batch[kBatchMean * g_n + g] = f64_bits(c ? sum / static_cast<double>(c) : 0.0);
  }
}

struct Mom {
  u64 n;
  double mean, m2, m3, m4;
};

__device__ __forceinline__ double neumaier(const double* v, int k) {
  double sum = 0, c = 0;
  for (int i = 0; i < k; ++i) {
    const double t = sum + v[i];
    if (isfinite(t)) c += fabs(sum) >= fabs(v[i]) ? (sum - t) + v[i] : (v[i] - t) + sum;
    sum = t;
  }
  return sum + c;
}

// Moments::Merge (aggregate_var_std_internal.h:116-152); the count products are formed in double, where the reference's
// int64 n * n * n overflows beyond 2^21 rows
__device__ Mom merge_moments(int level, const Mom& a, const Mom& b) {
  if (a.n == 0) return b;
  if (b.n == 0) return a;
  const double na = static_cast<double>(a.n), nb = static_cast<double>(b.n);
  const u64 nn = a.n + b.n;
  const double n = static_cast<double>(nn);
  Mom r{nn, (a.mean * na + b.mean * nb) / n, 0, 0, 0};
  double t[5] = {a.m2, b.m2, na * (a.mean - r.mean) * (a.mean - r.mean), nb * (b.mean - r.mean) * (b.mean - r.mean)};
  r.m2 = neumaier(t, 4);
  if (level >= 3) {
    const double delta = b.mean - a.mean, delta2 = delta * delta;
    t[0] = a.m3;
    t[1] = b.m3;
    t[2] = delta2 * delta * na * nb * (na - nb) / (n * n);
    t[3] = 3 * delta * (na * b.m2 - nb * a.m2) / n;
    r.m3 = neumaier(t, 4);
    if (level >= 4) {
      t[0] = a.m4;
      t[1] = b.m4;
      t[2] = (delta2 * delta2) * na * nb * (na * na - na * nb + nb * nb) / (n * n * n);
      t[3] = 6 * delta2 * (na * na * b.m2 + nb * nb * a.m2) / (n * n);
      t[4] = 4 * delta * (na * b.m3 - nb * a.m3) / n;
      r.m4 = neumaier(t, 5);
    }
  }
  return r;
}

__device__ __forceinline__ Mom load_state(const u64* st, int64_t cap, int64_t g) {
  return Mom{st[g], as_f64(st[cap + g]), as_f64(st[2 * cap + g]), as_f64(st[3 * cap + g]), as_f64(st[4 * cap + g])};
}
__device__ __forceinline__ void store_state(u64* st, int64_t cap, int64_t g, const Mom& m) {
  st[g] = m.n;
  st[cap + g] = f64_bits(m.mean);
  st[2 * cap + g] = f64_bits(m.m2);
  st[3 * cap + g] = f64_bits(m.m3);
  st[4 * cap + g] = f64_bits(m.m4);
}

// state[g] = Merge(state[g], batch[g])
__global__ void __launch_bounds__(kBlock) moments_merge_batch_kernel(u64* st, int64_t cap, const u64* batch, int64_t g_n, int level) {
  for (int64_t g = blockIdx.x * (int64_t)kBlock + threadIdx.x; g < g_n; g += (int64_t)gridDim.x * kBlock) {
    const Mom b{batch[g], as_f64(batch[kBatchMean * g_n + g]), as_f64(batch[kBatchMom * g_n + g]),
                as_f64(batch[(kBatchMom + 1) * g_n + g]), as_f64(batch[(kBatchMom + 2) * g_n + g])};
    if (b.n == 0) continue;
    store_state(st, cap, g, merge_moments(level, load_state(st, cap, g), b));
  }
}

// validate the mapping before any state changes: bad[0] = an entry >= num_groups; bad[1] = a repeated destination, which a
// two-pass merge (a read-modify-write per group) would race on -- counted only when claims is given
__global__ void __launch_bounds__(kBlock) moments_check_map_kernel(const uint32_t* map, int64_t n, int64_t num_groups,
                                                                   uint32_t* claims, int64_t* bad) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const uint32_t g = map[i];
    if (static_cast<int64_t>(g) >= num_groups) bad[0] = 1;
    else if (claims && atomicAdd(&claims[g], 1u) != 0u) bad[1] = 1;
  }
}

__global__ void __launch_bounds__(kBlock) moments_merge_state_kernel(u64* dst, int64_t dcap, uint8_t* dflags, const u64* src,
                                                                     int64_t scap, const uint8_t* sflags, const uint32_t* map,
                                                                     int64_t n, int exact, int level) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const uint32_t g = map[i];
    if (sflags[i] & 1) dflags[g] |= 1;
    if (exact) add_planes<int32_t, PASS_EXACT, true>(dst + g, dcap, src + i, scap, level);
    else store_state(dst, dcap, g, merge_moments(level, load_state(dst, dcap, g), load_state(src, scap, i)));
  }
}

// ---- exact finalize: round(N / D) with N < 2^192, D < 2^128 ----
struct U256 {
  u64 w[4];
};

__device__ __forceinline__ U256 mul_u128(u128 a, u128 b) {
  const u64 a0 = (u64)a, a1 = (u64)(a >> 64), b0 = (u64)b, b1 = (u64)(b >> 64);
  const u128 p00 = (u128)a0 * b0, p01 = (u128)a0 * b1, p10 = (u128)a1 * b0, p11 = (u128)a1 * b1;
  U256 r;
  r.w[0] = (u64)p00;
  u128 c = (p00 >> 64) + (u64)p01 + (u64)p10;
  r.w[1] = (u64)c;
  c = (c >> 64) + (p01 >> 64) + (p10 >> 64) + (u64)p11;
  r.w[2] = (u64)c;
  r.w[3] = (u64)((c >> 64) + (p11 >> 64));
  return r;
}
__device__ __forceinline__ bool u256_ge(const U256& a, const U256& b) {
  for (int i = 3; i >= 0; --i)
    if (a.w[i] != b.w[i]) return a.w[i] > b.w[i];
  return true;
}
__device__ __forceinline__ U256 u256_sub(const U256& a, const U256& b) {
  U256 r;
  u64 borrow = 0;
  for (int i = 0; i < 4; ++i) {
    const u64 d = a.w[i] - b.w[i];
    r.w[i] = d - borrow;
    borrow = (a.w[i] < b.w[i]) || (d < borrow) ? 1ull : 0ull;
  }
  return r;
}
__device__ __forceinline__ int u256_bits(const U256& a) {
  for (int i = 3; i >= 0; --i)
    if (a.w[i]) return 64 * i + 64 - __clzll((long long)a.w[i]);
  return 0;
}
__device__ __forceinline__ U256 u256_shl(const U256& a, int k) {
  U256 r = {{0, 0, 0, 0}};
  const int q = k >> 6, s = k & 63;
  for (int i = 3; i >= q; --i) {
    u64 v = a.w[i - q] << s;
    if (s && i - q - 1 >= 0) v |= a.w[i - q - 1] >> (64 - s);
    r.w[i] = v;
  }
  return r;
}
__device__ __forceinline__ U256 u256_shr1(const U256& a) {
  U256 r;
  for (int i = 0; i < 3; ++i) r.w[i] = (a.w[i] >> 1) | (a.w[i + 1] << 63);
  r.w[3] = a.w[3] >> 1;
  return r;
}

// N / D rounded to the nearest double, ties to even (D > 0)
__device__ double div_round(const U256& num, const U256& den) {
  const int nb = u256_bits(num);
  if (nb == 0) return 0.0;
  const int k = 56 - (nb - u256_bits(den));  // quotient of A / B below has 56..57 bits
  U256 a = k >= 0 ? u256_shl(num, k) : num;
  U256 bs = u256_shl(k >= 0 ? den : u256_shl(den, -k), 57);
  u64 q = 0;
  for (int i = 57; i >= 0; --i) {
    if (u256_ge(a, bs)) {
      a = u256_sub(a, bs);
      q |= 1ull << i;
    }
    bs = u256_shr1(bs);
  }
  const bool sticky = (a.w[0] | a.w[1] | a.w[2] | a.w[3]) != 0;
  const int drop = 64 - __clzll((long long)q) - 53;
  u64 mant = q >> drop;
  const u64 rem = q & ((1ull << drop) - 1), half = 1ull << (drop - 1);
  if (rem > half || (rem == half && (sticky || (mant & 1)))) ++mant;
  return ldexp(static_cast<double>(mant), drop - k);
}

__global__ void __launch_bounds__(kBlock) moments_finalize_kernel(const u64* st, int64_t cap, const uint8_t* flags, int64_t g_n,
                                                                  int kind, int exact, int param, int skip_nulls, uint32_t min_count,
                                                                  double* out, uint32_t* out_validity, int64_t* valid_count) {
  const int64_t nw = (g_n + 31) >> 5;
  int64_t local = 0;
  const bool unbiased = (kind == B2_HASH_SKEW || kind == B2_HASH_KURTOSIS) && param != 0;
  const u64 ddof = (kind == B2_HASH_VARIANCE || kind == B2_HASH_STDDEV) ? static_cast<u64>(param) : 0ull;
  for (int64_t w = (blockIdx.x * (int64_t)kBlock + threadIdx.x) >> 5; w < nw; w += ((int64_t)gridDim.x * kBlock) >> 5) {
    const int64_t g = (w << 5) + lane_id();
    bool valid = false;
    if (g < g_n) {
      const u64 c = st[g];
      valid = c > ddof && c >= min_count && (skip_nulls || !(flags[g] & 1)) &&
              !(unbiased && kind == B2_HASH_SKEW && c < 3) && !(unbiased && kind == B2_HASH_KURTOSIS && c < 4);
      double r = 0.0;
      if (valid && exact) {
        const u128 s1 = ((u128)st[2 * cap + g] << 64) | st[cap + g];
        const u128 s2 = ((u128)st[4 * cap + g] << 64) | st[3 * cap + g];
        const u128 abs_s1 = (s1 >> 127) ? (u128)0 - s1 : s1;  // |Sx| < 2^96
        const U256 num = u256_sub(mul_u128(c, s2), mul_u128(abs_s1, abs_s1));
        r = div_round(num, mul_u128(c, c - ddof));
        if (kind == B2_HASH_STDDEV) r = sqrt(r);
      } else if (valid) {
        // Moments::Variance / Stddev / Skew / Kurtosis (aggregate_var_std_internal.h:72-112)
        const Mom m = load_state(st, cap, g);
        const double n = static_cast<double>(c);
        if (kind == B2_HASH_VARIANCE || kind == B2_HASH_STDDEV) {
          r = m.m2 / static_cast<double>(c - ddof);
          if (kind == B2_HASH_STDDEV) r = sqrt(r);
        } else if (kind == B2_HASH_SKEW) {
          if (!unbiased) {
            r = sqrt(n) * m.m3 / sqrt(m.m2 * m.m2 * m.m2);
          } else {
            const double m2_avg = m.m2 / n;
            r = sqrt(n * (n - 1)) / (n - 2) * (m.m3 / n) / sqrt(m2_avg * m2_avg * m2_avg);
          }
        } else if (!unbiased) {
          r = n * m.m4 / (m.m2 * m.m2) - 3;
        } else {
          const double m2_avg = m.m2 / n;
          r = 1.0 / ((n - 2) * (n - 3)) * ((n * n - 1.0) * (m.m4 / n) / (m2_avg * m2_avg) - 3 * ((n - 1) * (n - 1)));
        }
      }
      out[g] = r;
    }
    const unsigned word = __ballot_sync(0xffffffffu, valid);
    if (lane_id() == 0) {
      out_validity[w] = word;
      local += __popc(word);
    }
  }
  const int64_t s = block_sum<kBlock>(local);
  if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(valid_count), (unsigned long long)s);
}

__global__ void __launch_bounds__(kBlock) moments_zero_kernel(u64* p, int64_t cap, int64_t from, int64_t to) {
  for (int64_t g = from + blockIdx.x * (int64_t)kBlock + threadIdx.x; g < to; g += (int64_t)gridDim.x * kBlock)
    for (int k = 0; k < kStatePlanes; ++k) p[k * cap + g] = 0ull;
}

}  // namespace

struct MomentAgg {
  B2Context* ctx;
  int kind;
  int value_type;
  int level;
  bool exact;
  B2HashAggOptions opt;
  u64* planes = nullptr;  // kStatePlanes x cap
  uint8_t* flags = nullptr;  // bit 0: the group saw a null
  int64_t num_groups = 0, cap = 0;
};

namespace {

// one pass over the rows into the planes dst[plane k of group g] = dst[k * stride + g]
template <typename T, int PASS>
int run_pass(MomentAgg* m, const T* v, BitmapReader valid, const uint32_t* id, int64_t n, u64* dst, int64_t stride,
             const double* means, uint8_t* flags, cudaStream_t s) {
  const int level = m->level;
  const int np = planes_of<T, PASS>(level);
  if (!id) {
    const int grid = grid_for(n, kBlock * 16, kSMs * 8);  // a function of n only: the fold order is fixed
    Temp slots(m->ctx, s);
    B2_RETURN_NOT_OK(slots.alloc((size_t)kStatePlanes * grid * 8));
    moments_rows_single_kernel<T, PASS><<<grid, kBlock, 0, s>>>(v, valid, n, slots.as<u64>(), means, flags, level);
    B2_LAUNCHED();
    moments_fold_kernel<T, PASS><<<1, 1, 0, s>>>(slots.as<u64>(), grid, dst, stride, level);
    B2_LAUNCHED();
    return B2_OK;
  }
  if (m->num_groups <= kMomentPrivateGroups && n >= (1 << 14)) {
    const int g = (int)m->num_groups;
    const size_t smem = (size_t)np * g * 8;
    if (smem > 48 * 1024)
      B2_CUDA(cudaFuncSetAttribute(moments_rows_private_kernel<T, PASS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int pgrid = grid_for(n, kBlock * 64, kSMs * 8);
    moments_rows_private_kernel<T, PASS><<<pgrid, kBlock, smem, s>>>(v, valid, id, n, dst, stride, means, flags, level, g);
    B2_LAUNCHED();
    return B2_OK;
  }
  // bytes of state a row can touch: the pass's planes, plus the mean pass 2 reads
  const int64_t per_group = 8 * (np + (PASS == PASS_MOM ? 1 : 0));
  const int64_t band_groups = hashagg_band_bytes() / per_group;
  int64_t bands = (m->num_groups + band_groups - 1) / band_groups;
  if (bands < 1 || n < (1 << 24)) bands = 1;
  const int64_t per_band = (m->num_groups + bands - 1) / bands;
  const int grid = grid_for(n, kBlock * 4, kSMs * 16);
  for (int64_t b = 0; b < bands; ++b) {
    const uint32_t lo = bands == 1 ? 0u : static_cast<uint32_t>(b * per_band);
    const uint32_t hi = (bands == 1 || b == bands - 1) ? 0xffffffffu : static_cast<uint32_t>((b + 1) * per_band);
    moments_rows_kernel<T, PASS><<<grid, kBlock, 0, s>>>(v, valid, id, n, dst, stride, means, flags, level, lo, hi);
    B2_LAUNCHED();
  }
  return B2_OK;
}

template <typename T>
int consume_typed(MomentAgg* m, const B2Array* values, const uint32_t* id, cudaStream_t s) {
  const int64_t n = values->length;
  const T* v = static_cast<const T*>(values->data) + values->offset;
  BitmapReader valid(values->null_count == 0 ? nullptr : values->validity, values->offset, n);
  if constexpr (kNarrowInt<T>) {
    if (m->exact) return run_pass<T, PASS_EXACT>(m, v, valid, id, n, m->planes, m->cap, nullptr, m->flags, s);
  }
  const int64_t g_n = m->num_groups;
  Temp batch(m->ctx, s);
  B2_RETURN_NOT_OK(batch.alloc((size_t)kBatchPlanes * g_n * 8));
  u64* b = batch.as<u64>();
  B2_CUDA(cudaMemsetAsync(b, 0, (size_t)kBatchPlanes * g_n * 8, s));
  B2_RETURN_NOT_OK((run_pass<T, PASS_SUM>(m, v, valid, id, n, b, g_n, nullptr, m->flags, s)));
  const int ggrid = grid_for(g_n, kBlock * 4, kSMs * 8);
  moments_means_kernel<<<ggrid, kBlock, 0, s>>>(b, g_n, std::is_integral<T>::value ? 1 : 0);
  B2_LAUNCHED();
  const double* means = reinterpret_cast<const double*>(b + kBatchMean * g_n);
  B2_RETURN_NOT_OK((run_pass<T, PASS_MOM>(m, v, valid, id, n, b + kBatchMom * g_n, g_n, means, nullptr, s)));
  moments_merge_batch_kernel<<<ggrid, kBlock, 0, s>>>(m->planes, m->cap, b, g_n, m->level);
  B2_LAUNCHED();
  return B2_OK;
}

}  // namespace

int moments_create(B2Context* ctx, int kind, int32_t value_type, const B2HashAggOptions& opt, MomentAgg** out) {
  if (!type_is_numeric(value_type)) return set_error(B2_NOT_IMPLEMENTED, "hash aggregate over value type id %d", value_type);
  if ((kind == B2_HASH_VARIANCE || kind == B2_HASH_STDDEV) && opt.stat_param < 0)
    return set_error(B2_INVALID, "ddof must be >= 0, got %d", opt.stat_param);
  MomentAgg* m = new MomentAgg();
  m->ctx = ctx;
  m->kind = kind;
  m->value_type = value_type;
  m->level = kind == B2_HASH_SKEW ? 3 : kind == B2_HASH_KURTOSIS ? 4 : 2;
  const bool narrow = value_type == B2_INT8 || value_type == B2_UINT8 || value_type == B2_INT16 || value_type == B2_UINT16 ||
                      value_type == B2_INT32 || value_type == B2_UINT32;
  m->exact = narrow && m->level == 2;
  m->opt = opt;
  *out = m;
  return B2_OK;
}

void moments_destroy(MomentAgg* m) {
  if (!m) return;
  cudaStream_t s = m->ctx->stream;
  if (m->planes) m->ctx->free(m->planes, s);
  if (m->flags) m->ctx->free(m->flags, s);
  delete m;
}

int moments_resize(MomentAgg* m, int64_t num_groups, cudaStream_t s) {
  B2Context* ctx = m->ctx;
  if (num_groups > m->cap) {
    const int64_t cap = static_cast<int64_t>(next_pow2(num_groups < 1024 ? 1024 : num_groups));
    void *p, *f;
    B2_RETURN_NOT_OK(ctx->alloc((size_t)kStatePlanes * cap * 8, &p, s));
    B2_RETURN_NOT_OK(ctx->alloc((size_t)cap, &f, s));
    for (int k = 0; k < kStatePlanes && m->num_groups; ++k)
      B2_CUDA(cudaMemcpyAsync(static_cast<u64*>(p) + k * cap, m->planes + k * m->cap, m->num_groups * 8, cudaMemcpyDeviceToDevice, s));
    if (m->num_groups) B2_CUDA(cudaMemcpyAsync(f, m->flags, m->num_groups, cudaMemcpyDeviceToDevice, s));
    if (m->planes) ctx->free(m->planes, s);
    if (m->flags) ctx->free(m->flags, s);
    m->planes = static_cast<u64*>(p);
    m->flags = static_cast<uint8_t*>(f);
    m->cap = cap;
  }
  const int64_t added = num_groups - m->num_groups;
  if (added > 0) {
    moments_zero_kernel<<<grid_for(added, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(m->planes, m->cap, m->num_groups, num_groups);
    B2_LAUNCHED();
    B2_CUDA(cudaMemsetAsync(m->flags + m->num_groups, 0, added, s));
  }
  m->num_groups = num_groups;
  return B2_OK;
}

int moments_consume(MomentAgg* m, const B2Array* values, const B2Array* ids, cudaStream_t s) {
  if (!values) return set_error(B2_INVALID, "hash aggregate needs a value column");
  if (ids && values->length != ids->length) return set_error(B2_INVALID, "values and group ids differ in length");
  if (!ids && m->num_groups != 1)
    return set_error(B2_INVALID, "group ids may be omitted only for a state with one group (it has %lld)", (long long)m->num_groups);
  if (values->type != m->value_type)
    return set_error(B2_TYPE_ERROR, "hash aggregate was created for type id %d, got %d", m->value_type, values->type);
  if (values->length == 0) return B2_OK;
  const uint32_t* id = ids ? static_cast<const uint32_t*>(ids->data) + ids->offset : nullptr;
  return visit_type(NumericTypes{}, values->type, [&](auto tag) { return consume_typed<decltype(tag)>(m, values, id, s); },
                    [&] { return set_error(B2_NOT_IMPLEMENTED, "hash aggregate over value type id %d", values->type); });
}

int moments_merge(MomentAgg* m, const MomentAgg* other, const B2Array* group_id_mapping, cudaStream_t s) {
  const int64_t n = other->num_groups;
  if (n == 0) return B2_OK;
  const uint32_t* map = static_cast<const uint32_t*>(group_id_mapping->data) + group_id_mapping->offset;
  const int grid = grid_for(n, kBlock * 4, kSMs * 8);
  {
    Temp claims(m->ctx, s);
    if (!m->exact) {
      B2_RETURN_NOT_OK(claims.alloc((size_t)m->num_groups * 4));
      B2_CUDA(cudaMemsetAsync(claims.ptr, 0, (size_t)m->num_groups * 4, s));
    }
    ScalarSlot slot(m->ctx);
    B2_RETURN_NOT_OK(slot.zero(s));
    moments_check_map_kernel<<<grid, kBlock, 0, s>>>(map, n, m->num_groups, claims.as<uint32_t>(), slot.dev());
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(slot.fetch(s));
    if (slot.host()[0]) return set_error(B2_INVALID, "group_id_mapping has an entry beyond the %lld groups of the state", (long long)m->num_groups);
    if (slot.host()[1]) return set_error(B2_INVALID, "group_id_mapping maps two groups to one (moments merge needs distinct ids)");
  }
  moments_merge_state_kernel<<<grid, kBlock, 0, s>>>(m->planes, m->cap, m->flags, other->planes, other->cap, other->flags, map, n,
                                                     m->exact ? 1 : 0, m->level);
  B2_LAUNCHED();
  return B2_OK;
}

int moments_finalize(MomentAgg* m, B2Array* out, cudaStream_t s) {
  const int64_t n = m->num_groups;
  Temp data(m->ctx, s), bits(m->ctx, s);
  B2_RETURN_NOT_OK(data.alloc((size_t)n * 8));
  int64_t nulls = 0;
  if (n > 0) {
    B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(n)));
    B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bitmap_alloc_bytes(n), s));
    ScalarSlot slot(m->ctx);
    B2_RETURN_NOT_OK(slot.zero(s));
    moments_finalize_kernel<<<grid_for(n, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(
        m->planes, m->cap, m->flags, n, m->kind, m->exact ? 1 : 0, m->opt.stat_param, m->opt.skip_nulls, m->opt.min_count,
        data.as<double>(), bits.as<uint32_t>(), slot.dev());
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(slot.fetch(s));
    nulls = n - slot.host()[0];
  }
  fill_out(out, B2_DOUBLE, n, nulls, nulls ? bits.release() : nullptr, data.release());
  return B2_OK;
}

}  // namespace b2
