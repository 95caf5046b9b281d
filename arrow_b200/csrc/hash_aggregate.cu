// hash_aggregate.cu -- grouped aggregators driven by uint32 group ids, plus the fused
// (key,value) -> table group-by used by the aggregate node.
//
// Replaces the HashAggregateKernel contract {init,resize,consume,merge,finalize}
// (cpp/src/arrow/compute/kernel.h:720-769) for
//   GroupedSumImpl / GroupedMeanImpl via GroupedReducingAggregator
//                                      kernels/hash_aggregate_numeric.cc:44-190,274-295,359-434
//   GroupedCountImpl / GroupedCountAllImpl      kernels/hash_aggregate.cc:61-272
//   GroupedMinMaxImpl (hash_min / hash_max)     kernels/hash_aggregate.cc:330-420
//   GroupedProductImpl (hash_product)           kernels/hash_aggregate_numeric.cc:311-335
//   GroupedAnyImpl / GroupedAllImpl             kernels/hash_aggregate.cc:1232-1397
//   GroupedStatisticImpl (variance / stddev / skew / kurtosis): hash_moments.cu, reached through the entry points below
//   VisitGroupedValues                          kernels/hash_aggregate_internal.h:148-171
// Semantics kept: integer sums accumulate in int64/uint64 with wrap-around (unsigned
// add), float sums and all means in double; count modes ONLY_VALID/ONLY_NULL/ALL;
// sum/mean are null where count < min_count, and (skip_nulls=false) where the group saw
// a null; min/max ignore NaN like std::fmin/fmax and are null for groups without values.
// Integer results are bit-exact; float sums differ from the reference only by summation
// order (the reference adds in row order, atomics do not) -- tests use a tolerance there.
//
// Design: one thread per row, coalesced id/value loads, three regimes by group count G
// (known from Resize):
//   G <= 2048        every CTA keeps a private copy of the state in shared memory and adds it
//                    to the global state once (same-address global atomics serialise);
//   state fits L2    one global atomic per state word;
//   state > L2       the batch is consumed in BANDS of group ids whose state stays
//                    L2-resident, re-streaming the ids once per band; otherwise every update
//                    is a 32-byte sector RMW in HBM.
// count / count_all additionally merge equal ids inside a warp (MATCH.ANY) before the atomic.
#include <cmath>
#include <cstdlib>
#include <limits>
#include <type_traits>

#include "bitmap.h"
#include "hash_moments.h"
#include "hash_table.cuh"

namespace b2 {

enum AccKind { ACC_I64 = 0, ACC_U64 = 1, ACC_F64 = 2 };

__host__ __device__ inline int acc_kind_for(int value_type) {
  switch (value_type) {
    case B2_INT8: case B2_INT16: case B2_INT32: case B2_INT64: return ACC_I64;
    case B2_UINT8: case B2_UINT16: case B2_UINT32: case B2_UINT64: return ACC_U64;
    default: return ACC_F64;
  }
}

template <typename T>
__device__ __forceinline__ T load_as(const void* p, int64_t i) {
  return static_cast<const T*>(p)[i];
}

// ordered encoding so min/max of any numeric type is an unsigned 64-bit atomicMin/Max
template <typename T>
__device__ __forceinline__ unsigned long long minmax_encode(T v) {
  if constexpr (std::is_floating_point<T>::value) {
    double d = static_cast<double>(v);
    unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(d));
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
  } else if constexpr (std::is_signed<T>::value) {
    return static_cast<unsigned long long>(static_cast<long long>(v)) ^ 0x8000000000000000ull;
  } else {
    return static_cast<unsigned long long>(v);
  }
}

struct AggState {
  unsigned long long* reduced;  // [G] sum bits / ordered min-max key
  unsigned long long* counts;   // [G]
  uint8_t* flags;               // [G] bit0 = saw a null, bit1 = has a value
};

// counts[g] += 1 for the lanes with inc: lanes of a warp holding the same group are merged first
// (MATCH.ANY, one atomic per distinct group per warp) so a hot group does not serialise on one address
__device__ __forceinline__ void count_merged(unsigned long long* counts, uint32_t g, bool inc) {
  const unsigned live = __ballot_sync(0xffffffffu, inc);
  if (inc) {
    const unsigned peers = __match_any_sync(live, g);
    if ((peers & lanemask_lt()) == 0) atomicAdd(&counts[g], static_cast<unsigned long long>(__popc(peers)));
  }
}

template <typename T, int KIND>
__global__ void __launch_bounds__(kBlock) hashagg_consume_kernel(const T* __restrict__ values,
                                                                 BitmapReader valid,
                                                                 const uint32_t* __restrict__ ids, int64_t n,
                                                                 AggState st, int count_mode, uint32_t g_lo,
                                                                 uint32_t g_hi) {
  if (KIND == B2_HASH_COUNT) {
    // a few hot groups would serialise their atomics on one L2 address: merge equal ids inside the warp first
    const unsigned lane = lane_id();
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t base = blockIdx.x * (int64_t)kBlock + (threadIdx.x & ~31u); base < n; base += stride) {
      const int64_t i = base + lane;
      bool inc = false;
      uint32_t g = 0;
      if (i < n) {
        g = __ldcs(ids + i);
        const bool ok = valid.bit(i);
        inc = g >= g_lo && g < g_hi && (count_mode == 2 || (count_mode == 0 ? ok : !ok));
      }
      count_merged(st.counts, g, inc);
    }
    return;
  }
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const uint32_t g = __ldcs(ids + i);
    if (g < g_lo || g >= g_hi) continue;  // another band's group (see launch_consume)
    const bool ok = valid.bit(i);
    if (!ok) {
      st.flags[g] |= 1;  // benign race: only ever sets bit 0 (byte store of an OR'd value)
      continue;
    }
    const T v = __ldcs(values + i);
    if (KIND == B2_HASH_SUM || KIND == B2_HASH_MEAN) {
      if (std::is_floating_point<T>::value || KIND == B2_HASH_MEAN) {
        atomicAdd(reinterpret_cast<double*>(&st.reduced[g]), static_cast<double>(v));
      } else if (std::is_signed<T>::value) {
        atomicAdd(&st.reduced[g], static_cast<unsigned long long>(static_cast<long long>(v)));
      } else {
        atomicAdd(&st.reduced[g], static_cast<unsigned long long>(v));
      }
      atomicAdd(&st.counts[g], 1ull);
    } else if (KIND == B2_HASH_PRODUCT) {
      // no hardware multiply-atomic: CAS loop.  Integers multiply mod 2^64 (MultiplyTraits, wrap-around as the
      // reference's to_unsigned product) so the result is order independent and bit-exact; floats in double.
      unsigned long long* p = &st.reduced[g];
      unsigned long long old = *reinterpret_cast<volatile unsigned long long*>(p), assumed;
      do {
        assumed = old;
        unsigned long long next;
        if (std::is_floating_point<T>::value) {
          next = static_cast<unsigned long long>(__double_as_longlong(__longlong_as_double((long long)assumed) * static_cast<double>(v)));
        } else if (std::is_signed<T>::value) {
          next = assumed * static_cast<unsigned long long>(static_cast<long long>(v));
        } else {
          next = assumed * static_cast<unsigned long long>(v);
        }
        old = atomicCAS(p, assumed, next);
      } while (old != assumed);
      atomicAdd(&st.counts[g], 1ull);
    } else {  // MIN / MAX
      if (v == v) {  // fmin/fmax skip NaN
        if (KIND == B2_HASH_MIN) atomicMin(&st.reduced[g], minmax_encode<T>(v));
        else atomicMax(&st.reduced[g], minmax_encode<T>(v));
      }
      atomicAdd(&st.counts[g], 1ull);
    }
  }
}

// hash_any / hash_all over a bit-packed boolean column (GroupedAnyImpl / GroupedAllImpl, hash_aggregate.cc:1232-1397):
// reduced[g] is 0/1; any = OR (starts 0), all = AND (starts 1); a null row only clears the group's no_nulls flag
__global__ void __launch_bounds__(kBlock) hashagg_bool_kernel(BitmapReader data, BitmapReader valid, const uint32_t* __restrict__ ids,
                                                              int64_t n, AggState st, int kind) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const uint32_t g = __ldcs(ids + i);
    if (!valid.bit(i)) {
      st.flags[g] |= 1;
      continue;
    }
    const bool v = data.bit(i);
    if (kind == B2_HASH_ANY) {
      if (v) st.reduced[g] = 1ull;   // benign race: every writer stores the same value
    } else if (!v) {
      st.reduced[g] = 0ull;
    }
    atomicAdd(&st.counts[g], 1ull);
  }
}

// any / all -> boolean column.  Validity: count >= min_count, and with skip_nulls = false a group that saw a null
// is null unless the value is already decided (any: true; all: false) -- AdjustForMinCount, hash_aggregate.cc:1376-1396
__global__ void __launch_bounds__(kBlock) hashagg_finalize_bool_kernel(AggState st, int64_t n, int kind, int skip_nulls,
                                                                       uint32_t min_count, uint32_t* out_data, uint32_t* out_validity,
                                                                       int64_t* valid_count) {
  int64_t nw = (n + 31) >> 5;
  int64_t local = 0;
  for (int64_t w = (blockIdx.x * (int64_t)kBlock + threadIdx.x) >> 5; w < nw; w += ((int64_t)gridDim.x * kBlock) >> 5) {
    const int64_t g = (w << 5) + lane_id();
    bool value = false, valid = false;
    if (g < n) {
      value = st.reduced[g] != 0ull;
      const bool saw_null = st.flags[g] & 1;
      valid = st.counts[g] >= min_count;
      if (!skip_nulls) valid = valid && (!saw_null || (kind == B2_HASH_ANY ? value : !value));
    }
    const unsigned dword = __ballot_sync(0xffffffffu, value), vword = __ballot_sync(0xffffffffu, valid);
    if (lane_id() == 0) {
      out_data[w] = dword;
      out_validity[w] = vword;
      local += __popc(vword);
    }
  }
  int64_t s = block_sum<kBlock>(local);
  if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(valid_count), (unsigned long long)s);
}

// Few groups (<= kPrivateMaxGroups): millions of rows update the same handful of state words, and
// same-address global atomics serialise (merging equal groups inside a warp does not help -- 32 rows
// over 100 groups are almost all distinct).  This
// variant keeps a private copy of the whole state in shared memory per CTA (integer sums as two
// 32-bit halves with an explicit carry: native ATOMS instead of a 64-bit CAS loop) and adds it to the
// global state once at the end: grid x G global atomics in total.
constexpr int kPrivateMaxGroups = 2048;

template <typename T, int KIND>
__global__ void __launch_bounds__(kBlock) hashagg_consume_private_kernel(const T* __restrict__ values, BitmapReader valid,
                                                                         const uint32_t* __restrict__ ids, int64_t n,
                                                                         AggState st, int num_groups, int count_mode) {
  constexpr bool kSum = KIND == B2_HASH_SUM || KIND == B2_HASH_MEAN;
  constexpr bool kDouble = kSum && (std::is_floating_point<T>::value || KIND == B2_HASH_MEAN);
  constexpr bool kCount = KIND == B2_HASH_COUNT || KIND == B2_HASH_COUNT_ALL;
  __shared__ unsigned long long s_red[kCount ? 1 : kPrivateMaxGroups];
  __shared__ unsigned int s_cnt[kPrivateMaxGroups];
  __shared__ uint8_t s_null[kPrivateMaxGroups];
  const unsigned long long identity = kSum ? 0ull : (KIND == B2_HASH_MIN ? ~0ull : 0ull);
  for (int g = threadIdx.x; g < num_groups; g += kBlock) {
    if (!kCount) s_red[g] = identity;
    s_cnt[g] = 0;
    s_null[g] = 0;
  }
  __syncthreads();
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const uint32_t g = __ldcs(ids + i);
    if (kCount) {  // count_mode: 0 only valid, 1 only null, 2 all (count_all passes 2)
      const bool ok = count_mode == 2 || valid.bit(i) == (count_mode == 0);
      if (ok) atomicAdd(&s_cnt[g], 1u);
      continue;
    }
    if (!valid.bit(i)) {
      s_null[g] = 1;
      continue;
    }
    const T v = __ldcs(values + i);
    if (kSum) {
      if (kDouble) {
        atomicAdd(reinterpret_cast<double*>(&s_red[g]), static_cast<double>(v));
      } else {
        const unsigned long long b = std::is_signed<T>::value ? static_cast<unsigned long long>(static_cast<long long>(v))
                                                             : static_cast<unsigned long long>(v);
        unsigned int* half = reinterpret_cast<unsigned int*>(&s_red[g]);  // little endian: [0] = lo, [1] = hi
        const unsigned int lo32 = static_cast<unsigned int>(b), hi32 = static_cast<unsigned int>(b >> 32);
        const unsigned int old = atomicAdd(half, lo32);
        const unsigned int carry = (old + lo32) < old ? 1u : 0u;
        if (hi32 + carry) atomicAdd(half + 1, hi32 + carry);
      }
    } else if (v == v) {  // fmin / fmax skip NaN
      if (KIND == B2_HASH_MIN) atomicMin(&s_red[g], minmax_encode<T>(v));
      else atomicMax(&s_red[g], minmax_encode<T>(v));
    }
    atomicAdd(&s_cnt[g], 1u);
  }
  __syncthreads();
  for (int g = threadIdx.x; g < num_groups; g += kBlock) {
    if (s_null[g]) st.flags[g] |= 1;
    const unsigned int c = s_cnt[g];
    if (!c) continue;
    if (kCount) {
      atomicAdd(&st.counts[g], static_cast<unsigned long long>(c));
      continue;
    }
    if (kSum) {
      if (kDouble) atomicAdd(reinterpret_cast<double*>(&st.reduced[g]), __longlong_as_double((long long)s_red[g]));
      else atomicAdd(&st.reduced[g], s_red[g]);
    } else if (KIND == B2_HASH_MIN) {
      atomicMin(&st.reduced[g], s_red[g]);
    } else {
      atomicMax(&st.reduced[g], s_red[g]);
    }
    atomicAdd(&st.counts[g], static_cast<unsigned long long>(c));
  }
}

__global__ void __launch_bounds__(kBlock) hashagg_countall_kernel(const uint32_t* __restrict__ ids, int64_t n,
                                                                  unsigned long long* counts) {
  const unsigned lane = lane_id();
  const int64_t stride = (int64_t)gridDim.x * kBlock;
  for (int64_t base = blockIdx.x * (int64_t)kBlock + (threadIdx.x & ~31u); base < n; base += stride) {
    const int64_t i = base + lane;
    count_merged(counts, i < n ? __ldcs(ids + i) : 0u, i < n);
  }
}

__global__ void __launch_bounds__(kBlock) hashagg_fill_kernel(unsigned long long* p, unsigned long long v,
                                                              int64_t from, int64_t to) {
  for (int64_t i = from + blockIdx.x * (int64_t)kBlock + threadIdx.x; i < to; i += (int64_t)gridDim.x * kBlock) p[i] = v;
}

// state[map[i]] (+)= other[i]
__global__ void __launch_bounds__(kBlock) hashagg_merge_kernel(AggState dst, AggState src, const uint32_t* map,
                                                               int64_t n, int kind, int acc) {
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const uint32_t g = map[i];
    atomicAdd(&dst.counts[g], src.counts[i]);
    if (src.flags[i] & 1) dst.flags[g] |= 1;
    if (kind == B2_HASH_SUM || kind == B2_HASH_MEAN) {
      if (acc == ACC_F64 || kind == B2_HASH_MEAN)
        atomicAdd(reinterpret_cast<double*>(&dst.reduced[g]), __longlong_as_double((long long)src.reduced[i]));
      else
        atomicAdd(&dst.reduced[g], src.reduced[i]);
    } else if (kind == B2_HASH_MIN) {
      atomicMin(&dst.reduced[g], src.reduced[i]);
    } else if (kind == B2_HASH_MAX) {
      atomicMax(&dst.reduced[g], src.reduced[i]);
    } else if (kind == B2_HASH_ANY) {
      atomicOr(&dst.reduced[g], src.reduced[i]);
    } else if (kind == B2_HASH_ALL) {
      atomicAnd(&dst.reduced[g], src.reduced[i]);
    } else if (kind == B2_HASH_PRODUCT) {
      unsigned long long* p = &dst.reduced[g];
      unsigned long long old = *reinterpret_cast<volatile unsigned long long*>(p), assumed;
      do {
        assumed = old;
        const unsigned long long next = acc == ACC_F64
            ? static_cast<unsigned long long>(__double_as_longlong(__longlong_as_double((long long)assumed) * __longlong_as_double((long long)src.reduced[i])))
            : assumed * src.reduced[i];
        old = atomicCAS(p, assumed, next);
      } while (old != assumed);
    }
  }
}

// state -> output column + validity (ballot) ; out_type is the finalized type id
__global__ void __launch_bounds__(kBlock) hashagg_finalize_kernel(AggState st, int64_t n, int kind, int acc,
                                                                  int out_type, int skip_nulls, uint32_t min_count,
                                                                  void* out, uint32_t* out_validity,
                                                                  int64_t* valid_count) {
  int64_t nw = (n + 31) >> 5;
  int64_t local = 0;
  for (int64_t w = (blockIdx.x * (int64_t)kBlock + threadIdx.x) >> 5; w < nw; w += ((int64_t)gridDim.x * kBlock) >> 5) {
    int64_t g = (w << 5) + lane_id();
    bool valid = false;
    if (g < n) {
      const unsigned long long c = st.counts[g];
      const unsigned long long r = st.reduced ? st.reduced[g] : 0ull;
      const bool saw_null = st.flags && (st.flags[g] & 1);
      if (kind == B2_HASH_COUNT || kind == B2_HASH_COUNT_ALL) {
        static_cast<long long*>(out)[g] = static_cast<long long>(c);
        valid = true;
      } else if (kind == B2_HASH_SUM || kind == B2_HASH_PRODUCT) {
        valid = c >= min_count && (skip_nulls || !saw_null);
        static_cast<unsigned long long*>(out)[g] = r;  // int64 / uint64 / double share the bits
      } else if (kind == B2_HASH_MEAN) {
        valid = c >= min_count && (skip_nulls || !saw_null);
        // an empty group with min_count == 0 is 0/0 = NaN, exactly as GroupedMeanImpl's sums[i] / counts[i]
        // (hash_aggregate_numeric.cc:402-421); null slots are zero-filled
        double m = c >= min_count ? __longlong_as_double((long long)r) / static_cast<double>(c) : 0.0;
        static_cast<double*>(out)[g] = m;
      } else {  // MIN / MAX: valid iff the group has a value (hash_aggregate.cc:401-411)
        valid = c > 0 && (skip_nulls || !saw_null);
        // decode the ordered key back into out_type
        unsigned long long k = r;
        if (out_type == B2_FLOAT || out_type == B2_DOUBLE) {
          unsigned long long b = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
          double d = __longlong_as_double((long long)b);
          // still the identity (~0 / 0 decode to NaN): the group's values were all NaN -> the canonical quiet NaN
          const bool nan = d != d;
          if (out_type == B2_FLOAT) static_cast<uint32_t*>(out)[g] = nan ? 0x7fc00000u : __float_as_uint(static_cast<float>(d));
          else static_cast<unsigned long long*>(out)[g] = nan ? 0x7ff8000000000000ull : static_cast<unsigned long long>(__double_as_longlong(d));
        } else {
          long long sv = (acc == ACC_I64) ? static_cast<long long>(k ^ 0x8000000000000000ull) : static_cast<long long>(k);
          switch (type_width(out_type)) {
            case 1: static_cast<uint8_t*>(out)[g] = static_cast<uint8_t>(sv); break;
            case 2: static_cast<uint16_t*>(out)[g] = static_cast<uint16_t>(sv); break;
            case 4: static_cast<uint32_t*>(out)[g] = static_cast<uint32_t>(sv); break;
            default: static_cast<unsigned long long*>(out)[g] = static_cast<unsigned long long>(sv); break;
          }
        }
      }
    }
    unsigned word = __ballot_sync(0xffffffffu, valid);
    if (lane_id() == 0) {
      out_validity[w] = word;
      local += __popc(word);
    }
  }
  int64_t s = block_sum<kBlock>(local);
  if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(valid_count), (unsigned long long)s);
}

}  // namespace b2

using namespace b2;

struct B2HashAgg {
  B2Context* ctx;
  int kind;
  int value_type;
  int acc;
  B2HashAggOptions opt;
  AggState st{};
  int64_t num_groups = 0;
  int64_t cap = 0;
  B2Grouper* pairs = nullptr;  // hash_count_distinct: the distinct (value, group id) pairs seen so far
  MomentAgg* mom = nullptr;    // variance / stddev / skew / kurtosis: their own state (hash_moments.cu)
};

static unsigned long long agg_identity(const B2HashAgg* a) {
  // anti-extrema in the ordered encoding (AntiExtrema<T>, hash_aggregate.cc:305-309 / 349-350): integers start at the
  // type's max / min; floats start at NaN, which std::fmin / std::fmax replace with the first non-NaN value, so a group
  // whose values are all NaN finalizes to NaN.  ~0 / 0 sit beyond the encodings of +inf / -inf and decode to NaN; the
  // NaN-skipping atomics and merge never produce them
  const bool flt = a->acc == ACC_F64;
  if (a->kind == B2_HASH_MIN) return ~0ull;
  if (a->kind == B2_HASH_MAX) return 0ull;
  if (a->kind == B2_HASH_PRODUCT) return flt ? 0x3ff0000000000000ull : 1ull;  // MultiplyTraits::one
  if (a->kind == B2_HASH_ALL) return 1ull;
  return 0ull;  // sum / mean: 0 (== 0.0); any: false
}

// B2_HASHAGG_BAND_MB: bytes of state one consume launch applies (L2 residency of the banded path below)
int64_t hashagg_band_bytes() {
  static const int64_t bytes = [] {
    const char* e = getenv("B2_HASHAGG_BAND_MB");
    return (e && atoll(e) > 0 ? atoll(e) : 24ll) << 20;
  }();
  return bytes;
}

template <typename T>
static int launch_consume(B2HashAgg* a, const B2Array* values, const B2Array* ids, cudaStream_t s) {
  const int64_t n = ids->length;
  const T* v = static_cast<const T*>(values->data) + values->offset;
  const uint32_t* id = static_cast<const uint32_t*>(ids->data) + ids->offset;
  BitmapReader valid(values->null_count == 0 ? nullptr : values->validity, values->offset, n);
  int grid = grid_for(n, kBlock * 4, kSMs * 16);
  // Every row is an atomic on its group's state.  While the state fits in L2 the atomics
  // resolve there; once reduced[] + counts[] outgrow it each one becomes a DRAM sector
  // read-modify-write.  Large batches are therefore consumed in BANDS of group ids whose state
  // stays L2-resident, re-streaming the ids (and the values of the band's rows) once per band.
  if (a->num_groups <= kPrivateMaxGroups && n >= (1 << 14) && a->kind != B2_HASH_PRODUCT) {
    const int g = (int)a->num_groups;
    const int pgrid = grid_for(n, kBlock * 64, kSMs * 8);  // few CTAs: each flushes the whole state once
    switch (a->kind) {
      case B2_HASH_SUM: hashagg_consume_private_kernel<T, B2_HASH_SUM><<<pgrid, kBlock, 0, s>>>(v, valid, id, n, a->st, g, 0); break;
      case B2_HASH_MEAN: hashagg_consume_private_kernel<T, B2_HASH_MEAN><<<pgrid, kBlock, 0, s>>>(v, valid, id, n, a->st, g, 0); break;
      case B2_HASH_MIN: hashagg_consume_private_kernel<T, B2_HASH_MIN><<<pgrid, kBlock, 0, s>>>(v, valid, id, n, a->st, g, 0); break;
      case B2_HASH_COUNT:
        hashagg_consume_private_kernel<T, B2_HASH_COUNT><<<pgrid, kBlock, 0, s>>>(v, valid, id, n, a->st, g, a->opt.count_mode);
        break;
      default: hashagg_consume_private_kernel<T, B2_HASH_MAX><<<pgrid, kBlock, 0, s>>>(v, valid, id, n, a->st, g, 0); break;
    }
    B2_LAUNCHED();
    return B2_OK;
  }
  // hash_sum over an integer column: the dense packed-state path of the fused group-by with the group ids as keys --
  // one RED per row instead of two atomics (groupby_fused.cu dense_sum_count_by_id).  The has-null flags it does not
  // maintain only matter to skip_nulls = false.
  if (a->kind == B2_HASH_SUM && std::is_integral<T>::value && (a->opt.skip_nulls || values->null_count == 0)) {
    bool done = false;
    B2_RETURN_NOT_OK(dense_sum_count_by_id(a->ctx, id, (uint64_t)a->num_groups, v, values->type, valid, n, a->st.reduced,
                                           a->st.counts, s, &done));
    if (done) return B2_OK;
  }
  const bool two_arrays = a->kind != B2_HASH_COUNT;
  const int64_t band_groups = hashagg_band_bytes() / (two_arrays ? 16 : 8);
  int64_t bands = (a->num_groups + band_groups - 1) / band_groups;
  if (bands < 1 || n < (1 << 24)) bands = 1;
  const int64_t per_band = (a->num_groups + bands - 1) / bands;
  for (int64_t b = 0; b < bands; ++b) {
    const uint32_t lo = bands == 1 ? 0u : static_cast<uint32_t>(b * per_band);
    const uint32_t hi = (bands == 1 || b == bands - 1) ? 0xffffffffu : static_cast<uint32_t>((b + 1) * per_band);
    switch (a->kind) {
      case B2_HASH_SUM: hashagg_consume_kernel<T, B2_HASH_SUM><<<grid, kBlock, 0, s>>>(v, valid, id, n, a->st, 0, lo, hi); break;
      case B2_HASH_MEAN: hashagg_consume_kernel<T, B2_HASH_MEAN><<<grid, kBlock, 0, s>>>(v, valid, id, n, a->st, 0, lo, hi); break;
      case B2_HASH_MIN: hashagg_consume_kernel<T, B2_HASH_MIN><<<grid, kBlock, 0, s>>>(v, valid, id, n, a->st, 0, lo, hi); break;
      case B2_HASH_MAX: hashagg_consume_kernel<T, B2_HASH_MAX><<<grid, kBlock, 0, s>>>(v, valid, id, n, a->st, 0, lo, hi); break;
      case B2_HASH_PRODUCT: hashagg_consume_kernel<T, B2_HASH_PRODUCT><<<grid, kBlock, 0, s>>>(v, valid, id, n, a->st, 0, lo, hi); break;
      case B2_HASH_COUNT:
        hashagg_consume_kernel<T, B2_HASH_COUNT><<<grid, kBlock, 0, s>>>(v, valid, id, n, a->st, a->opt.count_mode, lo, hi);
        break;
      default: return set_error(B2_NOT_IMPLEMENTED, "hash aggregate kind %d", a->kind);
    }
    B2_LAUNCHED();
  }
  return B2_OK;
}

extern "C" {

int b2_hashagg_create(B2Context* ctx, int kind, int32_t value_type, const B2HashAggOptions* options,
                      B2HashAgg** out) {
  if (!ctx || !out) return set_error(B2_INVALID, "b2_hashagg_create: null argument");
  if (kind < B2_HASH_SUM || kind > B2_HASH_KURTOSIS)
    return set_error(B2_NOT_IMPLEMENTED, "hash aggregate kind %d is not implemented", kind);
  if (is_moment_kind(kind)) {
    // VarianceOptions / SkewOptions defaults: skip_nulls, min_count 0, ddof 0 / biased (api_aggregate.h:103-134)
    const B2HashAggOptions opt = options ? *options : B2HashAggOptions{1, 0, 0, 0};
    MomentAgg* m = nullptr;
    B2_RETURN_NOT_OK(moments_create(ctx, kind, value_type, opt, &m));
    B2HashAgg* a = new B2HashAgg();
    a->ctx = ctx;
    a->kind = kind;
    a->value_type = value_type;
    a->acc = ACC_F64;
    a->opt = opt;
    a->mom = m;
    *out = a;
    return B2_OK;
  }
  if (kind == B2_HASH_COUNT_DISTINCT) {
    // GroupedCountDistinctImpl keeps a Grouper over (value, group id) (hash_aggregate.cc:1400-1478, made by
    // GroupedDistinctInit :1560-1575); the pair is wider than 64 bits for 8-byte and string values: grouper_wide.cu
    if (!type_is_numeric(value_type) && !type_is_binary_like(value_type))
      return set_error(B2_NOT_IMPLEMENTED, "hash_count_distinct over value type id %d", value_type);
    B2HashAgg* a = new B2HashAgg();
    a->ctx = ctx;
    a->kind = kind;
    a->value_type = value_type;
    a->acc = ACC_I64;
    a->opt = options ? *options : B2HashAggOptions{1, 1, 0, 0};
    const int32_t kt[2] = {value_type, B2_UINT32};
    const int st = b2_grouper_create(ctx, kt, 2, &a->pairs);
    if (st != B2_OK) {
      delete a;
      return st;
    }
    *out = a;
    return B2_OK;
  }
  if (kind == B2_HASH_ANY || kind == B2_HASH_ALL) {
    if (value_type != B2_BOOL) return set_error(B2_NOT_IMPLEMENTED, "hash_any / hash_all need a boolean column (type id %d)", value_type);
  } else if (kind != B2_HASH_COUNT_ALL && kind != B2_HASH_COUNT && !type_is_numeric(value_type)) {
    return set_error(B2_NOT_IMPLEMENTED, "hash aggregate over value type id %d", value_type);
  }
  B2HashAgg* a = new B2HashAgg();
  a->ctx = ctx;
  a->kind = kind;
  a->value_type = value_type;
  a->acc = acc_kind_for(value_type);
  if (options) a->opt = *options;
  else a->opt = B2HashAggOptions{1, 1, 0, 0};
  *out = a;
  return B2_OK;
}

void b2_hashagg_destroy(B2HashAgg* a) {
  if (!a) return;
  cudaSetDevice(a->ctx->device);
  cudaStream_t s = a->ctx->stream;
  if (a->st.reduced) a->ctx->free(a->st.reduced, s);
  if (a->st.counts) a->ctx->free(a->st.counts, s);
  if (a->st.flags) a->ctx->free(a->st.flags, s);
  if (a->pairs) b2_grouper_destroy(a->pairs);
  if (a->mom) moments_destroy(a->mom);
  delete a;
}

int32_t b2_hashagg_out_type(const B2HashAgg* a) {
  if (!a) return B2_NA;
  switch (a->kind) {
    case B2_HASH_COUNT: case B2_HASH_COUNT_ALL: case B2_HASH_COUNT_DISTINCT: return B2_INT64;
    case B2_HASH_MEAN: case B2_HASH_VARIANCE: case B2_HASH_STDDEV: case B2_HASH_SKEW: case B2_HASH_KURTOSIS: return B2_DOUBLE;
    case B2_HASH_SUM: case B2_HASH_PRODUCT: return a->acc == ACC_I64 ? B2_INT64 : a->acc == ACC_U64 ? B2_UINT64 : B2_DOUBLE;
    case B2_HASH_ANY: case B2_HASH_ALL: return B2_BOOL;
    default: return a->value_type;
  }
}

int b2_hashagg_resize(B2HashAgg* a, int64_t num_groups, void* stream) {
  if (!a) return set_error(B2_INVALID, "b2_hashagg_resize: null argument");
  if (num_groups < a->num_groups) return set_error(B2_INVALID, "hash aggregate state cannot shrink");
  B2Context* ctx = a->ctx;
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  if (a->kind == B2_HASH_COUNT_DISTINCT) {  // the state is the pair grouper; only the group count is kept (:1408-1411)
    a->num_groups = num_groups;
    return B2_OK;
  }
  if (a->mom) {
    B2_RETURN_NOT_OK(moments_resize(a->mom, num_groups, s));
    a->num_groups = num_groups;
    return B2_OK;
  }
  if (num_groups > a->cap) {
    int64_t cap = static_cast<int64_t>(next_pow2(num_groups < 1024 ? 1024 : num_groups));
    void *r, *c, *f;
    B2_RETURN_NOT_OK(ctx->alloc(cap * 8, &r, s));
    B2_RETURN_NOT_OK(ctx->alloc(cap * 8, &c, s));
    B2_RETURN_NOT_OK(ctx->alloc(cap, &f, s));
    if (a->num_groups) {
      B2_CUDA(cudaMemcpyAsync(r, a->st.reduced, a->num_groups * 8, cudaMemcpyDeviceToDevice, s));
      B2_CUDA(cudaMemcpyAsync(c, a->st.counts, a->num_groups * 8, cudaMemcpyDeviceToDevice, s));
      B2_CUDA(cudaMemcpyAsync(f, a->st.flags, a->num_groups, cudaMemcpyDeviceToDevice, s));
    }
    if (a->st.reduced) ctx->free(a->st.reduced, s);
    if (a->st.counts) ctx->free(a->st.counts, s);
    if (a->st.flags) ctx->free(a->st.flags, s);
    a->st.reduced = static_cast<unsigned long long*>(r);
    a->st.counts = static_cast<unsigned long long*>(c);
    a->st.flags = static_cast<uint8_t*>(f);
    a->cap = cap;
  }
  const int64_t added = num_groups - a->num_groups;
  if (added > 0) {
    hashagg_fill_kernel<<<grid_for(added, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(a->st.reduced, agg_identity(a),
                                                                                 a->num_groups, num_groups);
    B2_LAUNCHED();
    B2_CUDA(cudaMemsetAsync(a->st.counts + a->num_groups, 0, added * 8, s));
    B2_CUDA(cudaMemsetAsync(a->st.flags + a->num_groups, 0, added, s));
  }
  a->num_groups = num_groups;
  return B2_OK;
}

int b2_hashagg_consume(B2HashAgg* a, const B2Array* values, const B2Array* ids, void* stream) {
  if (!a || (!ids && !(a->mom && a->num_groups == 1))) return set_error(B2_INVALID, "b2_hashagg_consume: null argument");
  if (ids && ids->type != B2_UINT32) return set_error(B2_TYPE_ERROR, "group ids must be uint32");
  B2Context* ctx = a->ctx;
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  if (a->mom) return moments_consume(a->mom, values, ids, s);
  const int64_t n = ids->length;
  if (n == 0) return B2_OK;
  if (a->kind == B2_HASH_COUNT_DISTINCT) {
    if (!values) return set_error(B2_INVALID, "hash aggregate needs a value column");
    if (values->length != n) return set_error(B2_INVALID, "values and group ids differ in length");
    if (values->type != a->value_type)
      return set_error(B2_TYPE_ERROR, "hash aggregate was created for type id %d, got %d", a->value_type, values->type);
    const B2Array keys[2] = {*values, *ids};
    PoolArray pair_ids(ctx, s);
    return b2_grouper_consume(a->pairs, keys, &pair_ids.a, s);
  }
  const uint32_t* id = static_cast<const uint32_t*>(ids->data) + ids->offset;
  const bool few_groups = a->num_groups <= kPrivateMaxGroups && n >= (1 << 14);
  const int pgrid = grid_for(n, kBlock * 64, kSMs * 8);
  if (a->kind == B2_HASH_COUNT_ALL) {
    if (few_groups) {
      hashagg_consume_private_kernel<uint8_t, B2_HASH_COUNT_ALL><<<pgrid, kBlock, 0, s>>>(
          nullptr, BitmapReader(nullptr, 0, n), id, n, a->st, (int)a->num_groups, 2);
    } else {
      hashagg_countall_kernel<<<grid_for(n, kBlock * 4, kSMs * 16), kBlock, 0, s>>>(id, n, a->st.counts);
    }
    B2_LAUNCHED();
    return B2_OK;
  }
  if (!values) return set_error(B2_INVALID, "hash aggregate needs a value column");
  if (values->length != n) return set_error(B2_INVALID, "values and group ids differ in length");
  if (a->kind == B2_HASH_COUNT && !type_is_numeric(values->type)) {
    // count only needs validity: any layout works
    BitmapReader valid(values->null_count == 0 ? nullptr : values->validity, values->offset, n);
    if (few_groups)
      hashagg_consume_private_kernel<uint8_t, B2_HASH_COUNT><<<pgrid, kBlock, 0, s>>>(nullptr, valid, id, n, a->st,
                                                                                      (int)a->num_groups, a->opt.count_mode);
    else
      hashagg_consume_kernel<uint8_t, B2_HASH_COUNT><<<grid_for(n, kBlock * 4, kSMs * 16), kBlock, 0, s>>>(
          nullptr, valid, id, n, a->st, a->opt.count_mode, 0u, 0xffffffffu);
    B2_LAUNCHED();
    return B2_OK;
  }
  if (values->type != a->value_type && a->kind != B2_HASH_COUNT)
    return set_error(B2_TYPE_ERROR, "hash aggregate was created for type id %d, got %d", a->value_type, values->type);
  if (a->kind == B2_HASH_ANY || a->kind == B2_HASH_ALL) {
    BitmapReader data(values->data, values->offset, n);
    BitmapReader valid(values->null_count == 0 ? nullptr : values->validity, values->offset, n);
    hashagg_bool_kernel<<<grid_for(n, kBlock * 4, kSMs * 16), kBlock, 0, s>>>(data, valid, id, n, a->st, a->kind);
    B2_LAUNCHED();
    return B2_OK;
  }
  switch (values->type) {
    case B2_INT8: return launch_consume<int8_t>(a, values, ids, s);
    case B2_UINT8: return launch_consume<uint8_t>(a, values, ids, s);
    case B2_INT16: return launch_consume<int16_t>(a, values, ids, s);
    case B2_UINT16: return launch_consume<uint16_t>(a, values, ids, s);
    case B2_INT32: return launch_consume<int32_t>(a, values, ids, s);
    case B2_UINT32: return launch_consume<uint32_t>(a, values, ids, s);
    case B2_INT64: return launch_consume<int64_t>(a, values, ids, s);
    case B2_UINT64: return launch_consume<uint64_t>(a, values, ids, s);
    case B2_FLOAT: return launch_consume<float>(a, values, ids, s);
    case B2_DOUBLE: return launch_consume<double>(a, values, ids, s);
    default: return set_error(B2_NOT_IMPLEMENTED, "hash aggregate over value type id %d", values->type);
  }
}

int b2_hashagg_merge(B2HashAgg* a, B2HashAgg* other, const B2Array* group_id_mapping, void* stream) {
  if (!a || !other || !group_id_mapping) return set_error(B2_INVALID, "b2_hashagg_merge: null argument");
  if (a->kind != other->kind || a->value_type != other->value_type)
    return set_error(B2_INVALID, "cannot merge different aggregators");
  if (group_id_mapping->type != B2_UINT32 || group_id_mapping->length != other->num_groups)
    return set_error(B2_INVALID, "group_id_mapping must be uint32 with one entry per group of `other`");
  B2Context* ctx = a->ctx;
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = other->num_groups;
  if (a->kind == B2_HASH_COUNT_DISTINCT) {
    // other's distinct (value, group) pairs with the group ids translated, consumed like a batch (:1418-1439)
    B2Array pairs[2] = {};
    B2_RETURN_NOT_OK(b2_grouper_uniques(other->pairs, pairs, s));
    PoolArray vals(ctx, s), gids(ctx, s), mapped(ctx, s), pair_ids(ctx, s);
    vals.a = pairs[0];
    gids.a = pairs[1];
    if (pairs[0].length == 0) return B2_OK;
    B2_RETURN_NOT_OK(b2_take(ctx, group_id_mapping, &gids.a, 1, &mapped.a, s));
    const B2Array keys[2] = {vals.a, mapped.a};
    return b2_grouper_consume(a->pairs, keys, &pair_ids.a, s);
  }
  if (a->mom) return moments_merge(a->mom, other->mom, group_id_mapping, s);
  if (n == 0) return B2_OK;
  const uint32_t* map = static_cast<const uint32_t*>(group_id_mapping->data) + group_id_mapping->offset;
  hashagg_merge_kernel<<<grid_for(n, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(a->st, other->st, map, n, a->kind, a->acc);
  B2_LAUNCHED();
  return B2_OK;
}

int b2_hashagg_finalize(B2HashAgg* a, B2Array* out, void* stream) {
  if (!a || !out) return set_error(B2_INVALID, "b2_hashagg_finalize: null argument");
  B2Context* ctx = a->ctx;
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  if (a->mom) return moments_finalize(a->mom, out, s);
  const int64_t n = a->num_groups;
  const int out_type = b2_hashagg_out_type(a);
  if (a->kind == B2_HASH_COUNT_DISTINCT) {
    // counts[g] = distinct values of group g that CountOptions::mode admits (:1441-1468) = hash_count over the pairs
    B2Array pairs[2] = {};
    B2_RETURN_NOT_OK(b2_grouper_uniques(a->pairs, pairs, s));
    PoolArray vals(ctx, s), gids(ctx, s);
    vals.a = pairs[0];
    gids.a = pairs[1];
    B2HashAgg* counter = nullptr;
    B2HashAggOptions co{1, 0, a->opt.count_mode, 0};
    B2_RETURN_NOT_OK(b2_hashagg_create(ctx, B2_HASH_COUNT, a->value_type, &co, &counter));
    int st = b2_hashagg_resize(counter, n, s);
    if (st == B2_OK) st = b2_hashagg_consume(counter, &vals.a, &gids.a, s);
    if (st == B2_OK) st = b2_hashagg_finalize(counter, out, s);
    b2_hashagg_destroy(counter);
    return st;
  }
  Temp data(ctx, s), bits(ctx, s);
  if (out_type == B2_BOOL) {
    B2_RETURN_NOT_OK(data.alloc(bitmap_alloc_bytes(n)));
    int64_t bnulls = 0;
    if (n > 0) {
      B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(n)));
      B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bitmap_alloc_bytes(n), s));
      B2_CUDA(cudaMemsetAsync(data.ptr, 0, bitmap_alloc_bytes(n), s));
      ScalarSlot slot(ctx);
      B2_RETURN_NOT_OK(slot.zero(s));
      hashagg_finalize_bool_kernel<<<grid_for(n, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(
          a->st, n, a->kind, a->opt.skip_nulls, a->opt.min_count, data.as<uint32_t>(), bits.as<uint32_t>(), slot.dev());
      B2_LAUNCHED();
      B2_RETURN_NOT_OK(slot.fetch(s));
      bnulls = n - slot.host()[0];
    }
    fill_out(out, B2_BOOL, n, bnulls, bnulls ? bits.release() : nullptr, data.release());
    return B2_OK;
  }
  B2_RETURN_NOT_OK(data.alloc((size_t)n * type_width(out_type)));
  int64_t nulls = 0;
  if (n > 0) {
    B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(n)));
    B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bitmap_alloc_bytes(n), s));
    ScalarSlot slot(ctx);
    B2_RETURN_NOT_OK(slot.zero(s));
    hashagg_finalize_kernel<<<grid_for(n, kBlock * 4, kSMs * 8), kBlock, 0, s>>>(
        a->st, n, a->kind, a->acc, out_type, a->opt.skip_nulls, a->opt.min_count, data.ptr, bits.as<uint32_t>(),
        slot.dev());
    B2_LAUNCHED();
    B2_RETURN_NOT_OK(slot.fetch(s));
    nulls = n - slot.host()[0];
  }
  fill_out(out, out_type, n, nulls, nulls ? bits.release() : nullptr, data.release());
  return B2_OK;
}

}  // extern "C"
