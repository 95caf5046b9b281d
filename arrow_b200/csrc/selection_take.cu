// selection_take.cu -- Take (gather) for fixed-width and dictionary-index columns.
//
// Replaces:
//   FixedWidthTakeExec + FixedWidthTakeImpl      kernels/vector_selection_take_internal.cc:336-468
//   Gather<..>::Execute / GatherBaseCRTP::ExecuteWithNulls   kernels/gather_internal.h:84-251
//   CheckIndexBounds                             util/int_util.cc:452-560 (IndexError)
//   DictionaryTake (takes the index column)      kernels/vector_selection_take_internal.cc:488-497
// Semantics kept: out[i] = values[idx[i]]; out valid = idx valid AND values valid at
// idx[i]; signed index types are bounds-checked then reinterpreted as unsigned; null
// indices are never dereferenced and produce a zero-filled null slot; with boundscheck
// the first out-of-range VALID index raises IndexError("Index <v> out of bounds").
//
// Design: one streaming pass.  Each lane loads V consecutive indices with one
// 16-byte coalesced load per unroll step (U steps issued back to back => U*V independent
// gathers in flight per lane, the only way to cover random-access DRAM latency), gathers
// values and validity bits, stores V results with one vector store, and the warp packs
// its 32*V validity bits into V words with redux.sync.  The gather itself is sector-
// granular (32 B fetched per 8 B element for random indices): algorithmic bytes/row are
// idx + 2*W + 2/8 (24.25 for int64 idx / float64, SURVEY section 8d) but DRAM traffic
// for uniformly random indices is ~idx + 32 + W.
#include <cstdlib>
#include <type_traits>

#include "bitmap.h"
#include "elementwise.cuh"
#include "selection.cuh"
#include "take_partitioned.h"

namespace b2 {

template <int W>
struct TakeBytes;
template <> struct TakeBytes<1> { using type = uint8_t; };
template <> struct TakeBytes<2> { using type = uint16_t; };
template <> struct TakeBytes<4> { using type = uint32_t; };
template <> struct TakeBytes<8> { using type = uint64_t; };
template <> struct TakeBytes<16> { using type = uint4; };

template <typename T>
__device__ __forceinline__ T zero_value() {
  return T{};
}
template <>
__device__ __forceinline__ uint4 zero_value<uint4>() {
  return make_uint4(0, 0, 0, 0);
}

struct TakeArgs {
  const void* values;  // advanced by offset * W
  BitmapReader values_valid;
  int64_t values_length;
  const void* indices;  // advanced by offset * sizeof(Idx)
  BitmapReader idx_valid;
  int64_t n;
  void* out;
  uint32_t* out_validity;  // NULL when no validity is produced
  int64_t* valid_count;    // device counter (popcount of out validity)
  unsigned long long* first_bad;  // device, ~0 initially
  bool vec_ok;
  int64_t band_rows;  // validity of values[j] is probed here only for j < band_rows (INT64_MAX: every row); see take_bands
};

// pack each lane's V bits (bit k = element lane*V+k) into V warp-wide words;
// lane j < V returns word j
template <int V>
__device__ __forceinline__ unsigned warp_pack_bits(unsigned m, unsigned lane) {
  const unsigned my_word = (lane * V) >> 5;
  const unsigned shifted = m << ((lane * V) & 31);
  unsigned mine = 0;
#pragma unroll
  for (int j = 0; j < V; ++j) {
    unsigned w = __reduce_or_sync(0xffffffffu, my_word == j ? shifted : 0u);
    if (lane == j) mine = w;
  }
  return mine;
}


// ---- validity probes in L2-sized bands ---------------------------------------------------------------------------------
// A random probe of the values' validity bitmap is a DRAM access whenever the bitmap does not stay in L2, and DRAM
// random accesses (not bytes) are what bounds Take, whatever is fetched (bench_micro/gather_probe.cu); a bitmap
// far larger than L2 adds a DRAM access for a large share of the probes.  So for big bitmaps the bitmap is cut
// into K bands of <= B2_TAKE_BAND_MB (default 32, two thirds of the H100's 50 MB L2) each: the gather kernel probes band 0 only (rows whose index falls in another
// band are provisionally valid), and K-1 follow-up launches re-stream the INDICES (sequential, 1.2 ps/row) and
// clear the bits of band b -- every launch's probes hit a bitmap slice that fits L2.  Results are identical.
__device__ __forceinline__ bool probe_band0(const BitmapReader& valid, uint64_t j, int64_t band_rows, uint64_t pol) {
  return static_cast<int64_t>(j) < band_rows ? valid.bit_hint(static_cast<int64_t>(j), pol) : true;
}

struct TakeBandArgs {
  const void* indices;  // advanced by offset
  BitmapReader values_valid;
  int64_t lo, rows;     // this launch probes lo <= j < lo + rows
  int64_t n;
  uint32_t* out_validity;  // bit i set: index i valid, in bounds (and the fused kernel's other operand valid)
  int64_t* valid_count;
  bool vec_ok;
};

template <typename UIdx>  // uint32_t / uint64_t: a set output bit implies 0 <= j < values_length, so signedness is moot
__global__ void __launch_bounds__(kBlock) take_validity_band_kernel(TakeBandArgs a) {
  constexpr int V = 16 / sizeof(UIdx);
  constexpr int UU = kUnroll;
  constexpr int64_t kWarpTile = 32 * V * UU;
  constexpr int64_t kTile = kWarpTile * kWarpsPerBlock;
  const unsigned lane = lane_id();
  const UIdx* __restrict__ idx = static_cast<const UIdx*>(a.indices);
  const uint64_t pol_bitmap = l2_policy_evict_last();
  const uint64_t lo = static_cast<uint64_t>(a.lo), rows = static_cast<uint64_t>(a.rows);
  int64_t cleared = 0;
  for (int64_t tile = (int64_t)blockIdx.x * kTile; tile < a.n; tile += (int64_t)gridDim.x * kTile) {
    const int64_t wb = tile + (int64_t)(threadIdx.x >> 5) * kWarpTile;
    if (wb >= a.n) continue;
    if (a.vec_ok && wb + kWarpTile <= a.n) {
      Vec<UIdx, V> ix[UU];
      unsigned cur[UU];
#pragma unroll
      for (int u = 0; u < UU; ++u) {
        const int64_t i0 = wb + u * 32 * V + lane * V;
        ix[u] = load_vec<UIdx, V>(idx + i0);
        cur[u] = (a.out_validity[i0 >> 5] >> (i0 & 31)) & ((1u << V) - 1u);  // V divides 32: no straddling
      }
      unsigned clear[UU];
#pragma unroll
      for (int u = 0; u < UU; ++u) {
        clear[u] = 0;
#pragma unroll
        for (int k = 0; k < V; ++k) {
          const uint64_t j = static_cast<uint64_t>(ix[u].v[k]);
          if (((cur[u] >> k) & 1u) && (j - lo) < rows)
            clear[u] |= (a.values_valid.bit_hint(static_cast<int64_t>(j), pol_bitmap) ? 0u : 1u) << k;
        }
      }
      __syncwarp();  // every lane has read its output word before the owners rewrite them
#pragma unroll
      for (int u = 0; u < UU; ++u) {
        const unsigned w = warp_pack_bits<V>(clear[u], lane);
        if (lane < V && w) {
          uint32_t* word = a.out_validity + ((wb + u * 32 * V) >> 5) + lane;
          *word &= ~w;  // this lane owns the word: probed bits were set, so exactly popc(w) bits go
          cleared += __popc(w);
        }
      }
    } else {
      const int64_t end = wb + kWarpTile < a.n ? wb + kWarpTile : a.n;
      for (int64_t base = wb; base < end; base += 32) {
        const int64_t i = base + lane;
        bool clr = false;
        const uint32_t curw = a.out_validity[base >> 5];
        if (i < end && ((curw >> lane) & 1u)) {
          const uint64_t j = static_cast<uint64_t>(idx[i]);
          if ((j - lo) < rows) clr = !a.values_valid.bit_hint(static_cast<int64_t>(j), pol_bitmap);
        }
        const unsigned w = __ballot_sync(0xffffffffu, clr);
        if (lane == 0 && w) {
          a.out_validity[base >> 5] = curw & ~w;
          cleared += __popc(w);
        }
      }
    }
  }
  const int64_t s = block_sum<kBlock>(cleared);
  if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(a.valid_count), static_cast<unsigned long long>(-s));
}

// Are the indices clustered?  2048 evenly spaced pairs (idx[p], idx[p+1]): the share whose targets lie within 64Ki rows
// (8 KB of bitmap) of each other.  Clustered / monotonic indices probe the bitmap almost sequentially -- banding would only
// add passes over the indices.
template <typename UIdx>
__global__ void __launch_bounds__(kBlock) idx_locality_kernel(const UIdx* __restrict__ idx, int64_t n, int64_t* near) {
  constexpr int kPairs = 2048;
  int local = 0;
  for (int s = threadIdx.x; s < kPairs; s += kBlock) {
    const int64_t p = (n - 1) / kPairs * s;
    const uint64_t a = static_cast<uint64_t>(idx[p]), b = static_cast<uint64_t>(idx[p + 1]);
    const uint64_t d = a > b ? a - b : b - a;
    local += d < 65536 ? 1 : 0;
  }
  const int64_t t = block_sum<kBlock>(local);
  if (threadIdx.x == 0) *near = t;
}

template <int W, typename Idx, bool HAS_VALID>
__global__ void __launch_bounds__(kBlock) take_kernel(TakeArgs a) {
  using T = typename TakeBytes<W>::type;
  constexpr int V = 16 / (sizeof(Idx) > W ? sizeof(Idx) : W);
  constexpr int UU = kUnroll;
  constexpr int64_t kWarpTile = 32 * V * UU;
  constexpr int64_t kTile = kWarpTile * kWarpsPerBlock;
  const unsigned lane = lane_id();
  const T* __restrict__ vals = static_cast<const T*>(a.values);
  const Idx* __restrict__ idx = static_cast<const Idx*>(a.indices);
  T* __restrict__ out = static_cast<T*>(a.out);
  const uint64_t vlen = static_cast<uint64_t>(a.values_length);
  int64_t valid_local = 0;
  // values are touched once per gather (evict-first); the validity bitmap is 1/64 of their
  // size and hit by every row: keep it resident in L2 (evict-last)
  const uint64_t pol_values = l2_policy_evict_first();
  const uint64_t pol_bitmap = l2_policy_evict_last();

  for (int64_t tile = (int64_t)blockIdx.x * kTile; tile < a.n; tile += (int64_t)gridDim.x * kTile) {
    int64_t wb = tile + (int64_t)(threadIdx.x >> 5) * kWarpTile;
    if (wb >= a.n) continue;
    if (a.vec_ok && wb + kWarpTile <= a.n) {
      Vec<Idx, V> ix[UU];
      unsigned ivalid[UU];
#pragma unroll
      for (int u = 0; u < UU; ++u) {
        int64_t i0 = wb + u * 32 * V + lane * V;
        ix[u] = load_vec<Idx, V>(idx + i0);
        // i0 is a multiple of V and V divides 64: the V bits never straddle a word
        ivalid[u] = HAS_VALID ? static_cast<unsigned>(a.idx_valid.word(i0 >> 6) >> (i0 & 63)) & ((1u << V) - 1u)
                              : ((1u << V) - 1u);
      }
      Vec<T, V> g[UU];
      unsigned gvalid[UU];
#pragma unroll
      for (int u = 0; u < UU; ++u) {
        gvalid[u] = 0;
#pragma unroll
        for (int k = 0; k < V; ++k) {
          // signed -> unsigned reinterpretation after the bounds check (gather_internal.h)
          uint64_t j = static_cast<uint64_t>(static_cast<int64_t>(ix[u].v[k]));
          if (std::is_unsigned<Idx>::value) j = static_cast<uint64_t>(ix[u].v[k]);
          bool iv = (ivalid[u] >> k) & 1;
          bool inb = j < vlen;
          if (iv && !inb) atomicMin(a.first_bad, static_cast<unsigned long long>(wb + u * 32 * V + lane * V + k));
          if (iv && inb) {
            g[u].v[k] = ld_hint<T>(vals + j, pol_values);
            if (HAS_VALID) gvalid[u] |= (probe_band0(a.values_valid, j, a.band_rows, pol_bitmap) ? 1u : 0u) << k;
          } else {
            g[u].v[k] = zero_value<T>();
          }
        }
      }
#pragma unroll
      for (int u = 0; u < UU; ++u) {
        int64_t i0 = wb + u * 32 * V + lane * V;
        store_vec<T, V>(out + i0, g[u]);
        if (HAS_VALID) {
          unsigned w = warp_pack_bits<V>(gvalid[u], lane);
          if (lane < V) {
            a.out_validity[((wb + u * 32 * V) >> 5) + lane] = w;
            valid_local += __popc(w);
          }
        }
      }
    } else {
      int64_t end = wb + kWarpTile < a.n ? wb + kWarpTile : a.n;
      for (int64_t base = wb; base < end; base += 32) {
        int64_t i = base + lane;
        bool ov = false;
        if (i < end) {
          bool iv = HAS_VALID ? a.idx_valid.bit(i) : true;
          Idx raw = idx[i];
          uint64_t j = std::is_unsigned<Idx>::value ? static_cast<uint64_t>(raw)
                                                    : static_cast<uint64_t>(static_cast<int64_t>(raw));
          bool inb = j < vlen;
          if (iv && !inb) atomicMin(a.first_bad, static_cast<unsigned long long>(i));
          if (iv && inb) {
            out[i] = ld_hint<T>(vals + j, pol_values);
            ov = HAS_VALID ? probe_band0(a.values_valid, j, a.band_rows, pol_bitmap) : true;
          } else {
            out[i] = zero_value<T>();
          }
        }
        if (HAS_VALID) {
          unsigned w = __ballot_sync(0xffffffffu, ov);
          if (lane == 0) {
            a.out_validity[base >> 5] = w;
            valid_local += __popc(w);
          }
        }
      }
    }
  }
  if (HAS_VALID) {
    int64_t s = block_sum<kBlock>(valid_local);
    if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(a.valid_count), (unsigned long long)s);
  }
}

template <int W, typename Idx>
static int launch_take(const TakeArgs& a, bool has_valid, cudaStream_t s) {
  constexpr int V = 16 / (sizeof(Idx) > W ? sizeof(Idx) : W);
  constexpr int64_t kTile = (int64_t)32 * V * kUnroll * kWarpsPerBlock;
  int grid = grid_for(a.n, kTile, kSMs * 8 * 16);
  if (has_valid) take_kernel<W, Idx, true><<<grid, kBlock, 0, s>>>(a);
  else take_kernel<W, Idx, false><<<grid, kBlock, 0, s>>>(a);
  B2_LAUNCHED();
  return B2_OK;
}

// ---- fused Take -> Cast -> arithmetic ---------------------------------------------------------------------------------
// out[i] = op(static_cast<OT>(values[idx[i]]), other[i]) in one pass: the expression add(cast(take(v, idx), T), other) of
// BASELINE configs[1], which the reference executes as three kernels with two materialised intermediates
// (ExecuteScalarExpression, compute/expression.cc:722-797).  Identical results: the cast is the unchecked static_cast
// (CastOptions::Unsafe; to a float type it never fails), the arithmetic a single IEEE operation, validity =
// idx valid AND values valid at idx AND other valid, out-of-range indices raise IndexError like b2_take.
// Saves writing and re-reading the taken column and the cast column (16 + 8 B/row of 48.9).
struct FusedTakeArgs {
  const void* values;
  BitmapReader values_valid;
  int64_t values_length;
  const void* indices;
  BitmapReader idx_valid;
  const void* other;       // NULL: broadcast scalar `other_scalar`
  double other_scalar;
  BitmapReader other_valid;
  int op;                  // B2_ADD / B2_SUBTRACT / B2_MULTIPLY
  int64_t n;
  void* out;
  uint32_t* out_validity;
  int64_t* valid_count;
  unsigned long long* first_bad;
  bool vec_ok;
  int64_t band_rows;  // as in TakeArgs
};

template <typename VT, typename Idx, typename OT, bool HAS_VALID>
__global__ void __launch_bounds__(kBlock) take_cast_arith_kernel(FusedTakeArgs a) {
  constexpr int V = 16 / (sizeof(Idx) > sizeof(OT) ? sizeof(Idx) : sizeof(OT));
  constexpr int UU = kUnroll;
  constexpr int64_t kWarpTile = 32 * V * UU;
  constexpr int64_t kTile = kWarpTile * kWarpsPerBlock;
  const unsigned lane = lane_id();
  const VT* __restrict__ vals = static_cast<const VT*>(a.values);
  const Idx* __restrict__ idx = static_cast<const Idx*>(a.indices);
  const OT* __restrict__ other = static_cast<const OT*>(a.other);
  OT* __restrict__ out = static_cast<OT*>(a.out);
  const OT oscalar = static_cast<OT>(a.other_scalar);
  const uint64_t vlen = static_cast<uint64_t>(a.values_length);
  int64_t valid_local = 0;
  const uint64_t pol_values = l2_policy_evict_first();
  const uint64_t pol_bitmap = l2_policy_evict_last();
  for (int64_t tile = (int64_t)blockIdx.x * kTile; tile < a.n; tile += (int64_t)gridDim.x * kTile) {
    int64_t wb = tile + (int64_t)(threadIdx.x >> 5) * kWarpTile;
    if (wb >= a.n) continue;
    if (a.vec_ok && wb + kWarpTile <= a.n) {
      Vec<Idx, V> ix[UU];
      Vec<OT, V> oth[UU];
      unsigned rvalid[UU];  // idx valid AND other valid
#pragma unroll
      for (int u = 0; u < UU; ++u) {
        const int64_t i0 = wb + u * 32 * V + lane * V;
        ix[u] = load_vec<Idx, V>(idx + i0);
        if (other) {
          oth[u] = load_vec<OT, V>(other + i0);
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) oth[u].v[k] = oscalar;
        }
        rvalid[u] = (1u << V) - 1u;
        if (HAS_VALID)  // i0 is a multiple of V and V divides 64: the V bits never straddle a word
          rvalid[u] &= static_cast<unsigned>((a.idx_valid.word(i0 >> 6) & a.other_valid.word(i0 >> 6)) >> (i0 & 63));
      }
      Vec<OT, V> r[UU];
      unsigned gvalid[UU];
#pragma unroll
      for (int u = 0; u < UU; ++u) {
        gvalid[u] = 0;
#pragma unroll
        for (int k = 0; k < V; ++k) {
          uint64_t j = std::is_unsigned<Idx>::value ? static_cast<uint64_t>(ix[u].v[k]) : static_cast<uint64_t>(static_cast<int64_t>(ix[u].v[k]));
          // bounds are checked for every VALID INDEX, whatever `other` holds (exactly what take alone would raise)
          const bool iv = HAS_VALID ? a.idx_valid.bit(wb + u * 32 * V + lane * V + k) : true;
          const bool inb = j < vlen;
          if (iv && !inb) atomicMin(a.first_bad, static_cast<unsigned long long>(wb + u * 32 * V + lane * V + k));
          VT g = VT(0);
          if (iv && inb) {
            g = ld_hint<VT>(vals + j, pol_values);
            if (HAS_VALID && ((rvalid[u] >> k) & 1u))
              gvalid[u] |= (probe_band0(a.values_valid, j, a.band_rows, pol_bitmap) ? 1u : 0u) << k;
          }
          r[u].v[k] = fused_apply<OT>(a.op, static_cast<OT>(g), oth[u].v[k]);
        }
      }
#pragma unroll
      for (int u = 0; u < UU; ++u) {
        const int64_t i0 = wb + u * 32 * V + lane * V;
        store_vec<OT, V>(out + i0, r[u]);
        if (HAS_VALID) {
          unsigned w = warp_pack_bits<V>(gvalid[u], lane);
          if (lane < V) {
            a.out_validity[((wb + u * 32 * V) >> 5) + lane] = w;
            valid_local += __popc(w);
          }
        }
      }
    } else {
      int64_t end = wb + kWarpTile < a.n ? wb + kWarpTile : a.n;
      for (int64_t base = wb; base < end; base += 32) {
        int64_t i = base + lane;
        bool ov = false;
        if (i < end) {
          const bool iv = HAS_VALID ? a.idx_valid.bit(i) : true;
          const Idx raw = idx[i];
          uint64_t j = std::is_unsigned<Idx>::value ? static_cast<uint64_t>(raw) : static_cast<uint64_t>(static_cast<int64_t>(raw));
          const bool inb = j < vlen;
          if (iv && !inb) atomicMin(a.first_bad, static_cast<unsigned long long>(i));
          VT g = VT(0);
          if (iv && inb) {
            g = ld_hint<VT>(vals + j, pol_values);
            ov = HAS_VALID ? (a.other_valid.bit(i) && probe_band0(a.values_valid, j, a.band_rows, pol_bitmap)) : true;
          }
          out[i] = fused_apply<OT>(a.op, static_cast<OT>(g), other ? other[i] : oscalar);
        }
        if (HAS_VALID) {
          unsigned w = __ballot_sync(0xffffffffu, ov);
          if (lane == 0) {
            a.out_validity[base >> 5] = w;
            valid_local += __popc(w);
          }
        }
      }
    }
  }
  if (HAS_VALID) {
    int64_t s = block_sum<kBlock>(valid_local);
    if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(a.valid_count), (unsigned long long)s);
  }
}

template <typename VT, typename Idx, typename OT>
static int launch_fused_take(const FusedTakeArgs& a, bool has_valid, cudaStream_t s) {
  constexpr int V = 16 / (sizeof(Idx) > sizeof(OT) ? sizeof(Idx) : sizeof(OT));
  constexpr int64_t kTile = (int64_t)32 * V * kUnroll * kWarpsPerBlock;
  int grid = grid_for(a.n, kTile, kSMs * 8 * 16);
  if (has_valid) take_cast_arith_kernel<VT, Idx, OT, true><<<grid, kBlock, 0, s>>>(a);
  else take_cast_arith_kernel<VT, Idx, OT, false><<<grid, kBlock, 0, s>>>(a);
  B2_LAUNCHED();
  return B2_OK;
}

template <typename OT>
static int launch_fused_take_val(int value_type, int idx_type, const FusedTakeArgs& a, bool has_valid, cudaStream_t s) {
  return visit_type(
      FusedTakeValueTypes{}, value_type,
      [&](auto vt) {
        return visit_type(
            WideIndexTypes{}, idx_type,
            [&](auto it) { return launch_fused_take<decltype(vt), decltype(it), OT>(a, has_valid, s); },
            [&] { return set_error(B2_NOT_IMPLEMENTED, "b2_take_cast_arith: 32- or 64-bit indices only (type id %d)", idx_type); });
      },
      [&] {
        return set_error(B2_NOT_IMPLEMENTED, "b2_take_cast_arith: float64 / float32 / int64 / int32 values only (type id %d)",
                         value_type);
      });
}


// Band plan (see probe_band0).  Banding pays when the probes would thrash: a bitmap well beyond what L2 keeps
// (bench_micro/gather_probe.cu measures the gather rate against the table size) and enough rows that every bitmap line is
// probed many times; each extra band costs one sequential pass over the indices.
struct TakeBands {
  int k = 1;
  int64_t rows = INT64_MAX;
};

static TakeBands take_bands(const B2Array* values, int64_t n, int iw) {
  TakeBands b;
  // B2_TAKE_BAND_MB: band size (0 disables); B2_TAKE_BAND_KB: the same in KB and without the size thresholds (tests)
  const char* ekb = getenv("B2_TAKE_BAND_KB");
  const char* emb = getenv("B2_TAKE_BAND_MB");
  int64_t band = ekb ? (strtol(ekb, nullptr, 10) << 10) : ((emb ? strtol(emb, nullptr, 10) : 32) << 20);
  if (band <= 0 || values->null_count == 0 || !values->validity || (iw != 4 && iw != 8)) return b;
  const int64_t bytes = values->length >> 3;
  if (!ekb && (bytes * 4 < band * 5 || n < (1 << 24))) return b;  // a bitmap up to 1.25 bands is left alone
  const int64_t k = (bytes + band - 1) / band;
  if (k < 2 || k > 6) return b;  // beyond 6 the index re-reads would cost what the misses do
  b.k = static_cast<int>(k);
  b.rows = (((values->length + k - 1) / k) + 1023) & ~int64_t(1023);
  return b;
}

// one tiny kernel + read-back; only reached for large takes
static int indices_clustered(B2Context* ctx, const void* indices, int iw, int64_t n, cudaStream_t s, bool* clustered) {
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  if (iw == 4) idx_locality_kernel<uint32_t><<<1, kBlock, 0, s>>>(static_cast<const uint32_t*>(indices), n, slot.dev());
  else idx_locality_kernel<uint64_t><<<1, kBlock, 0, s>>>(static_cast<const uint64_t*>(indices), n, slot.dev());
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(slot.fetch(s));
  *clustered = slot.host()[0] > 1024;
  return B2_OK;
}

// drop the banding for clustered indices
static int take_bands_check_locality(B2Context* ctx, TakeBands* bands, const void* indices, int iw, int64_t n, cudaStream_t s) {
  if (bands->k < 2 || getenv("B2_TAKE_BAND_KB")) return B2_OK;
  bool clustered = false;
  B2_RETURN_NOT_OK(indices_clustered(ctx, indices, iw, n, s, &clustered));
  if (clustered) *bands = TakeBands{};
  return B2_OK;
}

// ---- partitioned path plan (take_partitioned.cu) ------------------------------------------------------------------------
// Random indices into values far larger than L2 are gathered band by band; below the thresholds (scripts/
// take_partition_sweep.py measures the crossover) and for clustered indices the direct kernels are faster.
// B2_TAKE_PARTITION=0|1 forces the direct / partitioned path (where the latter applies: 4- or 8-byte values, 32- or 64-bit
// indices, n < 2^30, 1 <= values_length <= 2^32); B2_TAKE_PART_BAND_KB sets the band (default 32 MB, 16 MB of the folded
// table) and, like B2_TAKE_BAND_KB, drops the size thresholds so tests reach the path at small sizes.  Both are read on
// every call.
constexpr int64_t kPartMinValueBytes = 1ll << 30;
constexpr int64_t kPartMinRows = 1ll << 26;

// the bucket shift of a band of `band` bytes over `vlen` rows of `width` bytes (bucket of index j = j >> shift, < 256)
static int band_shift(int64_t vlen, int width, int64_t band) {
  int shift = 0;
  while ((static_cast<int64_t>(width) << (shift + 1)) <= band) ++shift;  // band rows: the largest power of two that fits
  while (((vlen - 1) >> shift) >= 256) ++shift;
  return shift;
}

// returns the bucket shift, or -1 for the direct kernels.  *fold: gather from a float32 copy of the values with the nulls
// folded in (take_partitioned.cu pass F): a cast to float32 of 8-byte values with nulls, in bands the sentinels can
// number.  Its bands are counted in bytes of the folded table.
static int take_partition_plan(const B2Array* values, int64_t n, int vw, int iw, int out_type, bool* fold) {
  *fold = false;
  const char* ep = getenv("B2_TAKE_PARTITION");
  if (ep && ep[0] == '0') return -1;
  const int64_t vlen = values->length;
  if ((vw != 4 && vw != 8) || (iw != 4 && iw != 8) || n >= (1ll << 30) || vlen < 1 || vlen > (1ll << 32)) return -1;
  const char* ekb = getenv("B2_TAKE_PART_BAND_KB");
  if (!(ep && ep[0] == '1') && !ekb && (vlen * vw < kPartMinValueBytes || n < kPartMinRows)) return -1;
  if (out_type == B2_FLOAT && (values->type == B2_DOUBLE || values->type == B2_INT64) && values->null_count > 0 &&
      values->validity) {
    const int shift = band_shift(vlen, sizeof(float), ekb ? (strtol(ekb, nullptr, 10) << 10) : (16ll << 20));
    *fold = shift >= kFoldMinShift && shift <= kFoldMaxShift;
    if (*fold) return shift;
  }
  return band_shift(vlen, vw, ekb ? (strtol(ekb, nullptr, 10) << 10) : (32ll << 20));
}

// runs the partitioned path when take_partition_plan picks it and the indices are not clustered; *ran = false leaves the
// call to the direct kernels
static int try_take_partitioned(B2Context* ctx, const B2Array* values, PartTakeArgs p, int vw, int idx_type, int out_type,
                                cudaStream_t s, bool* ran) {
  *ran = false;
  const int iw = type_width(idx_type);
  p.shift = take_partition_plan(values, p.n, vw, iw, out_type, &p.fold);
  if (p.shift < 0) return B2_OK;
  p.value_nulls = values->null_count;
  const char* ep = getenv("B2_TAKE_PARTITION");
  if (!(ep && ep[0] == '1') && !getenv("B2_TAKE_PART_BAND_KB")) {
    bool clustered = false;
    B2_RETURN_NOT_OK(indices_clustered(ctx, p.indices, iw, p.n, s, &clustered));
    if (clustered) return B2_OK;
  }
  return take_partitioned(ctx, p, vw, values->type, idx_type, out_type, s, ran);
}

static int launch_take_bands(const TakeBands& bands, const void* indices, int iw, const BitmapReader& values_valid, int64_t n,
                             uint32_t* out_validity, int64_t* valid_count, cudaStream_t s) {
  for (int b = 1; b < bands.k; ++b) {
    TakeBandArgs a;
    a.indices = indices;
    a.values_valid = values_valid;
    a.lo = b * bands.rows;
    a.rows = bands.rows;
    a.n = n;
    a.out_validity = out_validity;
    a.valid_count = valid_count;
    a.vec_ok = aligned_to(indices, 16);
    const int64_t tile = (int64_t)32 * (16 / iw) * kUnroll * kWarpsPerBlock;
    const int grid = grid_for(n, tile, kSMs * 8 * 16);
    if (iw == 4) take_validity_band_kernel<uint32_t><<<grid, kBlock, 0, s>>>(a);
    else take_validity_band_kernel<uint64_t><<<grid, kBlock, 0, s>>>(a);
    B2_LAUNCHED();
  }
  return B2_OK;
}

int take_bool(B2Context* ctx, const B2Array* values, const B2Array* indices, B2Array* out, cudaStream_t s);  // selection_bool.cu
int take_binary(B2Context* ctx, const B2Array* values, const B2Array* indices, int boundscheck,
                B2Array* out, cudaStream_t s);  // selection_binary.cu

// Reads the offending index back for the IndexError message (util/int_util.cc:554-555)
int index_error(const B2Array* indices, uint64_t row, cudaStream_t s) {
  int iw = type_width(indices->type);
  uint64_t raw = 0;
  B2_CUDA(cudaMemcpyAsync(&raw, static_cast<const char*>(indices->data) + (indices->offset + row) * iw, iw,
                          cudaMemcpyDeviceToHost, s));
  B2_CUDA(cudaStreamSynchronize(s));
  bool is_signed = indices->type == B2_INT8 || indices->type == B2_INT16 || indices->type == B2_INT32 ||
                   indices->type == B2_INT64;
  if (is_signed) {
    int64_t v = iw == 1 ? (int8_t)raw : iw == 2 ? (int16_t)raw : iw == 4 ? (int32_t)raw : (int64_t)raw;
    return set_error(B2_INDEX_ERROR, "Index %lld out of bounds", (long long)v);
  }
  return set_error(B2_INDEX_ERROR, "Index %llu out of bounds", (unsigned long long)raw);
}

}  // namespace b2

using namespace b2;

extern "C" int b2_binary_data_size(B2Context* ctx, const B2Array* array, int64_t* out_bytes, void* stream) {
  if (!ctx || !array || !out_bytes) return set_error(B2_INVALID, "b2_binary_data_size: null argument");
  if (!type_is_binary_like(array->type)) return set_error(B2_TYPE_ERROR, "b2_binary_data_size: not a binary-like array");
  *out_bytes = 0;
  if (array->length == 0 || !array->data) return B2_OK;
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int ow = offset_width(array->type);
  int64_t first = 0, last = 0;
  const char* base = static_cast<const char*>(array->data);
  B2_CUDA(cudaMemcpyAsync(&first, base + array->offset * ow, ow, cudaMemcpyDeviceToHost, s));
  B2_CUDA(cudaMemcpyAsync(&last, base + (array->offset + array->length) * ow, ow, cudaMemcpyDeviceToHost, s));
  B2_CUDA(cudaStreamSynchronize(s));
  *out_bytes = last - first;  // little-endian: the low `ow` bytes were filled
  return B2_OK;
}

extern "C" int b2_take_cast_arith(B2Context* ctx, const B2Array* values, const B2Array* indices, int32_t to_type, int op,
                                  const B2Value* other, B2Array* out, void* stream) {
  if (!ctx || !values || !indices || !other || !out) return set_error(B2_INVALID, "b2_take_cast_arith: null argument");
  if (to_type != B2_FLOAT && to_type != B2_DOUBLE) return set_error(B2_NOT_IMPLEMENTED, "b2_take_cast_arith: the cast target must be float32 or float64");
  if (op != B2_ADD && op != B2_SUBTRACT && op != B2_MULTIPLY) return set_error(B2_NOT_IMPLEMENTED, "b2_take_cast_arith: add / subtract / multiply only");
  if (values->length < 0 || indices->length < 0 || values->offset < 0 || indices->offset < 0) return set_error(B2_INVALID, "negative length/offset");
  const B2Array* oa = other->array;
  if (oa && (oa->type != to_type || oa->length != indices->length))
    return set_error(B2_INVALID, "b2_take_cast_arith: `other` must have the cast target type and the indices' length");
  if (!oa && (!other->scalar || other->scalar->type != to_type)) return set_error(B2_INVALID, "b2_take_cast_arith: scalar `other` must have the cast target type");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = indices->length;
  const int ow = type_width(to_type), iw = type_width(indices->type), vw = type_width(values->type);
  if (n == 0) {
    fill_out(out, to_type, 0, 0, nullptr, nullptr);
    return B2_OK;
  }
  const bool scalar_null = !oa && !other->scalar->is_valid;
  const bool has_valid = (values->null_count != 0 && values->validity) || (indices->null_count != 0 && indices->validity) ||
                         (oa && oa->null_count != 0 && oa->validity) || scalar_null;
  Temp data(ctx, s), bits(ctx, s);
  B2_RETURN_NOT_OK(data.alloc(static_cast<size_t>(n) * ow));
  const size_t bit_bytes = bitmap_alloc_bytes(n);
  if (has_valid) {
    B2_RETURN_NOT_OK(bits.alloc(bit_bytes));
    const size_t tail = bit_bytes >= 24 ? bit_bytes - 24 : 0;
    B2_CUDA(cudaMemsetAsync(static_cast<char*>(bits.ptr) + tail, 0, bit_bytes - tail, s));
  }
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  B2_CUDA(cudaMemsetAsync(slot.dev() + 1, 0xff, 8, s));
  FusedTakeArgs a;
  a.values = static_cast<const char*>(values->data) + values->offset * vw;
  a.values_valid = BitmapReader(values->null_count == 0 ? nullptr : values->validity, values->offset, values->length);
  a.values_length = values->length;
  a.indices = static_cast<const char*>(indices->data) + indices->offset * iw;
  a.idx_valid = BitmapReader(indices->null_count == 0 ? nullptr : indices->validity, indices->offset, n);
  a.other = oa ? static_cast<const char*>(oa->data) + oa->offset * ow : nullptr;
  a.other_scalar = 0.0;
  if (!oa && other->scalar->is_valid) {
    if (to_type == B2_FLOAT) {
      float f;
      const uint32_t b = static_cast<uint32_t>(other->scalar->bits);
      memcpy(&f, &b, 4);
      a.other_scalar = f;
    } else {
      memcpy(&a.other_scalar, &other->scalar->bits, 8);
    }
  }
  a.other_valid = BitmapReader((oa && oa->null_count != 0) ? oa->validity : nullptr, oa ? oa->offset : 0, n);
  a.op = op;
  a.n = n;
  a.out = data.ptr;
  a.out_validity = bits.as<uint32_t>();
  a.valid_count = slot.dev();
  a.first_bad = reinterpret_cast<unsigned long long*>(slot.dev() + 1);
  a.vec_ok = aligned_to(a.indices, 16) && aligned_to(a.out, 16) && (!a.other || aligned_to(a.other, 16));
  if (scalar_null) return set_error(B2_NOT_IMPLEMENTED, "b2_take_cast_arith: null scalar operand (the result is all null; use the unfused kernels)");
  PartTakeArgs p;
  p.values = a.values;
  p.values_valid = a.values_valid;
  p.values_length = a.values_length;
  p.indices = a.indices;
  p.idx_valid = a.idx_valid;
  p.n = n;
  p.other = a.other;
  p.other_scalar = a.other_scalar;
  p.other_valid = a.other_valid;
  p.op = op;
  p.out = a.out;
  p.out_validity = has_valid ? a.out_validity : nullptr;
  p.valid_count = a.valid_count;
  p.first_bad = a.first_bad;
  p.stalled = reinterpret_cast<unsigned long long*>(slot.dev() + 2);
  bool partitioned = false;
  if (vw == 4 || vw == 8) B2_RETURN_NOT_OK(try_take_partitioned(ctx, values, p, vw, indices->type, to_type, s, &partitioned));
  if (!partitioned) {
    TakeBands bands = take_bands(values, n, iw);
    B2_RETURN_NOT_OK(take_bands_check_locality(ctx, &bands, a.indices, iw, n, s));
    a.band_rows = bands.rows;
    int st = to_type == B2_FLOAT ? launch_fused_take_val<float>(values->type, indices->type, a, has_valid, s)
                                 : launch_fused_take_val<double>(values->type, indices->type, a, has_valid, s);
    if (st != B2_OK) return st;
    B2_RETURN_NOT_OK(launch_take_bands(bands, a.indices, iw, a.values_valid, n, a.out_validity, a.valid_count, s));
  }
  B2_RETURN_NOT_OK(slot.fetch(s));
  const uint64_t bad = static_cast<uint64_t>(slot.host()[1]);
  if (slot.host()[2])
    return set_error(B2_UNKNOWN_ERROR, "b2_take_cast_arith: the folded gather pass waited too long for a fold item it depends on");
  if (bad != ~0ull) return index_error(indices, bad, s);
  const int64_t null_count = has_valid ? n - slot.host()[0] : 0;
  fill_out(out, to_type, n, null_count, (has_valid && null_count) ? bits.release() : nullptr, data.release());
  return B2_OK;
}

extern "C" int b2_take(B2Context* ctx, const B2Array* values, const B2Array* indices, int boundscheck,
                       B2Array* out, void* stream) {
  if (!ctx || !values || !indices || !out) return set_error(B2_INVALID, "b2_take: null argument");
  if (values->length < 0 || indices->length < 0 || values->offset < 0 || indices->offset < 0)
    return set_error(B2_INVALID, "negative length/offset");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  if (type_is_binary_like(values->type)) return take_binary(ctx, values, indices, boundscheck, out, s);
  if (values->type == B2_BOOL) return take_bool(ctx, values, indices, out, s);
  int width = values->type == B2_FIXED_SIZE_BINARY ? values->byte_width : type_width(values->type);
  if (width != 1 && width != 2 && width != 4 && width != 8 && width != 16)
    return set_error(B2_NOT_IMPLEMENTED, "take: unsupported value type id %d (width %d)", values->type, width);
  int iw = type_width(indices->type);
  if (iw == 0 || indices->type == B2_FLOAT || indices->type == B2_DOUBLE || indices->type == B2_HALF_FLOAT)
    return index_type_error(indices->type);
  const int64_t n = indices->length;
  if (n == 0) {
    fill_out(out, values->type, 0, 0, nullptr, nullptr);
    out->byte_width = values->byte_width;
    return B2_OK;
  }
  const bool has_valid = (values->null_count != 0 && values->validity) ||
                         (indices->null_count != 0 && indices->validity);
  Temp data(ctx, s), bits(ctx, s);
  B2_RETURN_NOT_OK(data.alloc(static_cast<size_t>(n) * width));
  size_t bit_bytes = bitmap_alloc_bytes(n);
  if (has_valid) {
    B2_RETURN_NOT_OK(bits.alloc(bit_bytes));
    size_t tail = bit_bytes >= 24 ? bit_bytes - 24 : 0;
    B2_CUDA(cudaMemsetAsync(static_cast<char*>(bits.ptr) + tail, 0, bit_bytes - tail, s));
  }
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  B2_CUDA(cudaMemsetAsync(slot.dev() + 1, 0xff, 8, s));
  TakeArgs a;
  a.values = static_cast<const char*>(values->data) + values->offset * width;
  a.values_valid = BitmapReader(values->null_count == 0 ? nullptr : values->validity, values->offset, values->length);
  a.values_length = values->length;
  a.indices = static_cast<const char*>(indices->data) + indices->offset * iw;
  a.idx_valid = BitmapReader(indices->null_count == 0 ? nullptr : indices->validity, indices->offset, n);
  a.n = n;
  a.out = data.ptr;
  a.out_validity = bits.as<uint32_t>();
  a.valid_count = slot.dev();
  a.first_bad = reinterpret_cast<unsigned long long*>(slot.dev() + 1);
  a.vec_ok = aligned_to(a.indices, 16) && aligned_to(a.out, 16);
  PartTakeArgs p;
  p.values = a.values;
  p.values_valid = a.values_valid;
  p.values_length = a.values_length;
  p.indices = a.indices;
  p.idx_valid = a.idx_valid;
  p.n = n;
  p.other = nullptr;
  p.other_scalar = 0.0;
  p.op = 0;
  p.out = a.out;
  p.out_validity = has_valid ? a.out_validity : nullptr;
  p.valid_count = a.valid_count;
  p.first_bad = a.first_bad;
  p.stalled = nullptr;  // only the folded gather of b2_take_cast_arith waits
  bool partitioned = false;
  if (width == 4 || width == 8) B2_RETURN_NOT_OK(try_take_partitioned(ctx, values, p, width, indices->type, -1, s, &partitioned));
  if (!partitioned) {
    TakeBands bands = take_bands(values, n, iw);
    B2_RETURN_NOT_OK(take_bands_check_locality(ctx, &bands, a.indices, iw, n, s));
    a.band_rows = bands.rows;
    B2_RETURN_NOT_OK((visit_width<1, 2, 4, 8, 16>(width, [&](auto w) {
      return visit_type(IndexTypes{}, indices->type, [&](auto it) { return launch_take<w, decltype(it)>(a, has_valid, s); });
    })));
    B2_RETURN_NOT_OK(launch_take_bands(bands, a.indices, iw, a.values_valid, n, a.out_validity, a.valid_count, s));
  }
  B2_RETURN_NOT_OK(slot.fetch(s));
  uint64_t bad = static_cast<uint64_t>(slot.host()[1]);
  if (bad != ~0ull) {
    // without boundscheck the reference's behaviour is undefined; we still refuse to
    // return garbage silently
    return index_error(indices, bad, s);
  }
  int64_t null_count = has_valid ? n - slot.host()[0] : 0;
  fill_out(out, values->type, n, null_count, (has_valid && null_count) ? bits.release() : nullptr, data.release());
  out->byte_width = values->byte_width;
  (void)boundscheck;
  return B2_OK;
}
