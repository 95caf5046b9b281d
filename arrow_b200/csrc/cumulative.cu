// cumulative.cu -- cumulative_sum / _checked, cumulative_prod / _checked, cumulative_min / max / mean over the integer
// types and float32 / float64, for one array or the chunks of one ChunkedArray.
//
// Replaces CumulativeBinaryOp, CumulativeMean, Accumulator, CumulativeKernel and CumulativeKernelChunked
// (kernels/vector_cumulative_ops.cc:67-203) over Add(Checked), Multiply(Checked), Min, Max and their identities
// (kernels/base_arithmetic_internal.h:678-775).
//
// The reference folds `current = Op(arg, current)` row by row.  Every one of these folds is associative once written
// as a combine of an EARLIER state e and a LATER one l: integer sum / prod wrap in two's complement; float min / max
// return the later value on a tie (std::min(arg, current) returns arg) and treat NaN as an identity on either side
// (Min / Max :678-720), so they pick the rightmost extreme; the mean carries {sum, count}.  Nulls join the state as a
// "null seen" bit under skip_nulls = false: combine(e, l) = e.null ? e : {op(e.v, l.v), l.null}.
//
// One single-pass scan (Merrill & Garland, "Single-pass Parallel Prefix Scan with Decoupled Look-back", 2016).
// Tiles of 256 threads x 16 rows take tickets from a per-chunk counter, so every earlier tile belongs to a CTA that is
// running or done and no residency is assumed.  A warp stages its 512 rows through shared memory so that each lane
// folds 16 consecutive rows; lanes and warps combine by shuffles; the tile publishes its aggregate, looks back 32
// predecessors per step, and publishes its inclusive state.  The state (a value of up to 16 bytes plus the null bit)
// does not fit one flag-and-count cell, so the value words are stored first and the status word after them with
// release semantics, and readers load the status with acquire semantics before the words.
//
// Chunks: one launch per non-empty chunk into one output.  The last tile of chunk k stores its inclusive state in a
// device carry that tile 0 of chunk k + 1 starts from, so chunks follow each other in stream order with no host
// synchronisation.  A chunk whose output starts inside a 64-bit validity word ORs its validity words in atomically
// (the previous chunk wrote the low bits of that word); an aligned chunk stores them.
//
// Checked ops need no second pass: until the first overflow the wrapped prefix equals the exact one, so the first
// row whose exact sum / product leaves T is the first row r with op_overflows(prefix_wrapped(r - 1), x_r).  Each lane
// holds that exclusive prefix while it writes its rows, and a call raises iff some combined row fails that check:
// if none fails, every prefix is exact and nothing overflowed; if one fails, the earliest failing row is the
// reference's first overflow (every earlier prefix was exact), and the reference raises too.
//
// Roofline: one read and one write of the values plus the bitmaps; int64 with a nullable input: 16.25 B/row.
#include <cuda/atomic>

#include <cmath>
#include <limits>
#include <type_traits>

#include "elementwise.cuh"

namespace b2 {

constexpr int kScanItems = 16;                     // rows per lane
constexpr int kScanWarpRows = 32 * kScanItems;     // 512 rows per warp
constexpr int kScanTile = kBlock * kScanItems;     // 4096 rows per tile

struct MeanAcc {
  double sum;
  int64_t count;
};

// The cumulative op over T: its scan identity, its combine of an earlier and a later value, and what a row outputs.
template <typename T, int OP>
struct CumOp {
  static constexpr bool kFloat = std::is_floating_point<T>::value;
  static constexpr bool kSum = OP == B2_CUMULATIVE_SUM || OP == B2_CUMULATIVE_SUM_CHECKED;
  static constexpr bool kProd = OP == B2_CUMULATIVE_PROD || OP == B2_CUMULATIVE_PROD_CHECKED;
  static constexpr bool kMean = OP == B2_CUMULATIVE_MEAN;
  static constexpr bool kChecked = !kFloat && (OP == B2_CUMULATIVE_SUM_CHECKED || OP == B2_CUMULATIVE_PROD_CHECKED);
  using V = typename std::conditional<kMean, MeanAcc, T>::type;
  using Out = typename std::conditional<kMean, double, T>::type;
  using UT = typename std::conditional<kFloat, std::common_type<T>, std::make_unsigned<T>>::type::type;

  // op(identity, x) == x bit for bit: -0.0 for a float sum (+0.0 + -0.0 is +0.0), NaN for float min / max (ignored)
  __host__ __device__ static V identity() {
    if constexpr (kMean) return MeanAcc{0.0, 0};
    else if constexpr (kSum) return kFloat ? -T(0) : T(0);
    else if constexpr (kProd) return T(1);
    else if constexpr (kFloat) return std::numeric_limits<T>::quiet_NaN();
    else if constexpr (OP == B2_CUMULATIVE_MIN) return std::numeric_limits<T>::max();
    else return std::numeric_limits<T>::lowest();
  }
  __device__ __forceinline__ static V lift(T x) {
    if constexpr (kMean) return MeanAcc{static_cast<double>(x), 1};
    else return x;
  }
  __device__ __forceinline__ static V combine(V e, V l) {
    if constexpr (kMean) {
      return MeanAcc{e.sum + l.sum, e.count + l.count};
    } else if constexpr (kSum) {
      if constexpr (kFloat) return e + l;
      else return static_cast<T>(static_cast<UT>(e) + static_cast<UT>(l));
    } else if constexpr (kProd) {
      if constexpr (kFloat) {
        return e * l;
      } else {
        T r;
        mul_overflow(e, l, &r);
        return r;
      }
    } else if constexpr (OP == B2_CUMULATIVE_MIN) {
      if constexpr (kFloat) {
        if (isnan(l)) return e;
        if (isnan(e)) return l;
      }
      return e < l ? e : l;
    } else {
      if constexpr (kFloat) {
        if (isnan(l)) return e;
        if (isnan(e)) return l;
      }
      return l < e ? e : l;
    }
  }
  // whether combining x onto the exact prefix e leaves T (AddChecked / MultiplyChecked)
  __device__ __forceinline__ static bool overflows(V e, T x) {
    if constexpr (!kChecked) {
      return false;
    } else if constexpr (kProd) {
      T r;
      return mul_overflow(e, x, &r);
    } else if constexpr (sizeof(T) < 8) {
      using Wide = typename std::conditional<std::is_signed<T>::value, int64_t, uint64_t>::type;
      const Wide s = static_cast<Wide>(e) + static_cast<Wide>(x);
      return static_cast<Wide>(static_cast<T>(s)) != s;
    } else {
      const T r = static_cast<T>(static_cast<UT>(e) + static_cast<UT>(x));
      if constexpr (std::is_signed<T>::value) return ((e ^ r) & (x ^ r)) < 0;
      else return r < e;
    }
  }
  __device__ __forceinline__ static Out output(V v) {
    if constexpr (kMean) return v.sum / static_cast<double>(v.count);
    else return v;
  }
};

template <typename V>
struct ScanState {
  V v;
  uint32_t null;  // a null row was combined (skip_nulls = false): later rows are not
};

template <typename Op, typename V>
__device__ __forceinline__ ScanState<V> combine_state(ScanState<V> e, ScanState<V> l) {
  if (e.null) return e;
  return ScanState<V>{Op::combine(e.v, l.v), l.null};
}

template <typename S>
__device__ __forceinline__ S shfl_state(S s, int lane_or_delta, int mode) {
  constexpr int W = (sizeof(S) + 3) / 4;
  uint32_t w[W] = {};
  memcpy(w, &s, sizeof(S));
#pragma unroll
  for (int i = 0; i < W; ++i) {
    if (mode == 0) w[i] = __shfl_sync(0xffffffffu, w[i], lane_or_delta);
    else if (mode == 1) w[i] = __shfl_up_sync(0xffffffffu, w[i], lane_or_delta);
    else w[i] = __shfl_down_sync(0xffffffffu, w[i], lane_or_delta);
  }
  memcpy(&s, w, sizeof(S));
  return s;
}

// A tile's published state.  status: 0 nothing yet, kCellAgg | null << 2 the tile's aggregate in agg,
// kCellIncl | null << 2 its inclusive prefix in incl.  The words are written before the status that announces them.
struct ScanCell {
  unsigned long long agg[2];
  unsigned long long incl[2];
  unsigned long long status;
};
constexpr unsigned long long kCellAgg = 1, kCellIncl = 2;

using DevAtomic = cuda::atomic_ref<unsigned long long, cuda::thread_scope_device>;

template <typename V>
__device__ __forceinline__ void publish(ScanCell* c, bool inclusive, ScanState<V> s) {
  unsigned long long w[2] = {0, 0};
  memcpy(w, &s.v, sizeof(V));
  unsigned long long* dst = inclusive ? c->incl : c->agg;
  DevAtomic(dst[0]).store(w[0], cuda::memory_order_relaxed);
  DevAtomic(dst[1]).store(w[1], cuda::memory_order_relaxed);
  DevAtomic(c->status).store((inclusive ? kCellIncl : kCellAgg) | (static_cast<unsigned long long>(s.null) << 2),
                             cuda::memory_order_release);
}

// The state folded over tiles [first published inclusive .. tile - 1], walked back 32 cells per step by one warp.
template <typename Op, typename V>
__device__ ScanState<V> look_back(ScanCell* cells, int64_t tile) {
  const int lane = static_cast<int>(lane_id());
  ScanState<V> excl{Op::identity(), 0};
  int64_t back = tile - 1;  // newest cell not folded in yet
  while (true) {
    const int64_t t = back - lane;
    unsigned long long st = kCellIncl;  // before tile 0: never reached, tile 0 publishes its inclusive state at once
    if (t >= 0) {
      do {
        st = DevAtomic(cells[t].status).load(cuda::memory_order_acquire);
      } while (st == 0);
    }
    const unsigned incl_mask = __ballot_sync(0xffffffffu, (st & 3) == kCellIncl);
    const int first = incl_mask ? __ffs(incl_mask) - 1 : 31;  // lanes 0 .. first contribute
    ScanState<V> s{Op::identity(), 0};
    if (t >= 0 && lane <= first) {
      const unsigned long long* src = (st & 3) == kCellIncl ? cells[t].incl : cells[t].agg;
      unsigned long long w[2];
      w[0] = DevAtomic(const_cast<unsigned long long&>(src[0])).load(cuda::memory_order_relaxed);
      w[1] = DevAtomic(const_cast<unsigned long long&>(src[1])).load(cuda::memory_order_relaxed);
      memcpy(&s.v, w, sizeof(V));
      s.null = static_cast<uint32_t>((st >> 2) & 1);
    }
    // lane j + o holds earlier tiles than lane j
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const ScanState<V> other = shfl_state(s, o, 2);
      if (lane + o < 32) s = combine_state<Op>(other, s);
    }
    excl = combine_state<Op>(shfl_state(s, 0, 0), excl);
    if (incl_mask) return excl;
    back -= 32;
  }
}

template <typename T, int OP>
struct CumArgs {
  using Op = CumOp<T, OP>;
  using V = typename Op::V;
  const T* src;             // chunk values, offset applied
  BitmapReader valid;       // chunk validity
  int64_t len;              // chunk rows
  typename Op::Out* dst;    // output values at the chunk's first row
  unsigned long long* out_bits;  // output validity (whole output, offset 0), NULL when the output has none
  int64_t out_row0;         // the chunk's first row in the output
  int64_t n_total;          // output rows
  ScanCell* cells;          // this chunk's tiles
  unsigned long long* ticket;
  const ScanState<V>* carry_in;  // the previous chunk's inclusive state, NULL for the first chunk
  ScanState<V>* carry_out;
  V start;                  // the first chunk's carry
  bool skip_nulls;
  unsigned long long* slot;  // [0] overflow, [1] nulls (skip_nulls), [2] rows from the first null on (otherwise)
};

template <typename T, int OP>
__global__ void __launch_bounds__(kBlock) cumulative_kernel(CumArgs<T, OP> a) {
  using Op = CumOp<T, OP>;
  using V = typename Op::V;
  using Out = typename Op::Out;
  using S = ScanState<V>;
  constexpr int kElem = sizeof(T) > sizeof(Out) ? sizeof(T) : sizeof(Out);
  // per-warp staging, padded so that the transposed reads of 16 consecutive rows per lane hit distinct banks
  constexpr int kStage = kScanWarpRows + kScanWarpRows / 16;
  __shared__ alignas(16) unsigned char s_stage[kWarpsPerBlock][kStage * kElem];
  __shared__ S s_warp[kWarpsPerBlock];
  __shared__ unsigned long long s_ticket;

  const int lane = static_cast<int>(lane_id()), warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_ticket = atomicAdd(a.ticket, 1ull);
  __syncthreads();
  const int64_t tile = static_cast<int64_t>(s_ticket);
  const int64_t seg0 = tile * kScanTile + static_cast<int64_t>(warp) * kScanWarpRows;  // warp's first chunk row
  const int64_t row0 = seg0 + lane * kScanItems;                                       // lane's first chunk row
  const int cnt = static_cast<int>(a.len - row0 < 0 ? 0 : (a.len - row0 > kScanItems ? kScanItems : a.len - row0));

  // ---- load: striped global reads, transposed through shared memory ----
  const auto pad = [](int i, int elem) { return i + (elem == 8 ? i >> 4 : i >> 5); };
  T* stage_in = reinterpret_cast<T*>(s_stage[warp]);
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int i = k * 32 + lane;
    if (seg0 + i < a.len) stage_in[pad(i, sizeof(T))] = ld_stream(a.src + seg0 + i);
  }
  __syncwarp();
  T x[kScanItems];
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) x[k] = stage_in[pad(lane * kScanItems + k, sizeof(T))];
  __syncwarp();
  // the lane's 16 validity bits (bits at or past len read as 0, and those rows are out of range anyway)
  const uint64_t vw = a.valid.word(row0 >> 6);
  const uint32_t vbits = static_cast<uint32_t>(vw >> (row0 & 63)) & 0xffffu;

  // ---- lane aggregate, then warp and tile scans ----
  S agg{Op::identity(), 0};
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    if (k < cnt && !agg.null) {
      if ((vbits >> k) & 1) agg.v = Op::combine(agg.v, Op::lift(x[k]));
      else if (!a.skip_nulls) agg.null = 1;
    }
  }
  S incl = agg;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const S other = shfl_state(incl, o, 1);
    if (lane >= o) incl = combine_state<Op>(other, incl);
  }
  S lane_excl = shfl_state(incl, 1, 1);
  if (lane == 0) lane_excl = S{Op::identity(), 0};
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    // exclusive scan of the warp totals, then the tile's own exclusive prefix
    S wt = lane < kWarpsPerBlock ? s_warp[lane] : S{Op::identity(), 0};
#pragma unroll
    for (int o = 1; o < kWarpsPerBlock; o <<= 1) {
      const S other = shfl_state(wt, o, 1);
      if (lane >= o) wt = combine_state<Op>(other, wt);
    }
    const S tile_agg = shfl_state(wt, kWarpsPerBlock - 1, 0);
    S tile_excl;
    if (tile == 0) {
      tile_excl = a.carry_in ? *a.carry_in : S{a.start, 0};
    } else {
      if (lane == 0) publish(&a.cells[tile], false, tile_agg);
      tile_excl = look_back<Op, V>(a.cells, tile);
    }
    const S tile_incl = combine_state<Op>(tile_excl, tile_agg);
    if (lane == 0) {
      publish(&a.cells[tile], true, tile_incl);
      if (tile * kScanTile + kScanTile >= a.len) *a.carry_out = tile_incl;  // the chunk's last tile
    }
    S w_excl = shfl_state(wt, 1, 1);
    w_excl = lane == 0 ? tile_excl : combine_state<Op>(tile_excl, w_excl);
    __syncwarp();
    if (lane < kWarpsPerBlock) s_warp[lane] = w_excl;
  }
  __syncthreads();

  // ---- outputs: each lane re-folds its rows from its exclusive prefix ----
  S st = combine_state<Op>(s_warp[warp], lane_excl);
  Out y[kScanItems];
  uint32_t obits = 0;
  bool bad = false;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    y[k] = Out(0);
    if (k < cnt && !st.null) {
      if ((vbits >> k) & 1) {
        bad |= Op::overflows(st.v, x[k]);
        st.v = Op::combine(st.v, Op::lift(x[k]));
        y[k] = Op::output(st.v);
        obits |= 1u << k;
      } else if (!a.skip_nulls) {
        st.null = 1;
      }
    }
  }
  if (Op::kChecked && bad) a.slot[0] = 1;

  Out* stage_out = reinterpret_cast<Out*>(s_stage[warp]);
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) stage_out[pad(lane * kScanItems + k, sizeof(Out))] = y[k];
  __syncwarp();
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int i = k * 32 + lane;
    if (seg0 + i < a.len) st_stream(a.dst + seg0 + i, stage_out[pad(i, sizeof(Out))]);
  }

  if (a.out_bits) {
    // null accounting: the null count under skip_nulls, else the rows from the first null on
    const uint32_t in_range = cnt >= 32 ? 0xffffffffu : ((1u << cnt) - 1u);
    const uint32_t nulls = ~vbits & in_range;
    if (a.skip_nulls) {
      const unsigned c = __reduce_add_sync(0xffffffffu, __popc(nulls));
      if (lane == 0 && c) atomicAdd(&a.slot[1], static_cast<unsigned long long>(c));
    } else {
      unsigned long long tail = nulls ? static_cast<unsigned long long>(a.n_total - (a.out_row0 + row0 + __ffs(nulls) - 1)) : 0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long other = __shfl_down_sync(0xffffffffu, tail, o);
        tail = other > tail ? other : tail;
      }
      if (lane == 0 && tail) atomicMax(&a.slot[2], tail);
    }
    // four lanes make one 64-bit word of output validity
    const uint64_t b1 = __shfl_down_sync(0xffffffffu, obits, 1), b2 = __shfl_down_sync(0xffffffffu, obits, 2),
                   b3 = __shfl_down_sync(0xffffffffu, obits, 3);
    if ((lane & 3) == 0 && row0 < a.len) {
      const uint64_t word = obits | (b1 << 16) | (b2 << 32) | (b3 << 48);
      const int64_t pos = a.out_row0 + row0;
      const int sh = static_cast<int>(pos & 63);
      unsigned long long* w = a.out_bits + (pos >> 6);
      if (sh == 0) {
        *w = word;
      } else if (word) {
        atomicOr(w, static_cast<unsigned long long>(word << sh));
        if (word >> (64 - sh)) atomicOr(w + 1, static_cast<unsigned long long>(word >> (64 - sh)));
      }
    }
  }
}

static const char* cumulative_name(int op) {
  switch (op) {
    case B2_CUMULATIVE_SUM: return "cumulative_sum";
    case B2_CUMULATIVE_SUM_CHECKED: return "cumulative_sum_checked";
    case B2_CUMULATIVE_PROD: return "cumulative_prod";
    case B2_CUMULATIVE_PROD_CHECKED: return "cumulative_prod_checked";
    case B2_CUMULATIVE_MIN: return "cumulative_min";
    case B2_CUMULATIVE_MAX: return "cumulative_max";
    case B2_CUMULATIVE_MEAN: return "cumulative_mean";
    default: return nullptr;
  }
}

// the reference's default start (Identity<Op>): for floats, max is numeric_limits<T>::min(), the smallest positive
// normal, and min starts from the largest finite value
template <typename T, int OP>
T default_start() {
  if constexpr (OP == B2_CUMULATIVE_SUM || OP == B2_CUMULATIVE_SUM_CHECKED) return T(0);
  else if constexpr (OP == B2_CUMULATIVE_PROD || OP == B2_CUMULATIVE_PROD_CHECKED) return T(1);
  else if constexpr (OP == B2_CUMULATIVE_MIN) return std::numeric_limits<T>::max();
  else return std::numeric_limits<T>::min();
}

template <typename T, int OP>
int run_cumulative(B2Context* ctx, const B2Array* chunks, int32_t n_chunks, const B2Scalar* start, bool skip_nulls,
                   void* out_data, unsigned long long* out_bits, int64_t n_total, unsigned long long* slot,
                   cudaStream_t s) {
  using Op = CumOp<T, OP>;
  using V = typename Op::V;
  using S = ScanState<V>;
  int64_t tiles = 0;
  for (int32_t c = 0; c < n_chunks; ++c) tiles += (chunks[c].length + kScanTile - 1) / kScanTile;
  // cells of every chunk's tiles, one ticket per chunk, two carries used in turn: one allocation, one memset
  const size_t cell_bytes = static_cast<size_t>(tiles) * sizeof(ScanCell);
  const size_t bytes = cell_bytes + static_cast<size_t>(n_chunks) * 8 + 2 * sizeof(S);
  Temp scratch(ctx, s);
  B2_RETURN_NOT_OK(scratch.alloc(bytes));
  B2_CUDA(cudaMemsetAsync(scratch.ptr, 0, cell_bytes + static_cast<size_t>(n_chunks) * 8, s));
  ScanCell* cells = scratch.as<ScanCell>();
  unsigned long long* tickets = reinterpret_cast<unsigned long long*>(static_cast<char*>(scratch.ptr) + cell_bytes);
  S* carries = reinterpret_cast<S*>(tickets + n_chunks);
  V v0;
  if constexpr (Op::kMean) {
    v0 = Op::identity();
  } else {
    v0 = start ? scalar_bits<T>(start) : default_start<T, OP>();
  }
  const S* carry_in = nullptr;
  int64_t row = 0;
  for (int32_t c = 0; c < n_chunks; ++c) {
    const B2Array& in = chunks[c];
    if (in.length == 0) continue;
    CumArgs<T, OP> a;
    a.src = static_cast<const T*>(in.data) + in.offset;
    a.valid = (in.validity && in.null_count != 0) ? BitmapReader(in.validity, in.offset, in.length)
                                                  : BitmapReader(nullptr, 0, in.length);
    a.len = in.length;
    a.dst = static_cast<typename Op::Out*>(out_data) + row;
    a.out_bits = out_bits;
    a.out_row0 = row;
    a.n_total = n_total;
    a.cells = cells;
    a.ticket = tickets + c;
    a.carry_in = carry_in;
    a.carry_out = carries + (carry_in == carries ? 1 : 0);
    a.start = v0;
    a.skip_nulls = skip_nulls;
    a.slot = slot;
    const int64_t chunk_tiles = (in.length + kScanTile - 1) / kScanTile;
    cumulative_kernel<T, OP><<<static_cast<unsigned>(chunk_tiles), kBlock, 0, s>>>(a);
    B2_LAUNCHED();
    cells += chunk_tiles;
    carry_in = a.carry_out;
    row += in.length;
  }
  return B2_OK;
}

}  // namespace b2

using namespace b2;

extern "C" int b2_cumulative(B2Context* ctx, int op, const B2Array* chunks, int32_t n_chunks, const B2Scalar* start,
                             int skip_nulls, B2Array* out, void* stream) {
  if (!ctx || !out || (n_chunks > 0 && !chunks)) return set_error(B2_INVALID, "b2_cumulative: null argument");
  const char* name = cumulative_name(op);
  if (!name) return set_error(B2_INVALID, "unknown cumulative op %d", op);
  if (n_chunks < 1) return set_error(B2_INVALID, "b2_cumulative: at least one chunk is required");
  const int type = chunks[0].type;
  int64_t n = 0;
  bool has_nulls = false;
  for (int32_t c = 0; c < n_chunks; ++c) {
    if (chunks[c].type != type) return set_error(B2_TYPE_ERROR, "b2_cumulative: chunks of different types");
    if (chunks[c].length < 0 || chunks[c].offset < 0) return set_error(B2_INVALID, "negative length/offset");
    n += chunks[c].length;
    has_nulls |= chunks[c].validity != nullptr && chunks[c].null_count != 0 && chunks[c].length > 0;
  }
  if (!type_is_numeric(type))
    return set_error(B2_NOT_IMPLEMENTED, "Function '%s' has no kernel matching input types (%s)", name,
                     type_name(type));
  if (start && op != B2_CUMULATIVE_MEAN && start->type != type)
    return set_error(B2_TYPE_ERROR, "b2_cumulative: start must have the input's type");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int out_type = op == B2_CUMULATIVE_MEAN ? B2_DOUBLE : type;

  Temp data(ctx, s);
  B2_RETURN_NOT_OK(data.alloc(static_cast<size_t>(n) * type_width(out_type)));
  if (n == 0) {
    fill_out(out, out_type, 0, 0, nullptr, data.release());
    return B2_OK;
  }
  Temp bits(ctx, s);
  if (has_nulls) {
    B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(n)));
    // a chunk that starts inside a word ORs into it; a single chunk stores every word
    if (n_chunks > 1) B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bitmap_alloc_bytes(n), s));
  }
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  unsigned long long* cell = reinterpret_cast<unsigned long long*>(slot.dev());
  B2_RETURN_NOT_OK(visit_type(NumericTypes{}, type, [&](auto tag) -> int {
    using T = decltype(tag);
    const auto run = [&](auto oc) -> int {
      return run_cumulative<T, decltype(oc)::value>(ctx, chunks, n_chunks, start, skip_nulls != 0, data.ptr,
                                                    bits.as<unsigned long long>(), n, cell, s);
    };
    if constexpr (std::is_floating_point<T>::value) {
      // float checked ops never raise: they run the unchecked kernels
      const int o = op == B2_CUMULATIVE_SUM_CHECKED ? B2_CUMULATIVE_SUM
                    : op == B2_CUMULATIVE_PROD_CHECKED ? B2_CUMULATIVE_PROD : op;
      return visit_width<B2_CUMULATIVE_SUM, B2_CUMULATIVE_PROD, B2_CUMULATIVE_MIN, B2_CUMULATIVE_MAX,
                         B2_CUMULATIVE_MEAN>(o, run);
    } else {
      return visit_width<B2_CUMULATIVE_SUM, B2_CUMULATIVE_SUM_CHECKED, B2_CUMULATIVE_PROD, B2_CUMULATIVE_PROD_CHECKED,
                         B2_CUMULATIVE_MIN, B2_CUMULATIVE_MAX, B2_CUMULATIVE_MEAN>(op, run);
    }
  }));
  B2_RETURN_NOT_OK(slot.fetch(s));
  if (slot.host()[0] != 0) return set_error(B2_INVALID, "overflow");
  const int64_t null_count = has_nulls ? slot.host()[skip_nulls ? 1 : 2] : 0;
  fill_out(out, out_type, n, null_count, null_count ? bits.release() : nullptr, data.release());
  return B2_OK;
}
