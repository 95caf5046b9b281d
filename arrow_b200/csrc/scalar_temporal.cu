// scalar_temporal.cu -- casts between temporal types, and calendar / clock fields.
//
// Replaces kernels/scalar_cast_temporal.cc (ShiftTime, the Date32 / Date64 / ExtractTime* functors and the zero-copy
// relabels) and the field extractors of kernels/scalar_temporal_unary.cc:222-691, for date32, date64, time32, time64,
// timestamp (naive, UTC or a fixed offset) and duration, every unit.
//
// Both entry points are one streaming pass over int32 / int64 storage (elementwise.cuh's map1_kernel; is_leap_year
// writes one ballot word per 32 rows).  The unit, the field and every divisor are template parameters, so each
// division is by a compile-time constant and none calls the generic 64-bit division routine.
//
// Exactness at full range: the reference computes dates through the vendored date library, whose day count is a 32-bit
// int and whose year is a 16-bit short.  floor<days>(t) truncates t / day to int32 and then steps back one day when that
// day, scaled back to t's unit in wrapping int64, lies after t; civil-from-days then runs in wrapping 32-bit arithmetic.
// The functions below restate those steps (not the library's code), so far-out values wrap to the reference's answers.
//
// Roofline: HBM-bound stream, algorithmic bytes/row = sizeof(In) + sizeof(Out) + 2/8 with a validity bitmap
// (int64 field of a timestamp: 16.25 B/row).
#include <limits>
#include <string>
#include <type_traits>

#include "bitmap.h"
#include "elementwise.cuh"

namespace b2 {

constexpr int kDays = 4;  // "unit" of date32: the value is a day count

__host__ __device__ constexpr int64_t per_second(int unit) {
  return unit == B2_SECOND ? 1 : unit == B2_MILLI ? 1000 : unit == B2_MICRO ? 1000000 : 1000000000;
}
__host__ __device__ constexpr int64_t per_day(int unit) { return 86400 * per_second(unit); }

// two's-complement arithmetic, as the reference's overflowing int / int64 expressions behave on x86-64
__host__ __device__ __forceinline__ int64_t wrap_add(int64_t a, int64_t b) {
  return static_cast<int64_t>(static_cast<uint64_t>(a) + static_cast<uint64_t>(b));
}
__host__ __device__ __forceinline__ int64_t wrap_sub(int64_t a, int64_t b) {
  return static_cast<int64_t>(static_cast<uint64_t>(a) - static_cast<uint64_t>(b));
}
__host__ __device__ __forceinline__ int64_t wrap_mul(int64_t a, int64_t b) {
  return static_cast<int64_t>(static_cast<uint64_t>(a) * static_cast<uint64_t>(b));
}
__host__ __device__ __forceinline__ int32_t narrow32(int64_t v) {
  return static_cast<int32_t>(static_cast<uint32_t>(static_cast<uint64_t>(v)));
}

template <int64_t D>
__host__ __device__ __forceinline__ int64_t floor_mod(int64_t x) {
  const int64_t r = x % D;
  return r < 0 ? r + D : r;
}

// the day count floor<days>(t) of a time point t counted in units of which PER_DAY make a day, as the reference's
// compiled code yields it: the narrowed quotient, less one without narrowing again (the time-of-day paths see
// INT32_MIN - 1 as such; the day-count paths narrow it)
template <int64_t PER_DAY>
__host__ __device__ __forceinline__ int64_t floor_days(int64_t t) {
  const int64_t d = narrow32(t / PER_DAY);
  return wrap_mul(d, PER_DAY) > t ? d - 1 : d;
}

struct Civil {
  int32_t year;    // the 16-bit year, sign-extended
  uint32_t month;  // 8-bit fields: a wrapped day count can give any byte
  uint32_t day;
};

// civil-from-days (H. Hinnant's public-domain algorithm) over a 32-bit day count, every step wrapping as 32-bit
// int / unsigned arithmetic does
__host__ __device__ __forceinline__ Civil civil_from_days(int32_t days) {
  const int32_t z = static_cast<int32_t>(static_cast<uint32_t>(days) + 719468u);
  const int32_t era = (z >= 0 ? z : static_cast<int32_t>(static_cast<uint32_t>(z) - 146096u)) / 146097;
  const uint32_t doe = static_cast<uint32_t>(z) - static_cast<uint32_t>(era) * 146097u;
  const uint32_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  const uint32_t y = yoe + static_cast<uint32_t>(era) * 400u;
  const uint32_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const uint32_t mp = (5 * doy + 2) / 153;
  const uint32_t d = doy - (153 * mp + 2) / 5 + 1;
  const uint32_t m = mp < 10 ? mp + 3 : mp - 9;
  return {static_cast<int16_t>(static_cast<uint16_t>(y + (m <= 2 ? 1u : 0u))), m & 0xffu, d & 0xffu};
}

// the day count of year/jan/0 (December 31 of the year before), days-from-civil over the 16-bit year
__host__ __device__ __forceinline__ int32_t days_before_year(int32_t year) {
  const int32_t y = year - 1;
  const int32_t era = (y >= 0 ? y : y - 399) / 400;
  const uint32_t yoe = static_cast<uint32_t>(y - era * 400);
  const uint32_t doe = yoe * 365 + yoe / 4 - yoe / 100 + 305u;  // day-of-era of March 1 + 305 = Dec 31 ... Jan 0
  return static_cast<int32_t>(static_cast<uint32_t>(era) * 146097u + doe - 719468u);
}

// 0 = Sunday .. 6 = Saturday of a 32-bit day count
__host__ __device__ __forceinline__ uint32_t weekday_of(int32_t z) {
  const uint32_t u = static_cast<uint32_t>(z);
  return z >= -4 ? (u + 4) % 7 : u % 7;
}

// day count of value x (local time already applied)
template <int U>
__host__ __device__ __forceinline__ int32_t day_count(int64_t x) {
  if constexpr (U == kDays) {
    return static_cast<int32_t>(x);
  } else {
    return narrow32(floor_days<per_day(U)>(x));
  }
}

// day_of_week's answer for each weekday (0 = Sunday .. 6 = Saturday), 4 bits each: DayOfWeek's lookup table
// (scalar_temporal_unary.cc:408-429) indexed by the ISO weekday
inline uint32_t day_of_week_table(int week_start, int count_from_zero) {
  uint32_t table = 0;
  for (int wd = 0; wd < 7; ++wd) {
    const int iso = wd == 0 ? 7 : wd;
    int v = iso - 1 + 8 - week_start;
    v = v > 6 ? v - 7 : v;
    table |= static_cast<uint32_t>(v + (count_from_zero ? 0 : 1)) << (4 * wd);
  }
  return table;
}

// One field of one value.  shift = the zone's offset in the value's unit (0 for naive, UTC and non-timestamps); the
// date fields, hour and minute read local time, the finer fields do not (an offset is a whole number of minutes).
template <int F, int U>
__host__ __device__ __forceinline__ int64_t field_int(int64_t x, int64_t shift, uint32_t dow_table) {
  if constexpr (F <= B2_FIELD_IS_LEAP_YEAR) {
    const int32_t d = day_count<U>(wrap_add(x, shift));
    if constexpr (F == B2_FIELD_DAY_OF_WEEK) {
      return (dow_table >> (4 * weekday_of(d))) & 0xfu;
    } else {
      const Civil c = civil_from_days(d);
      if constexpr (F == B2_FIELD_YEAR) return c.year;
      if constexpr (F == B2_FIELD_MONTH) return c.month;
      if constexpr (F == B2_FIELD_DAY) return c.day;
      if constexpr (F == B2_FIELD_QUARTER) return (c.month - 1) / 3 + 1;
      if constexpr (F == B2_FIELD_DAY_OF_YEAR)
        return static_cast<int32_t>(static_cast<uint32_t>(d) - static_cast<uint32_t>(days_before_year(c.year)));
      if constexpr (F == B2_FIELD_IS_LEAP_YEAR) return c.year % 4 == 0 && (c.year % 100 != 0 || c.year % 400 == 0);
    }
  } else if constexpr (U == kDays) {
    return 0;  // no clock field on date32: refused on the host
  } else {
    constexpr int64_t S = per_second(U);
    if constexpr (F == B2_FIELD_HOUR) {
      const int64_t t = wrap_add(x, shift);
      return wrap_sub(t, wrap_mul(floor_days<per_day(U)>(t), per_day(U))) / (3600 * S);
    }
    if constexpr (F == B2_FIELD_MINUTE) return floor_mod<3600 * S>(wrap_add(x, shift)) / (60 * S);
    if constexpr (F == B2_FIELD_SECOND) return floor_mod<60 * S>(x) / S;
    const int64_t sub = floor_mod<S>(x);  // units past the second
    if constexpr (F == B2_FIELD_MILLISECOND) return U >= B2_MILLI ? sub / (S / 1000) % 1000 : 0;
    if constexpr (F == B2_FIELD_MICROSECOND) return U >= B2_MICRO ? sub / (S / 1000000) % 1000 : 0;
    if constexpr (F == B2_FIELD_NANOSECOND) return U == B2_NANO ? sub % 1000 : 0;
  }
  return 0;
}

template <typename In, typename Out, int F, int U>
struct FieldOp {
  int64_t shift;
  uint32_t dow_table;
  __device__ __forceinline__ Out operator()(In x, int64_t) const {
    if constexpr (F == B2_FIELD_SUBSECOND) {
      constexpr int64_t S = U == kDays ? 1 : per_second(U);
      return static_cast<double>(floor_mod<S>(x)) / static_cast<double>(S);  // duration<double> of the remainder
    } else {
      return field_int<F, U>(x, shift, dow_table);
    }
  }
};

// is_leap_year: lane l of a warp evaluates row 32w + l and lane 0 stores the ballot as output word w; the words past
// the last row (up to the allocation's end) are stored as zero.
template <typename In, int U>
__global__ void __launch_bounds__(kBlock) leap_year_kernel(const In* __restrict__ in, uint32_t* __restrict__ out,
                                                           int64_t n, int64_t n_words, int64_t shift) {
  const unsigned lane = lane_id();
  const int64_t warps = static_cast<int64_t>(gridDim.x) * kWarpsPerBlock;
  for (int64_t w = static_cast<int64_t>(blockIdx.x) * kWarpsPerBlock + (threadIdx.x >> 5); w < n_words; w += warps) {
    const int64_t i = w * 32 + lane;
    const bool leap = i < n && field_int<B2_FIELD_IS_LEAP_YEAR, U>(__ldcs(in + i), shift, 0) != 0;
    const uint32_t bits = __ballot_sync(0xffffffffu, leap);
    if (lane == 0) __stcs(out + w, bits);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// casts
// ---------------------------------------------------------------------------------------------------------------

// ShiftTime: out = in * F or in / F (F = 1: a copy).  checked: a multiply whose result leaves int64, or a division
// with a remainder, reports its row if the row is valid.
template <typename In, typename Out, bool MUL, int64_t F, bool CHECK>
struct ShiftOp {
  BitmapReader valid;
  ErrorCell err;
  __device__ __forceinline__ Out operator()(In x, int64_t i) const {
    const int64_t v = x;
    if constexpr (MUL) {
      if constexpr (CHECK) {
        constexpr int64_t lo = std::numeric_limits<int64_t>::min() / F, hi = std::numeric_limits<int64_t>::max() / F;
        if ((v < lo || v > hi) && valid.bit(i)) err.report(i);
      }
      return static_cast<Out>(wrap_mul(v, F));
    } else {
      const Out y = static_cast<Out>(v / F);
      if constexpr (CHECK) {
        if (wrap_mul(static_cast<int64_t>(y), F) != v && valid.bit(i)) err.report(i);
      }
      return y;
    }
  }
};

// timestamp (unit FROM) -> date32 / date64 of its local day
template <int FROM, bool DATE64>
struct TsDateOp {
  int64_t shift;
  __device__ __forceinline__ typename std::conditional<DATE64, int64_t, int32_t>::type operator()(int64_t x,
                                                                                               int64_t) const {
    const int64_t d = floor_days<per_day(FROM)>(wrap_add(x, shift));
    if constexpr (DATE64) {
      // the step back from INT32_MIN stays unnarrowed here too, except from seconds (the reference's compiled code
      // differs by unit)
      return (FROM == B2_SECOND ? static_cast<int64_t>(narrow32(d)) : d) * 86400000;
    } else {
      return narrow32(d);
    }
  }
};

// the time of day of a timestamp in its own unit (local time), as (t - floor<days>(t)) wraps in the reference
template <int FROM>
__host__ __device__ __forceinline__ int64_t time_of_day(int64_t x, int64_t shift) {
  const int64_t t = wrap_add(x, shift);
  return wrap_sub(t, wrap_mul(floor_days<per_day(FROM)>(t), per_day(FROM)));
}

__host__ __device__ constexpr int64_t unit_ratio(int a, int b) { return per_second(a) / per_second(b); }

// timestamp (unit FROM) -> time32 / time64 (unit TO) of its local time of day
// (the reference's extraction sets the status at every offending row and keeps going, so the last one is named)
template <int FROM, int TO, bool CHECK>
struct TsTimeOp {
  using Out = typename std::conditional<(TO <= B2_MILLI), int32_t, int64_t>::type;
  int64_t shift;
  BitmapReader valid;
  LastErrorCell err;
  __device__ __forceinline__ Out operator()(int64_t x, int64_t i) const {
    const int64_t tod = time_of_day<FROM>(x, shift);
    if constexpr (TO >= FROM) {
      return static_cast<Out>(wrap_mul(tod, unit_ratio(TO, FROM)));
    } else {
      constexpr int64_t F = unit_ratio(FROM, TO);
      const Out y = static_cast<Out>(tod / F);
      if (CHECK && wrap_mul(static_cast<int64_t>(y), F) != tod && valid.bit(i)) err.report(i);
      return y;
    }
  }
};

// two 16-byte accesses in flight per lane: with kUnroll the 64-bit constant divisions of the field and cast ops spill
constexpr int kTemporalUnroll = 2;

template <typename In, typename Out, typename Op>
static int launch_map(const B2Array* in, void* out_data, const Op& op, cudaStream_t s) {
  constexpr int V = vec_elems<In, Out>();
  const In* src = static_cast<const In*>(in->data) + in->offset;
  Out* dst = static_cast<Out*>(out_data);
  const bool vec_ok = aligned_to(src, sizeof(In) * V) && aligned_to(dst, sizeof(Out) * V);
  map1_kernel<In, Out, V, Op, kTemporalUnroll>
      <<<map_grid<In, Out, V>(in->length), kBlock, 0, s>>>(src, dst, in->length, vec_ok, op);
  B2_LAUNCHED();
  return B2_OK;
}

static bool is_32bit(int kind) {
  return kind == B2_TEMPORAL_DATE32 || kind == B2_TEMPORAL_TIME32 || kind == B2_TEMPORAL_INT32;
}
static int storage_of(int kind) { return is_32bit(kind) ? B2_INT32 : B2_INT64; }
static bool has_unit(int kind) {
  return kind == B2_TEMPORAL_TIME32 || kind == B2_TEMPORAL_TIME64 || kind == B2_TEMPORAL_TIMESTAMP ||
         kind == B2_TEMPORAL_DURATION;
}

static int check_type(const B2TemporalType* t, const char* what) {
  if (!t) return set_error(B2_INVALID, "%s: null temporal type", what);
  if (t->kind < B2_TEMPORAL_DATE32 || t->kind > B2_TEMPORAL_INT64)
    return set_error(B2_INVALID, "%s: unknown temporal kind %d", what, t->kind);
  if (has_unit(t->kind)) {
    const int lo = t->kind == B2_TEMPORAL_TIME64 ? B2_MICRO : B2_SECOND;
    const int hi = t->kind == B2_TEMPORAL_TIME32 ? B2_MILLI : B2_NANO;
    if (t->unit < lo || t->unit > hi) return set_error(B2_INVALID, "%s: invalid unit %d for kind %d", what, t->unit, t->kind);
  }
  if (t->has_zone && (t->kind != B2_TEMPORAL_TIMESTAMP || t->offset_minutes < -(23 * 60 + 59) ||
                      t->offset_minutes > 23 * 60 + 59))
    return set_error(B2_INVALID, "%s: invalid zone", what);
  return B2_OK;
}

static const char* const kUnitNames[] = {"s", "ms", "us", "ns"};
static const char* const kKindNames[] = {"date32", "date64", "time32", "time64", "timestamp", "duration", "int32", "int64"};

// DataType::ToString; a zone is written from its offset
static std::string temporal_name(const B2TemporalType& t) {
  std::string s = kKindNames[t.kind];
  switch (t.kind) {
    case B2_TEMPORAL_DATE32: return s + "[day]";
    case B2_TEMPORAL_DATE64: return s + "[ms]";
    case B2_TEMPORAL_INT32:
    case B2_TEMPORAL_INT64: return s;
    default: break;
  }
  s += std::string("[") + kUnitNames[t.unit];
  if (t.kind == B2_TEMPORAL_TIMESTAMP && t.has_zone) {
    if (t.offset_minutes == 0) {
      s += ", tz=UTC";
    } else {
      const int m = t.offset_minutes < 0 ? -t.offset_minutes : t.offset_minutes;
      char b[16];
      snprintf(b, sizeof(b), "%c%02d:%02d", t.offset_minutes < 0 ? '-' : '+', m / 60, m % 60);
      s += std::string(", tz=") + b;
    }
  }
  return s + "]";
}

static int64_t zone_shift(const B2TemporalType& t) {
  return t.kind == B2_TEMPORAL_TIMESTAMP && t.has_zone ? static_cast<int64_t>(t.offset_minutes) * 60 * per_second(t.unit)
                                                       : 0;
}

template <int... Us, typename F>
static int visit_unit(int u, F&& f) {
  return visit_width<Us...>(u, f);
}

// the int64 constant factors a ShiftTime of the reference can use
template <typename F>
static int visit_factor(int64_t factor, F&& f) {
  int st = B2_OK;
  const auto one = [&](auto c) {
    if (factor != decltype(c)::value) return false;
    st = f(c);
    return true;
  };
  const bool hit = one(std::integral_constant<int64_t, 1>{}) || one(std::integral_constant<int64_t, 1000>{}) ||
                   one(std::integral_constant<int64_t, 1000000>{}) || one(std::integral_constant<int64_t, 1000000000>{}) ||
                   one(std::integral_constant<int64_t, 86400>{}) || one(std::integral_constant<int64_t, 86400000>{}) ||
                   one(std::integral_constant<int64_t, 86400000000>{}) ||
                   one(std::integral_constant<int64_t, 86400000000000>{});
  return hit ? st : set_error(B2_UNKNOWN_ERROR, "no cast kernel for factor %lld", static_cast<long long>(factor));
}

// How a cast runs: a ShiftTime with a factor, or one of the two timestamp extractions
struct CastPlan {
  enum Kind { kNone, kShift, kTsDate, kTsTime } kind = kNone;
  bool mul = true;
  int64_t factor = 1;
};

static CastPlan plan_cast(const B2TemporalType& f, const B2TemporalType& t) {
  CastPlan p;
  const auto shift = [&p](bool mul, int64_t factor) {
    p.kind = CastPlan::kShift;
    p.mul = mul;
    p.factor = factor;
  };
  // GetTimestampConversion: finer target multiplies, coarser divides
  const auto convert = [&](int from_unit, int to_unit) {
    if (to_unit >= from_unit) {
      shift(true, unit_ratio(to_unit, from_unit));
    } else {
      shift(false, unit_ratio(from_unit, to_unit));
    }
  };
  const int a = f.kind, b = t.kind;
  const bool same = a == b && (!has_unit(a) || f.unit == t.unit);
  const bool relabel = (a == B2_TEMPORAL_INT32 && (b == B2_TEMPORAL_DATE32 || b == B2_TEMPORAL_TIME32)) ||
                       ((a == B2_TEMPORAL_DATE32 || a == B2_TEMPORAL_TIME32) && b == B2_TEMPORAL_INT32) ||
                       (a == B2_TEMPORAL_INT64 && b != B2_TEMPORAL_INT64 && !is_32bit(b)) ||
                       (b == B2_TEMPORAL_INT64 && a != B2_TEMPORAL_INT64 && !is_32bit(a));
  if (same || relabel) {
    shift(true, 1);
  } else if ((a == B2_TEMPORAL_TIMESTAMP && b == B2_TEMPORAL_TIMESTAMP) ||
             (a == B2_TEMPORAL_DURATION && b == B2_TEMPORAL_DURATION) ||
             ((a == B2_TEMPORAL_TIME32 || a == B2_TEMPORAL_TIME64) &&
              (b == B2_TEMPORAL_TIME32 || b == B2_TEMPORAL_TIME64))) {
    convert(f.unit, t.unit);
  } else if (a == B2_TEMPORAL_DATE32 && b == B2_TEMPORAL_DATE64) {
    shift(true, 86400000);
  } else if (a == B2_TEMPORAL_DATE64 && b == B2_TEMPORAL_DATE32) {
    shift(false, 86400000);
  } else if (a == B2_TEMPORAL_DATE32 && b == B2_TEMPORAL_TIMESTAMP) {
    shift(true, per_day(t.unit));
  } else if (a == B2_TEMPORAL_DATE64 && b == B2_TEMPORAL_TIMESTAMP) {
    convert(B2_MILLI, t.unit);
  } else if (a == B2_TEMPORAL_TIMESTAMP && (b == B2_TEMPORAL_DATE32 || b == B2_TEMPORAL_DATE64)) {
    p.kind = CastPlan::kTsDate;
  } else if (a == B2_TEMPORAL_TIMESTAMP && (b == B2_TEMPORAL_TIME32 || b == B2_TEMPORAL_TIME64)) {
    p.kind = CastPlan::kTsTime;
    p.mul = t.unit >= f.unit;
  }
  return p;
}

// true when some value of In leaves int64 when multiplied by factor
template <typename In>
static bool can_overflow(int64_t factor) {
  return static_cast<__int128>(std::numeric_limits<In>::max()) * factor > std::numeric_limits<int64_t>::max() ||
         static_cast<__int128>(std::numeric_limits<In>::min()) * factor < std::numeric_limits<int64_t>::min();
}

static int64_t time_of_day_host(int64_t x, int unit, int64_t shift) {
  switch (unit) {
    case B2_SECOND: return time_of_day<B2_SECOND>(x, shift);
    case B2_MILLI: return time_of_day<B2_MILLI>(x, shift);
    case B2_MICRO: return time_of_day<B2_MICRO>(x, shift);
    default: return time_of_day<B2_NANO>(x, shift);
  }
}

}  // namespace b2

using namespace b2;

extern "C" int b2_cast_temporal(B2Context* ctx, const B2Array* in, const B2TemporalType* from,
                                const B2TemporalType* to, int allow_time_truncate, int allow_time_overflow,
                                B2Array* out, void* stream) {
  if (!ctx || !in || !out) return set_error(B2_INVALID, "b2_cast_temporal: null argument");
  B2_RETURN_NOT_OK(check_type(from, "b2_cast_temporal from"));
  B2_RETURN_NOT_OK(check_type(to, "b2_cast_temporal to"));
  if (in->length < 0 || in->offset < 0) return set_error(B2_INVALID, "negative length/offset");
  if (in->type != storage_of(from->kind))
    return set_error(B2_TYPE_ERROR, "b2_cast_temporal: storage type id %d does not hold %s", in->type,
                     temporal_name(*from).c_str());
  const CastPlan plan = plan_cast(*from, *to);
  if (plan.kind == CastPlan::kNone)
    return set_error(B2_NOT_IMPLEMENTED, "Unsupported cast from %s to %s using function cast_%s",
                     temporal_name(*from).c_str(), kKindNames[to->kind], kKindNames[to->kind]);
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = in->length;
  const int out_type = storage_of(to->kind);

  Temp data(ctx, s);
  B2_RETURN_NOT_OK(data.alloc(static_cast<size_t>(n) * type_width(out_type)));
  void* validity = nullptr;
  int64_t null_count = 0;
  B2_RETURN_NOT_OK(make_validity(ctx, in, nullptr, n, &validity, &null_count, s));
  Temp vguard(ctx, s);
  vguard.ptr = validity;
  if (n == 0) {
    fill_out(out, out_type, 0, 0, vguard.release(), data.release());
    return B2_OK;
  }

  const bool in32 = in->type == B2_INT32;
  const BitmapReader valid(in->null_count == 0 ? nullptr : in->validity, in->offset, n);
  bool checked = false;
  if (plan.kind == CastPlan::kShift && plan.factor != 1) {
    checked = plan.mul ? !allow_time_overflow && (in32 ? can_overflow<int32_t>(plan.factor) : can_overflow<int64_t>(plan.factor))
                       : !allow_time_truncate;
  } else if (plan.kind == CastPlan::kTsTime) {
    checked = !plan.mul && !allow_time_truncate;
  }
  ScalarSlot slot(ctx);
  ErrorCell err{nullptr};            // ShiftTime stops at the first offending row
  LastErrorCell last_err{nullptr};   // timestamp -> time names the last
  if (checked) {
    if (!slot.ok()) return set_error(B2_UNKNOWN_ERROR, "no free scalar slot");
    B2_CUDA(cudaMemsetAsync(slot.dev(), plan.kind == CastPlan::kTsTime ? 0 : 0xff, 8, s));
    err.first_row = reinterpret_cast<unsigned long long*>(slot.dev());
    last_err.last_row1 = err.first_row;
  }
  const int64_t shift = zone_shift(*from);

  int st;
  if (plan.kind == CastPlan::kShift) {
    st = visit_factor(plan.factor, [&](auto fc) -> int {
      constexpr int64_t F = decltype(fc)::value;
      const auto run = [&](auto in_tag, auto out_tag) -> int {
        using In = decltype(in_tag);
        using Out = decltype(out_tag);
        if (plan.mul) {
          if (checked) return launch_map<In, Out>(in, data.ptr, ShiftOp<In, Out, true, F, true>{valid, err}, s);
          return launch_map<In, Out>(in, data.ptr, ShiftOp<In, Out, true, F, false>{valid, err}, s);
        }
        if (checked) return launch_map<In, Out>(in, data.ptr, ShiftOp<In, Out, false, F, true>{valid, err}, s);
        return launch_map<In, Out>(in, data.ptr, ShiftOp<In, Out, false, F, false>{valid, err}, s);
      };
      // the storage pairs and factors the plans use: time32 changes units by 1000 only, and only date64 -> date32
      // and time64 -> time32 narrow
      if (in32 && out_type == B2_INT32) {
        if constexpr (F == 1 || F == 1000) return run(int32_t{}, int32_t{});
      } else if (in32) {
        return run(int32_t{}, int64_t{});
      } else if (out_type == B2_INT32) {
        if constexpr (F == 1 || F == 1000 || F == 1000000 || F == 1000000000 || F == 86400000)
          return run(int64_t{}, int32_t{});
      } else {
        return run(int64_t{}, int64_t{});
      }
      return set_error(B2_UNKNOWN_ERROR, "no cast kernel for this storage pair and factor");
    });
  } else if (plan.kind == CastPlan::kTsDate) {
    st = visit_unit<B2_SECOND, B2_MILLI, B2_MICRO, B2_NANO>(from->unit, [&](auto uc) -> int {
      constexpr int U = decltype(uc)::value;
      if (to->kind == B2_TEMPORAL_DATE64) return launch_map<int64_t, int64_t>(in, data.ptr, TsDateOp<U, true>{shift}, s);
      return launch_map<int64_t, int32_t>(in, data.ptr, TsDateOp<U, false>{shift}, s);
    });
  } else {
    st = visit_unit<B2_SECOND, B2_MILLI, B2_MICRO, B2_NANO>(from->unit, [&](auto fu) -> int {
      return visit_unit<B2_SECOND, B2_MILLI, B2_MICRO, B2_NANO>(to->unit, [&](auto tu) -> int {
        constexpr int FU = decltype(fu)::value, TU = decltype(tu)::value;
        using Out = typename TsTimeOp<FU, TU, false>::Out;
        if (checked) return launch_map<int64_t, Out>(in, data.ptr, TsTimeOp<FU, TU, true>{shift, valid, last_err}, s);
        return launch_map<int64_t, Out>(in, data.ptr, TsTimeOp<FU, TU, false>{shift, valid, last_err}, s);
      });
    });
  }
  B2_RETURN_NOT_OK(st);

  if (checked) {
    B2_RETURN_NOT_OK(slot.fetch(s));
    uint64_t row = static_cast<uint64_t>(slot.host()[0]);
    if (plan.kind == CastPlan::kTsTime) row = row == 0 ? ~0ull : row - 1;
    if (row != ~0ull) {
      int64_t bad = 0;
      if (in32) {
        int32_t v;
        B2_CUDA(cudaMemcpyAsync(&v, static_cast<const int32_t*>(in->data) + in->offset + row, 4,
                                cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaStreamSynchronize(s));
        bad = v;
      } else {
        B2_CUDA(cudaMemcpyAsync(&bad, static_cast<const int64_t*>(in->data) + in->offset + row, 8,
                                cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaStreamSynchronize(s));
      }
      if (plan.kind == CastPlan::kTsTime)
        return set_error(B2_INVALID, "Cast would lose data: %lld",
                         static_cast<long long>(time_of_day_host(bad, from->unit, shift)));
      return set_error(B2_INVALID, "Casting from %s to %s would %s: %lld", temporal_name(*from).c_str(),
                       temporal_name(*to).c_str(), plan.mul ? "result in out of bounds timestamp" : "lose data",
                       static_cast<long long>(bad));
    }
  }
  fill_out(out, out_type, n, null_count, vguard.release(), data.release());
  return B2_OK;
}

static const char* const kFieldNames[] = {"year", "month", "day", "day_of_year", "day_of_week",
                                          "quarter", "is_leap_year", "hour", "minute", "second",
                                          "millisecond", "microsecond", "nanosecond", "subsecond"};

extern "C" int b2_temporal_field(B2Context* ctx, const B2Array* in, const B2TemporalType* type, int field,
                                 int week_start, int count_from_zero, B2Array* out, void* stream) {
  if (!ctx || !in || !out) return set_error(B2_INVALID, "b2_temporal_field: null argument");
  B2_RETURN_NOT_OK(check_type(type, "b2_temporal_field"));
  if (field < B2_FIELD_YEAR || field > B2_FIELD_SUBSECOND) return set_error(B2_INVALID, "unknown temporal field %d", field);
  if (in->length < 0 || in->offset < 0) return set_error(B2_INVALID, "negative length/offset");
  if (in->type != storage_of(type->kind))
    return set_error(B2_TYPE_ERROR, "b2_temporal_field: storage type id %d does not hold %s", in->type,
                     temporal_name(*type).c_str());
  const int k = type->kind;
  const bool date_field = field <= B2_FIELD_IS_LEAP_YEAR;
  const bool ok = k == B2_TEMPORAL_TIMESTAMP ||
                  (date_field ? (k == B2_TEMPORAL_DATE32 || k == B2_TEMPORAL_DATE64)
                              : (k == B2_TEMPORAL_TIME32 || k == B2_TEMPORAL_TIME64));
  if (!ok)
    return set_error(B2_NOT_IMPLEMENTED, "Function '%s' has no kernel matching input types (%s)", kFieldNames[field],
                     temporal_name(*type).c_str());
  if (field == B2_FIELD_DAY_OF_WEEK && (week_start < 1 || week_start > 7))
    return set_error(B2_INVALID, "week_start must follow ISO convention (Monday=1, Sunday=7). Got week_start=%d",
                     week_start);
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = in->length;
  const bool leap = field == B2_FIELD_IS_LEAP_YEAR;
  const int out_type = leap ? B2_BOOL : field == B2_FIELD_SUBSECOND ? B2_DOUBLE : B2_INT64;

  Temp data(ctx, s);
  const size_t out_bytes = leap ? static_cast<size_t>(bitmap_alloc_bytes(n)) : static_cast<size_t>(n) * 8;
  B2_RETURN_NOT_OK(data.alloc(out_bytes));
  void* validity = nullptr;
  int64_t null_count = 0;
  B2_RETURN_NOT_OK(make_validity(ctx, in, nullptr, n, &validity, &null_count, s));
  Temp vguard(ctx, s);
  vguard.ptr = validity;

  if (n > 0) {
    const int64_t shift = zone_shift(*type);
    const uint32_t dow_table = day_of_week_table(week_start, count_from_zero);
    // date32 counts days, date64 milliseconds; the others count their unit
    const int unit = k == B2_TEMPORAL_DATE32 ? kDays : k == B2_TEMPORAL_DATE64 ? B2_MILLI : type->unit;
    const auto run = [&](auto in_tag, auto uc) -> int {
      using In = decltype(in_tag);
      constexpr int U = decltype(uc)::value;
      if (leap) {
        const int64_t n_words = static_cast<int64_t>(out_bytes / 4);
        const int grid = grid_for(n_words, kWarpsPerBlock, kSMs * 8 * 16);
        leap_year_kernel<In, U><<<grid, kBlock, 0, s>>>(static_cast<const In*>(in->data) + in->offset,
                                                        static_cast<uint32_t*>(data.ptr), n, n_words, shift);
        B2_LAUNCHED();
        return B2_OK;
      }
      return visit_width<B2_FIELD_YEAR, B2_FIELD_MONTH, B2_FIELD_DAY, B2_FIELD_DAY_OF_YEAR, B2_FIELD_DAY_OF_WEEK,
                         B2_FIELD_QUARTER, B2_FIELD_HOUR, B2_FIELD_MINUTE, B2_FIELD_SECOND, B2_FIELD_MILLISECOND,
                         B2_FIELD_MICROSECOND, B2_FIELD_NANOSECOND, B2_FIELD_SUBSECOND>(field, [&](auto fc) -> int {
        constexpr int F = decltype(fc)::value;
        using Out = typename std::conditional<F == B2_FIELD_SUBSECOND, double, int64_t>::type;
        return launch_map<In, Out>(in, data.ptr, FieldOp<In, Out, F, U>{shift, dow_table}, s);
      });
    };
    int st;
    if (unit == kDays) {
      st = run(int32_t{}, std::integral_constant<int, kDays>{});
    } else if (k == B2_TEMPORAL_TIME32) {
      st = visit_unit<B2_SECOND, B2_MILLI>(unit, [&](auto uc) { return run(int32_t{}, uc); });
    } else {
      st = visit_unit<B2_SECOND, B2_MILLI, B2_MICRO, B2_NANO>(unit, [&](auto uc) { return run(int64_t{}, uc); });
    }
    B2_RETURN_NOT_OK(st);
  } else if (leap) {
    B2_CUDA(cudaMemsetAsync(data.ptr, 0, out_bytes, s));
  }
  fill_out(out, out_type, n, null_count, vguard.release(), data.release());
  return B2_OK;
}
