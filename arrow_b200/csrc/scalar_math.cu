// scalar_math.cu -- unary numeric math (abs, negate, sign, sqrt, floor / ceil / trunc, bit_wise_not, the _checked
// variants) and rounding (round, round_to_multiple, round_binary) over the integer types and float32 / float64.
//
// Replaces the reference's op functors and applicators:
//   AbsoluteValue(Checked), Negate(Checked), SquareRoot(Checked), Sign   kernels/base_arithmetic_internal.h:126-660
//   BitWiseNot                                                           kernels/scalar_arithmetic.cc:65-70
//   RoundUtil::Pow10, RoundImpl, RoundToMultiple, Round, RoundBinary, Floor / Ceil / Trunc
//                                                                        kernels/scalar_round.cc:89-1036
// Every op is one streaming pass on elementwise.cuh's map1_kernel (map2_kernel, with an int32 right operand, for
// round_binary).  Floats are rounded by the reference's own sequence of IEEE operations (scale, floor, compare the
// fraction, round, unscale), each a single correctly rounded operation; -fmad=false keeps `v - floor(v)` from being
// contracted.  Only valid rows are checked (ScalarUnaryNotNull*), and the message is the last failing row's.
//
// Integer rounding divides by the call's multiple.  That divisor is a run-time value, and a 64-bit division by one
// costs a call to the emulated division routine per row, so the host computes a multiply-high reciprocal for it
// (Granlund & Montgomery, "Division by invariant integers using multiplication", 1994, section 4): q = (t + ((n - t)
// >> sh1)) >> sh2 with t = mulhi(m, n), exact for every 64-bit n and every divisor.  round_binary's divisor changes per
// row; it divides plainly.
//
// Roofline: HBM-bound stream, algorithmic bytes/row = 2 * sizeof(T) + 2/8 with a nullable input (float64: 16.25 B/row).
#include <cmath>
#include <limits>
#include <type_traits>

#include "bitmap.h"
#include "elementwise.cuh"

namespace b2 {

// the bit pattern of a float as an unsigned integer of its width
template <typename T>
using FloatBits = typename std::conditional<sizeof(T) == 4, uint32_t, uint64_t>::type;

template <typename T>
__host__ __device__ __forceinline__ FloatBits<T> to_bits(T x) {
  FloatBits<T> b;
  memcpy(&b, &x, sizeof(T));
  return b;
}
template <typename T>
__host__ __device__ __forceinline__ T from_bits(FloatBits<T> b) {
  T x;
  memcpy(&x, &b, sizeof(T));
  return x;
}

// ---------------------------------------------------------------------------------------------------------------------
// unary ops
// ---------------------------------------------------------------------------------------------------------------------
template <typename T, int OP>
struct UnaryOp {
  using Out = typename std::conditional<OP == B2_SIGN && std::is_integral<T>::value, int8_t, T>::type;
  BitmapReader valid;  // output validity (offset 0): only consulted on a failure
  LastErrorCell err;
  __device__ __forceinline__ Out operator()(T x, int64_t i) const {
    bool bad = false;
    Out res;
    if constexpr (std::is_floating_point<T>::value) {
      constexpr FloatBits<T> kSign = FloatBits<T>(1) << (8 * sizeof(T) - 1);
      // fabs and unary minus touch the sign bit alone (andpd / xorpd), so a NaN keeps its payload
      if constexpr (OP == B2_ABS || OP == B2_ABS_CHECKED) res = from_bits<T>(to_bits(x) & ~kSign);
      else if constexpr (OP == B2_NEGATE || OP == B2_NEGATE_CHECKED) res = from_bits<T>(to_bits(x) ^ kSign);
      else if constexpr (OP == B2_SIGN) res = isnan(x) ? x : (x == T(0) ? T(0) : (signbit(x) ? T(-1) : T(1)));
      else if constexpr (OP == B2_SQRT) res = x < T(0) ? std::numeric_limits<T>::quiet_NaN() : sqrt(x);
      else if constexpr (OP == B2_SQRT_CHECKED) {
        bad = x < T(0);
        res = bad ? x : sqrt(x);
      } else if constexpr (OP == B2_FLOOR) res = floor(x);
      else if constexpr (OP == B2_CEIL) res = ceil(x);
      else res = trunc(x);  // B2_TRUNC
    } else {
      using UT = typename std::make_unsigned<T>::type;
      constexpr bool kSigned = std::is_signed<T>::value;
      const T neg = static_cast<T>(static_cast<UT>(0) - static_cast<UT>(x));  // wraps: -INT_MIN is INT_MIN
      if constexpr (OP == B2_ABS) res = (kSigned && x < T(0)) ? neg : x;
      else if constexpr (OP == B2_ABS_CHECKED) {
        bad = kSigned && x == std::numeric_limits<T>::min();
        res = (kSigned && x < T(0)) ? neg : x;
      } else if constexpr (OP == B2_NEGATE) res = neg;
      else if constexpr (OP == B2_NEGATE_CHECKED) {  // signed only
        bad = x == std::numeric_limits<T>::min();
        res = neg;
      } else if constexpr (OP == B2_SIGN) res = x > T(0) ? 1 : (x == T(0) ? 0 : -1);
      else res = static_cast<T>(~x);  // B2_BIT_WISE_NOT
    }
    if (bad && valid.bit(i)) err.report(i);
    return res;
  }
};

// ---------------------------------------------------------------------------------------------------------------------
// rounding
// ---------------------------------------------------------------------------------------------------------------------
// RoundUtil::Pow10<double>: 10^|power| from a table of FLOAT literals (so 10^11 .. 10^15 are the float-rounded values),
// beyond 10^15 by repeated * 10 in double; 1 / that for a negative power.  Each table entry is the float nearest 10^k,
// which is the float rounding of the exact double 10^k (k <= 15).  Once the product is infinite it stays so, which
// bounds the loop.
__host__ __device__ inline double pow10_ref(int64_t power) {
  const uint64_t abs_power = power < 0 ? 0 - static_cast<uint64_t>(power) : static_cast<uint64_t>(power);
  double exact = 1.0;
  for (uint64_t k = 0; k < (abs_power < 15 ? abs_power : 15); ++k) exact *= 10.0;
  double p = static_cast<double>(static_cast<float>(exact));
  for (uint64_t k = 15; k < abs_power && p <= std::numeric_limits<double>::max(); ++k) p *= 10.0;
  return power >= 0 ? p : 1.0 / p;
}

// RoundImpl<T, MODE>::Round for a float: the value rounded in the mode's direction (a tie mode reaches it only at a
// fraction of exactly 0.5)
template <typename T, int MODE>
__host__ __device__ __forceinline__ T round_float_mode(T v) {
  if constexpr (MODE == B2_ROUND_DOWN || MODE == B2_ROUND_HALF_DOWN) return floor(v);
  else if constexpr (MODE == B2_ROUND_UP || MODE == B2_ROUND_HALF_UP) return ceil(v);
  else if constexpr (MODE == B2_ROUND_TOWARDS_ZERO || MODE == B2_ROUND_HALF_TOWARDS_ZERO) return trunc(v);
  else if constexpr (MODE == B2_ROUND_TOWARDS_INFINITY || MODE == B2_ROUND_HALF_TOWARDS_INFINITY)
    return signbit(v) ? floor(v) : ceil(v);
  else if constexpr (MODE == B2_ROUND_HALF_TO_EVEN) return round(v * T(0.5)) * T(2);
  else return floor(v * T(0.5)) + ceil(v * T(0.5));  // B2_ROUND_HALF_TO_ODD
}

// Round::Call / RoundToMultiple::Call / RoundBinary::Call for a float, in type C.  The value is scaled by `p` (multiplied
// when scale_mul, else divided) and unscaled the other way (divided when unscale_div).  Returns false on the overflow
// error, with *out = arg.
template <typename C, int MODE>
__host__ __device__ __forceinline__ bool round_float(C arg, C p, bool scale_mul, bool unscale_div, C* out) {
  *out = arg;
  if (!isfinite(arg)) return true;
  C r = scale_mul ? arg * p : arg / p;
  const C frac = r - floor(r);
  if (frac == C(0)) return true;  // already on the grid: the input itself (keeps -0.0)
  r = (MODE >= B2_ROUND_HALF_DOWN && frac != C(0.5)) ? round(r) : round_float_mode<C, MODE>(r);
  r = unscale_div ? r / p : r * p;
  if (!isfinite(r)) return false;
  *out = r;
  return true;
}

// error codes of integer rounding, named by the texts they produce
enum RoundError : int {
  kRoundOk = 0,
  kUpToMultiple = 1,     // "Rounding X up to multiple of M would overflow"
  kDownToMultiple = 2,   // "... down to multiple of ..."
  kUpToMultiples = 3,    // "... up to multiples of ...": the nearest-value branch
  kDownToMultiples = 4,
  kDigitsOutOfRange = 5  // "Rounding to N digits is out of range for type T"
};

// 64-bit unsigned division by an invariant divisor d >= 1 as a multiply-high and two shifts
struct Divider {
  uint64_t m;
  int sh1, sh2;
  static Divider make(uint64_t d) {
    int l = 0;
    while (l < 64 && (static_cast<unsigned __int128>(1) << l) < d) ++l;  // ceil(log2 d)
    const unsigned __int128 two_l = static_cast<unsigned __int128>(1) << l;
    Divider r;
    r.m = static_cast<uint64_t>(((two_l - d) << 64) / d + 1);
    r.sh1 = l < 1 ? l : 1;
    r.sh2 = l > 1 ? l - 1 : 0;
    return r;
  }
  __host__ __device__ __forceinline__ uint64_t div(uint64_t n) const {
#ifdef __CUDA_ARCH__
    const uint64_t t = __umul64hi(m, n);
#else
    const uint64_t t = static_cast<uint64_t>((static_cast<unsigned __int128>(m) * n) >> 64);
#endif
    return (t + ((n - t) >> sh1)) >> sh2;
  }
};

// a divisor divided by plainly (round_binary's per-row power of ten)
struct PlainDivider {
  uint64_t d;
  __host__ __device__ __forceinline__ uint64_t div(uint64_t n) const { return n / d; }
};

// a / multiple truncated toward zero, through the divider of `multiple` (> 0)
template <typename T, typename D>
__host__ __device__ __forceinline__ T trunc_div(T a, const D& dv) {
  if constexpr (std::is_signed<T>::value) {
    const uint64_t mag = a < T(0) ? 0 - static_cast<uint64_t>(static_cast<int64_t>(a)) : static_cast<uint64_t>(a);
    const uint64_t q = dv.div(mag);
    return static_cast<T>(a < T(0) ? 0 - q : q);
  } else {
    return static_cast<T>(dv.div(static_cast<uint64_t>(a)));
  }
}

// RoundToMultiple<integer>::Call with RoundImpl<integer, MODE>::Round.  remainder * 2 is computed as the reference's
// compiled code does: in int for the types narrower than int, wrapping in T for the others.
template <typename T, int MODE, typename D>
__host__ __device__ __forceinline__ T round_int(T arg, T multiple, const D& dv, int* code) {
  constexpr bool kSigned = std::is_signed<T>::value;
  constexpr T kMin = std::numeric_limits<T>::min(), kMax = std::numeric_limits<T>::max();
  using UT = typename std::make_unsigned<T>::type;
  const T q = trunc_div(arg, dv);
  const T floor = static_cast<T>(static_cast<UT>(q) * static_cast<UT>(multiple));
  const T remainder = arg > floor ? static_cast<T>(arg - floor) : static_cast<T>(floor - arg);
  if (remainder == T(0)) return arg;
  int m = MODE;
  if constexpr (MODE >= B2_ROUND_HALF_DOWN) {
    using P = typename std::conditional<(sizeof(T) < sizeof(int)), int, T>::type;
    const P twice = static_cast<P>(static_cast<typename std::make_unsigned<P>::type>(remainder) * 2u);
    if (twice != static_cast<P>(multiple)) {
      if (twice > static_cast<P>(multiple)) {
        if (arg >= T(0)) {
          if (kMax - multiple < floor) return *code = kUpToMultiples, arg;
          return static_cast<T>(floor + multiple);
        }
        if (kMin + multiple > floor) return *code = kDownToMultiples, arg;
        return static_cast<T>(floor - multiple);
      }
      return floor;
    }
    // a tie: the mode's RoundImpl
    if (MODE == B2_ROUND_HALF_TO_EVEN || MODE == B2_ROUND_HALF_TO_ODD) {
      const bool odd = (q & T(1)) != T(0);
      if (odd == (MODE == B2_ROUND_HALF_TO_ODD)) return floor;
      m = B2_ROUND_TOWARDS_INFINITY;
    } else {
      m = MODE - B2_ROUND_HALF_DOWN;  // HALF_DOWN .. HALF_TOWARDS_INFINITY run DOWN .. TOWARDS_INFINITY
    }
  }
  const bool down = m == B2_ROUND_DOWN || m == B2_ROUND_TOWARDS_INFINITY;
  const bool up = m == B2_ROUND_UP || m == B2_ROUND_TOWARDS_INFINITY;
  if (kSigned && down && arg < T(0)) {
    if (kMin + multiple > floor) return *code = kDownToMultiple, arg;
    return static_cast<T>(floor - multiple);
  }
  if (up && arg > T(0)) {
    if (kMax - multiple < floor) return *code = kUpToMultiple, arg;
    return static_cast<T>(floor + multiple);
  }
  if (!kSigned && m == B2_ROUND_TOWARDS_INFINITY) return static_cast<T>(floor + multiple);  // arg == 0 was returned
  return floor;
}

// digits10 of T, and 10^k in T for k up to it (10^19 for uint64: the reference's table stops at 10^18 and reads past
// its end there)
template <typename T>
__host__ __device__ __forceinline__ T pow10_int(int k) {
  uint64_t p = 1;
  for (int j = 0; j < k; ++j) p *= 10;
  return static_cast<T>(p);
}

// round_binary over an integer: s >= 0 is the identity, else round to a multiple of 10^-s
template <typename T, int MODE>
__host__ __device__ __forceinline__ T round_binary_int(T arg, int32_t s, int* code) {
  if (s >= 0) return arg;
  // -INT32_MIN is out of range too (the reference would index its table with a negative value there)
  if (s < -std::numeric_limits<T>::digits10) return *code = kDigitsOutOfRange, arg;
  const T multiple = pow10_int<T>(-s);
  return round_int<T, MODE>(arg, multiple, PlainDivider{static_cast<uint64_t>(multiple)}, code);
}

// round_binary over a float: Pow10 per row, every step in double, the result cast back to T
template <typename T, int MODE>
__host__ __device__ __forceinline__ T round_binary_float(T arg, int32_t s, bool* ok) {
  // std::abs of an int32: INT32_MIN stays negative, and Pow10 of it is 1 / inf = 0
  const int32_t a = s < 0 ? static_cast<int32_t>(0u - static_cast<uint32_t>(s)) : s;
  const double p = pow10_ref(a);
  double r;
  *ok = round_float<double, MODE>(static_cast<double>(arg), p, s >= 0, s > 0, &r);
  return *ok ? static_cast<T>(r) : arg;
}

template <typename T, int MODE>
struct RoundFloatOp {
  T p;
  bool scale_mul, unscale_div;
  BitmapReader valid;
  LastErrorCell err;
  __device__ __forceinline__ T operator()(T x, int64_t i) const {
    T r;
    if (!round_float<T, MODE>(x, p, scale_mul, unscale_div, &r) && valid.bit(i)) err.report(i);
    return r;
  }
};

template <typename T, int MODE>
struct RoundIntOp {
  T multiple;
  Divider dv;
  BitmapReader valid;
  LastErrorCell err;
  __device__ __forceinline__ T operator()(T x, int64_t i) const {
    int code = kRoundOk;
    const T r = round_int<T, MODE>(x, multiple, dv, &code);
    if (code != kRoundOk && valid.bit(i)) err.report(i);
    return r;
  }
};

template <typename T, int MODE>
struct RoundBinaryOp {
  BitmapReader valid;
  LastErrorCell err;
  __device__ __forceinline__ T operator()(T x, int32_t s, int64_t i) const {
    bool failed;
    T r;
    if constexpr (std::is_floating_point<T>::value) {
      bool ok;
      r = round_binary_float<T, MODE>(x, s, &ok);
      failed = !ok;
    } else {
      int code = kRoundOk;
      r = round_binary_int<T, MODE>(x, s, &code);
      failed = code != kRoundOk;
    }
    if (failed && valid.bit(i)) err.report(i);
    return r;
  }
};

template <typename In, typename Out, typename Op>
static int launch_map1(const In* src, Out* dst, int64_t n, const Op& op, cudaStream_t s) {
  constexpr int V = vec_elems<In, Out>();
  const bool vec_ok = aligned_to(src, sizeof(In) * V) && aligned_to(dst, sizeof(Out) * V);
  map1_kernel<In, Out, V, Op><<<map_grid<In, Out, V>(n), kBlock, 0, s>>>(src, dst, n, vec_ok, op);
  B2_LAUNCHED();
  return B2_OK;
}

// a unary rounding op as a map2_kernel op with no right operand, two accesses of at most four values in flight per lane:
// map2_kernel's tail loop is kept rolled, and with these bounds ptxas spills none of these heavier ops' registers
template <typename T, typename Op>
struct NoRight {
  Op op;
  __device__ __forceinline__ T operator()(T x, T, int64_t i) const { return op(x, i); }
};
template <typename T, typename Op>
static int launch_round(const T* src, T* dst, int64_t n, const Op& op, cudaStream_t s) {
  constexpr int V = sizeof(T) >= 4 ? 16 / sizeof(T) : 4;  // at most four narrow values per access
  const bool vec_ok = aligned_to(src, sizeof(T) * V) && aligned_to(dst, sizeof(T) * V);
  map2_kernel<T, T, V, NoRight<T, Op>, T, 2><<<map_grid<T, T, V, 2>(n), kBlock, 0, s>>>(src, T(0), static_cast<const T*>(nullptr), T(0), dst, n, vec_ok,
                                                                               NoRight<T, Op>{op});
  B2_LAUNCHED();
  return B2_OK;
}

template <typename F>
static int visit_mode(int mode, F&& f) {
  return visit_width<B2_ROUND_DOWN, B2_ROUND_UP, B2_ROUND_TOWARDS_ZERO, B2_ROUND_TOWARDS_INFINITY, B2_ROUND_HALF_DOWN,
                     B2_ROUND_HALF_UP, B2_ROUND_HALF_TOWARDS_ZERO, B2_ROUND_HALF_TOWARDS_INFINITY,
                     B2_ROUND_HALF_TO_EVEN, B2_ROUND_HALF_TO_ODD>(mode, f);
}

template <typename T>
static void format_value(T v, char* buf, size_t size) {
  if constexpr (std::is_signed<T>::value) snprintf(buf, size, "%lld", static_cast<long long>(v));
  else snprintf(buf, size, "%llu", static_cast<unsigned long long>(v));
}

// the message of an integer rounding failure; int8 / uint8 values are printed as numbers (the reference prints them
// as characters)
template <typename T>
static int round_int_error(int code, T arg, T multiple, int32_t s, int type) {
  if (code == kDigitsOutOfRange)
    return set_error(B2_INVALID, "Rounding to %d digits is out of range for type %s", s, type_name(type));
  char a[32], m[32];
  format_value(arg, a, sizeof(a));
  format_value(multiple, m, sizeof(m));
  const bool up = code == kUpToMultiple || code == kUpToMultiples;
  const bool plural = code == kUpToMultiples || code == kDownToMultiples;
  return set_error(B2_INVALID, "Rounding %s %s to multiple%s of %s would overflow", a, up ? "up" : "down",
                   plural ? "s" : "", m);
}

static const char* unary_name(int op) {
  switch (op) {
    case B2_ABS: return "abs";
    case B2_NEGATE: return "negate";
    case B2_SIGN: return "sign";
    case B2_SQRT: return "sqrt";
    case B2_FLOOR: return "floor";
    case B2_CEIL: return "ceil";
    case B2_TRUNC: return "trunc";
    case B2_BIT_WISE_NOT: return "bit_wise_not";
    case B2_ABS_CHECKED: return "abs_checked";
    case B2_NEGATE_CHECKED: return "negate_checked";
    case B2_SQRT_CHECKED: return "sqrt_checked";
    default: return nullptr;
  }
}

// whether the reference registers a kernel of unary op `op` for type id t
static bool unary_accepts(int op, int t) {
  const bool is_float = t == B2_FLOAT || t == B2_DOUBLE;
  switch (op) {
    case B2_SQRT: case B2_SQRT_CHECKED: case B2_FLOOR: case B2_CEIL: case B2_TRUNC: return is_float;
    case B2_BIT_WISE_NOT: return !is_float;
    case B2_NEGATE_CHECKED: return is_float || type_is_signed_int(t);
    default: return true;
  }
}

}  // namespace b2

using namespace b2;

extern "C" int b2_unary_arith(B2Context* ctx, int op, const B2Array* in, B2Array* out, void* stream) {
  if (!ctx || !in || !out) return set_error(B2_INVALID, "b2_unary_arith: null argument");
  const char* name = unary_name(op);
  if (!name) return set_error(B2_INVALID, "unknown unary op %d", op);
  if (in->length < 0 || in->offset < 0) return set_error(B2_INVALID, "negative length/offset");
  const int type = in->type;
  if (!type_is_numeric(type) || !unary_accepts(op, type))
    return set_error(B2_NOT_IMPLEMENTED, "Function '%s' has no kernel matching input types (%s)", name,
                     type_name(type));
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = in->length;
  const int out_type = (op == B2_SIGN && type != B2_FLOAT && type != B2_DOUBLE) ? B2_INT8 : type;

  Temp data(ctx, s);
  B2_RETURN_NOT_OK(data.alloc(static_cast<size_t>(n) * type_width(out_type)));
  void* validity = nullptr;
  int64_t null_count = 0;
  B2_RETURN_NOT_OK(make_validity(ctx, in, nullptr, n, &validity, &null_count, s));
  Temp vguard(ctx, s);
  vguard.ptr = validity;
  if (n > 0) {
    const bool can_fail = op >= B2_ABS_CHECKED;
    ScalarSlot slot(ctx);
    LastErrorCell err{nullptr};
    if (can_fail) {
      if (!slot.ok()) return set_error(B2_UNKNOWN_ERROR, "no free scalar slot");
      B2_CUDA(cudaMemsetAsync(slot.dev(), 0, 8, s));
      err.last_row1 = reinterpret_cast<unsigned long long*>(slot.dev());
    }
    const BitmapReader valid(validity, 0, n);
    B2_RETURN_NOT_OK(visit_type(NumericTypes{}, type, [&](auto tag) -> int {
      using T = decltype(tag);
      const T* src = static_cast<const T*>(in->data) + in->offset;
      const auto run = [&](auto oc) -> int {
        constexpr int OP = decltype(oc)::value;
        using Op = UnaryOp<T, OP>;
        return launch_map1<T, typename Op::Out>(src, static_cast<typename Op::Out*>(data.ptr), n, Op{valid, err}, s);
      };
      if constexpr (std::is_floating_point<T>::value) {
        return visit_width<B2_ABS, B2_NEGATE, B2_SIGN, B2_SQRT, B2_FLOOR, B2_CEIL, B2_TRUNC, B2_ABS_CHECKED,
                           B2_NEGATE_CHECKED, B2_SQRT_CHECKED>(op, run);
      } else if constexpr (std::is_signed<T>::value) {
        return visit_width<B2_ABS, B2_NEGATE, B2_SIGN, B2_BIT_WISE_NOT, B2_ABS_CHECKED, B2_NEGATE_CHECKED>(op, run);
      } else {
        return visit_width<B2_ABS, B2_NEGATE, B2_SIGN, B2_BIT_WISE_NOT, B2_ABS_CHECKED>(op, run);
      }
    }));
    if (can_fail) {
      B2_RETURN_NOT_OK(slot.fetch(s));
      if (slot.host()[0] != 0)
        return set_error(B2_INVALID, op == B2_SQRT_CHECKED ? "square root of negative number" : "overflow");
    }
  }
  fill_out(out, out_type, n, null_count, vguard.release(), data.release());
  return B2_OK;
}

extern "C" int b2_round(B2Context* ctx, const B2Value* x, const B2Value* digits, int64_t ndigits,
                        const B2Scalar* multiple, int round_mode, B2Array* out, void* stream) {
  if (!ctx || !x || !out) return set_error(B2_INVALID, "b2_round: null argument");
  if (round_mode < B2_ROUND_DOWN || round_mode > B2_ROUND_HALF_TO_ODD)
    return set_error(B2_INVALID, "unknown round mode %d", round_mode);
  const B2Array* xa = x->array;
  const B2Array* da = digits ? digits->array : nullptr;
  if (!xa && !x->scalar) return set_error(B2_INVALID, "b2_round: x has neither array nor scalar");
  if (digits && !da && !digits->scalar) return set_error(B2_INVALID, "b2_round: digits has neither array nor scalar");
  if (!xa && !da) return set_error(B2_INVALID, "at least one operand must be an array");
  if (!digits && !xa) return set_error(B2_INVALID, "b2_round: x must be an array");
  const int type = xa ? xa->type : x->scalar->type;
  const char* fname = digits ? "round_binary" : multiple ? "round_to_multiple" : "round";
  if (!type_is_numeric(type))
    return set_error(B2_NOT_IMPLEMENTED, "Function '%s' has no kernel matching input types (%s)", fname,
                     type_name(type));
  if (digits && (da ? da->type : digits->scalar->type) != B2_INT32)
    return set_error(B2_TYPE_ERROR, "b2_round: digits must be int32");
  if (xa && da && xa->length != da->length) return set_error(B2_INVALID, "Array arguments must all be the same length");
  if ((xa && (xa->length < 0 || xa->offset < 0)) || (da && (da->length < 0 || da->offset < 0)))
    return set_error(B2_INVALID, "negative length/offset");
  const bool is_float = type == B2_FLOAT || type == B2_DOUBLE;
  const int w = type_width(type);
  if (multiple) {
    if (multiple->type != type) return set_error(B2_TYPE_ERROR, "b2_round: multiple must have x's type");
    if (!multiple->is_valid) return set_error(B2_INVALID, "Rounding multiple must be non-null and valid");
    // the reference checks the sign before its cast to x's type, so a positive float64 that became float32 +0 is let
    // through (and overflows); a float +0 is accepted here for that reason, -0.0 is not
    bool positive = false;
    visit_type(NumericTypes{}, type, [&](auto tag) {
      using T = decltype(tag);
      const T m = scalar_bits<T>(multiple);
      positive = m > T(0) || (std::is_floating_point<T>::value && m == T(0) && !signbit(static_cast<double>(m)));
      return B2_OK;
    });
    if (!positive) return set_error(B2_INVALID, "Rounding multiple must be positive");
  }
  // round over an integer: the digit count is checked once, before any row (RoundOptionsWrapper::Init)
  int int_digits10 = 0;
  visit_type(NumericTypes{}, type, [&](auto tag) {
    int_digits10 = std::numeric_limits<decltype(tag)>::digits10;
    return B2_OK;
  });
  if (!digits && !multiple && !is_float && ndigits < 0 && -static_cast<double>(ndigits) > int_digits10)
    return set_error(B2_INVALID, "Rounding to %lld digits is out of range for type %s", static_cast<long long>(ndigits),
                     type_name(type));
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = xa ? xa->length : da->length;

  Temp data(ctx, s);
  B2_RETURN_NOT_OK(data.alloc(static_cast<size_t>(n) * w));
  if ((!xa && !x->scalar->is_valid) || (digits && !da && !digits->scalar->is_valid)) {
    // a null scalar operand nulls every row
    Temp bits(ctx, s);
    B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(n)));
    B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bitmap_alloc_bytes(n), s));
    B2_CUDA(cudaMemsetAsync(data.ptr, 0, static_cast<size_t>(n) * w + (n == 0), s));
    fill_out(out, type, n, n, n ? bits.release() : nullptr, data.release());
    return B2_OK;
  }
  void* validity = nullptr;
  int64_t null_count = 0;
  B2_RETURN_NOT_OK(make_validity(ctx, xa, da, n, &validity, &null_count, s));
  Temp vguard(ctx, s);
  vguard.ptr = validity;
  if (n > 0 && !digits && !multiple && !is_float && ndigits >= 0) {
    // round over an integer to ndigits >= 0 is the identity
    B2_CUDA(cudaMemcpyAsync(data.ptr, static_cast<const char*>(xa->data) + xa->offset * w, static_cast<size_t>(n) * w,
                            cudaMemcpyDeviceToDevice, s));
  } else if (n > 0) {
    ScalarSlot slot(ctx);
    if (!slot.ok()) return set_error(B2_UNKNOWN_ERROR, "no free scalar slot");
    B2_CUDA(cudaMemsetAsync(slot.dev(), 0, 8, s));
    const LastErrorCell err{reinterpret_cast<unsigned long long*>(slot.dev())};
    const BitmapReader valid(validity, 0, n);
    B2_RETURN_NOT_OK(visit_type(NumericTypes{}, type, [&](auto tag) -> int {
      using T = decltype(tag);
      T* dst = static_cast<T*>(data.ptr);
      const T* src = xa ? static_cast<const T*>(xa->data) + xa->offset : nullptr;
      const T mult = is_float ? T(0) : multiple ? scalar_bits<T>(multiple) : pow10_int<T>(ndigits < 0 ? -ndigits : 0);
      B2_RETURN_NOT_OK(visit_mode(round_mode, [&](auto mc) -> int {
        constexpr int MODE = decltype(mc)::value;
        if (digits) {
          constexpr int V = vec_elems<T, int32_t>();
          const int32_t* ds = da ? static_cast<const int32_t*>(da->data) + da->offset : nullptr;
          const bool vec_ok = aligned_to(dst, sizeof(T) * V) && (!src || aligned_to(src, sizeof(T) * V)) &&
                              (!ds || aligned_to(ds, sizeof(int32_t) * V));
          // an integer row divides by its own power of ten: one access in flight per lane, so that it does not spill
          constexpr int U = std::is_integral<T>::value ? 1 : kUnroll;
          map2_kernel<T, T, V, RoundBinaryOp<T, MODE>, int32_t, U><<<map_grid<T, int32_t, V, U>(n), kBlock, 0, s>>>(
              src, scalar_bits<T>(x->scalar), ds, scalar_bits<int32_t>(digits ? digits->scalar : nullptr), dst, n,
              vec_ok, RoundBinaryOp<T, MODE>{valid, err});
          B2_LAUNCHED();
          return B2_OK;
        }
        if constexpr (std::is_floating_point<T>::value) {
          // round: scale by Pow10(|ndigits|), cast to T (RoundOptionsWrapper keeps it in double); round_to_multiple:
          // divide by the multiple, multiply back
          const T p = multiple ? scalar_bits<T>(multiple) : static_cast<T>(pow10_ref(ndigits < 0 ? -ndigits : ndigits));
          const bool scale_mul = !multiple && ndigits >= 0, unscale_div = !multiple && ndigits > 0;
          return launch_round<T>(src, dst, n, RoundFloatOp<T, MODE>{p, scale_mul, unscale_div, valid, err}, s);
        } else {
          const Divider dv = Divider::make(static_cast<uint64_t>(mult));
          return launch_round<T>(src, dst, n, RoundIntOp<T, MODE>{mult, dv, valid, err}, s);
        }
      }));
      B2_RETURN_NOT_OK(slot.fetch(s));
      const uint64_t row1 = static_cast<uint64_t>(slot.host()[0]);
      if (row1 == 0) return B2_OK;
      if constexpr (std::is_floating_point<T>::value) {
        return set_error(B2_INVALID, "overflow occurred during rounding");
      } else {
        // recompute the last failing row on the host for its message
        const int64_t row = static_cast<int64_t>(row1 - 1);
        uint64_t xb = 0, sb = 0;
        B2_RETURN_NOT_OK(operand_bits(x, row, w, &xb, s));
        T arg;
        memcpy(&arg, &xb, sizeof(T));
        int code = kRoundOk;
        int32_t sv = 0;
        if (digits) {
          B2_RETURN_NOT_OK(operand_bits(digits, row, 4, &sb, s));
          sv = static_cast<int32_t>(static_cast<uint32_t>(sb));
          visit_mode(round_mode, [&](auto mc) {
            round_binary_int<T, decltype(mc)::value>(arg, sv, &code);
            return B2_OK;
          });
          if (code == kDigitsOutOfRange) return round_int_error<T>(code, arg, T(0), sv, type);
          return round_int_error<T>(code, arg, pow10_int<T>(-sv), sv, type);
        }
        const Divider dv = Divider::make(static_cast<uint64_t>(mult));
        visit_mode(round_mode, [&](auto mc) {
          round_int<T, decltype(mc)::value>(arg, mult, dv, &code);
          return B2_OK;
        });
        return round_int_error<T>(code, arg, mult, 0, type);
      }
    }));
  }
  fill_out(out, type, n, null_count, vguard.release(), data.release());
  return B2_OK;
}
