// scalar_cast.cu -- number -> number casts.
//
// Replaces, for the ten numeric types:
//   CastNumberToNumberUnsafe / CastPrimitive  kernels/scalar_cast_internal.cc:41-53,155
//   CastIntegerToInteger + IntegersCanFit     kernels/scalar_cast_numeric.cc:45-54,
//                                             util/int_util.cc:594-660,896-929
//   CastFloatingToInteger + CheckFloatTruncation   kernels/scalar_cast_numeric.cc:91-209
//   CastIntegerToFloating + 2^24 / 2^53 bound      kernels/scalar_cast_numeric.cc:214-279
// Semantics kept: every slot is converted (also under nulls), only VALID slots are
// checked, the error names the first offending element; validity is the input's
// validity re-based to offset 0 (NullHandling::INTERSECTION).
//
// Roofline: HBM-bound stream, algorithmic bytes/row = sizeof(In) + sizeof(Out) +
// 2/8 when a validity bitmap is present (f64->f32: 12.25 B/row, SURVEY section 8d).
#include <cmath>
#include <limits>
#include <type_traits>

#include "bitmap.h"
#include "elementwise.cuh"

namespace b2 {

// float -> integer conversion of out-of-range inputs (and of NaN / +-inf) is UB in the
// reference (ARROW_DISABLE_UBSAN("float-cast-overflow"), scalar_cast_internal.cc:42).  We
// define it as x86-64's scalar conversion: cvttsd2si / cvttss2si of the instruction's width,
// whose out-of-range answer is the "integer indefinite" value INT_MIN, narrowed to the target.
// That is what the reference's scalar loop produces; its vectorised loop body can differ
// (for float -> uint32 pyarrow 24's answer depends on where the element sits in the array),
// so a `safe=false` cast agrees with the reference only where the reference agrees with itself.
template <typename F>
__device__ __forceinline__ int32_t x86_cvtt32(F x) {
  // fits iff trunc(x) is in [-2^31, 2^31): compare in double so -2147483648.9 still fits
  const double d = static_cast<double>(x);
  return (d > -2147483649.0 && d < 2147483648.0) ? static_cast<int32_t>(x)
                                                 : std::numeric_limits<int32_t>::min();
}
template <typename F>
__device__ __forceinline__ int64_t x86_cvtt64(F x) {
  return (x >= static_cast<F>(-9223372036854775808.0) && x < static_cast<F>(9223372036854775808.0))
             ? static_cast<int64_t>(x)
             : std::numeric_limits<int64_t>::min();
}

template <typename Out, typename In>
__device__ __forceinline__ Out convert(In x) {
  if constexpr (std::is_floating_point<In>::value && std::is_integral<Out>::value) {
    if constexpr (std::is_same<Out, int64_t>::value) {
      return x86_cvtt64(x);
    } else if constexpr (std::is_same<Out, uint64_t>::value) {
      const In two63 = static_cast<In>(9223372036854775808.0);
      if (x >= two63) return static_cast<uint64_t>(x86_cvtt64(x - two63)) ^ 0x8000000000000000ull;
      return static_cast<uint64_t>(x86_cvtt64(x));
    } else if constexpr (std::is_same<Out, uint32_t>::value) {
      return static_cast<uint32_t>(x86_cvtt64(x));
    } else {
      return static_cast<Out>(x86_cvtt32(x));
    }
  } else {
    return static_cast<Out>(x);
  }
}

template <typename In, typename Out, bool CHECK>
struct CastOp {
  BitmapReader valid;
  ErrorCell err;
  In lo, hi;
  __device__ __forceinline__ Out operator()(In x, int64_t i) const {
    Out y = convert<Out, In>(x);
    if constexpr (CHECK) {
      bool bad;
      if constexpr (std::is_floating_point<In>::value && std::is_integral<Out>::value) {
        bad = static_cast<In>(y) != x;  // WasTruncated::Check, scalar_cast_numeric.cc:65-67
      } else {
        bad = x < lo || x > hi;  // IntegersInRange, int_util.cc:601-603
      }
      if (bad && valid.bit(i)) err.report(i);
    }
    return y;
  }
};

template <typename In, typename Out, bool CHECK>
static int run_cast(const B2Array* in, void* out_data, In lo, In hi, unsigned long long* d_err,
                    cudaStream_t s) {
  constexpr int V = vec_elems<In, Out>();
  const In* src = static_cast<const In*>(in->data) + in->offset;
  Out* dst = static_cast<Out*>(out_data);
  bool vec_ok = aligned_to(src, sizeof(In) * V) && aligned_to(dst, sizeof(Out) * V);
  CastOp<In, Out, CHECK> op;
  op.valid = BitmapReader(in->null_count == 0 ? nullptr : in->validity, in->offset, in->length);
  op.err.first_row = d_err;
  op.lo = lo;
  op.hi = hi;
  map1_kernel<In, Out, V, CastOp<In, Out, CHECK>>
      <<<map_grid<In, Out, V>(in->length), kBlock, 0, s>>>(src, dst, in->length, vec_ok, op);
  B2_LAUNCHED();
  return B2_OK;
}

const char* type_name(int t) {
  switch (t) {
    case B2_BOOL: return "bool";
    case B2_INT8: return "int8";
    case B2_UINT8: return "uint8";
    case B2_INT16: return "int16";
    case B2_UINT16: return "uint16";
    case B2_INT32: return "int32";
    case B2_UINT32: return "uint32";
    case B2_INT64: return "int64";
    case B2_UINT64: return "uint64";
    case B2_FLOAT: return "float";
    case B2_DOUBLE: return "double";
    case B2_STRING: return "string";
    case B2_BINARY: return "binary";
    case B2_LARGE_STRING: return "large_string";
    case B2_LARGE_BINARY: return "large_binary";
    default: return "?";
  }
}

template <typename T>
static std::string to_chars(T v) {
  if constexpr (std::is_floating_point<T>::value) {
    char b[512];
    snprintf(b, sizeof(b), "%f", static_cast<double>(v));  // the reference formats with std::to_string
    return b;
  } else if constexpr (std::is_signed<T>::value) {
    return std::to_string(static_cast<long long>(v));
  } else {
    return std::to_string(static_cast<unsigned long long>(v));
  }
}

}  // namespace b2

using namespace b2;

extern "C" int b2_cast_numeric(B2Context* ctx, const B2Array* in, const B2CastOptions* options,
                               B2Array* out, void* stream) {
  if (!ctx || !in || !options || !out) return set_error(B2_INVALID, "b2_cast_numeric: null argument");
  if (!type_is_numeric(in->type) || !type_is_numeric(options->to_type))
    return set_error(B2_NOT_IMPLEMENTED, "Unsupported cast from %s to %s using function cast_%s",
                     type_name(in->type), type_name(options->to_type), type_name(options->to_type));
  if (in->length < 0 || in->offset < 0) return set_error(B2_INVALID, "negative length/offset");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const int64_t n = in->length;
  const int to = options->to_type;

  Temp data(ctx, s);
  B2_RETURN_NOT_OK(data.alloc(static_cast<size_t>(n) * type_width(to)));
  void* validity = nullptr;
  int64_t null_count = 0;
  B2_RETURN_NOT_OK(make_validity(ctx, in, nullptr, n, &validity, &null_count, s));
  Temp vguard(ctx, s);
  vguard.ptr = validity;

  if (n > 0) {
    ScalarSlot slot(ctx);
    bool checked = false;
    int st = visit_type(NumericTypes{}, in->type, [&](auto in_tag) -> int {
      using In = decltype(in_tag);
      return visit_type(NumericTypes{}, to, [&](auto out_tag) -> int {
        using Out = decltype(out_tag);
        In lo = std::numeric_limits<In>::lowest(), hi = std::numeric_limits<In>::max();
        bool need = false;
        constexpr bool in_int = std::is_integral<In>::value, out_int = std::is_integral<Out>::value;
        if constexpr (in_int && out_int) {
          if (!options->allow_int_overflow) {
            // GetSafeMinMax: intersection of the two ranges, expressed in In
            __int128 imin = std::numeric_limits<In>::lowest(), imax = std::numeric_limits<In>::max();
            __int128 omin = std::numeric_limits<Out>::lowest(), omax = std::numeric_limits<Out>::max();
            __int128 l = imin > omin ? imin : omin, h = imax < omax ? imax : omax;
            lo = static_cast<In>(l);
            hi = static_cast<In>(h);
            need = (l > imin) || (h < imax);
          }
        } else if constexpr (!in_int && out_int) {
          need = !options->allow_float_truncate;
        } else if constexpr (in_int && !out_int) {
          if (!options->allow_float_truncate && sizeof(In) >= 4 &&
              !(sizeof(In) == 4 && std::is_same<Out, double>::value)) {
            const int64_t limit = std::is_same<Out, float>::value ? (1ll << 24) : (1ll << 53);
            __int128 imin = std::numeric_limits<In>::lowest(), imax = std::numeric_limits<In>::max();
            __int128 l = std::is_signed<In>::value ? -static_cast<__int128>(limit) : 0, h = limit;
            need = (l > imin) || (h < imax);
            lo = static_cast<In>(l > imin ? l : imin);
            hi = static_cast<In>(h < imax ? h : imax);
          }
        }
        if (!need) return run_cast<In, Out, false>(in, data.ptr, lo, hi, nullptr, s);
        checked = true;
        if (!slot.ok()) return set_error(B2_UNKNOWN_ERROR, "no free scalar slot");
        B2_CUDA(cudaMemsetAsync(slot.dev(), 0xff, 8, s));
        B2_RETURN_NOT_OK((run_cast<In, Out, true>(
            in, data.ptr, lo, hi, reinterpret_cast<unsigned long long*>(slot.dev()), s)));
        B2_RETURN_NOT_OK(slot.fetch(s));
        uint64_t row = static_cast<uint64_t>(slot.host()[0]);
        if (row == ~0ull) return B2_OK;
        In bad;
        B2_CUDA(cudaMemcpyAsync(&bad, static_cast<const In*>(in->data) + in->offset + row,
                                sizeof(In), cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaStreamSynchronize(s));
        if constexpr (!in_int && out_int) {
          return set_error(B2_INVALID, "Float value %s was truncated converting to %s",
                           to_chars(bad).c_str(), type_name(to));
        } else {
          return set_error(B2_INVALID, "Integer value %s not in range: %s to %s",
                           to_chars(bad).c_str(), to_chars(lo).c_str(), to_chars(hi).c_str());
        }
      });
    });
    (void)checked;
    if (st != B2_OK) return st;
  }
  fill_out(out, to, n, null_count, vguard.release(), data.release());
  return B2_OK;
}
