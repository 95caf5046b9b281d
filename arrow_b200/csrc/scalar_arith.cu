// scalar_arith.cu -- add / subtract / multiply / divide / power (+ _checked variants), bit_wise_and / or / xor and
// shift_left / shift_right (+ _checked).
//
// Replaces the reference's arithmetic applicators and op functors:
//   ScalarBinary<..>::{ArrayArray,ArrayScalar,ScalarArray}   kernels/codegen_internal.h:813-874
//   ScalarBinaryNotNull* (checked ops, divide: null slots are never checked)  :878-976
//   Add/AddChecked/Subtract/SubtractChecked/Multiply/MultiplyChecked/Divide/DivideChecked
//                                                  kernels/base_arithmetic_internal.h:44-423
//   Power/PowerChecked                             kernels/base_arithmetic_internal.h:558-618
//   BitWiseAnd/Or/Xor, ShiftLeft(Checked), ShiftRight(Checked)   kernels/scalar_arithmetic.cc:72-161
// Semantics kept: unchecked signed-integer ops wrap (computed in unsigned arithmetic),
// floats are a single IEEE operation (bit-exact; no FMA contraction possible, no
// flush-to-zero), checked ops raise Invalid("overflow") / Invalid("divide by zero") with the
// message of the last offending VALID slot, integer INT_MIN / -1 is 0 for `divide`, overflow for
// `divide_checked`.  Unchecked power is a plain ScalarBinary: its negative-exponent error is raised from null slots
// too.  Both operands arrive with the dispatched common type
// (ArithmeticFunction::DispatchBest, kernels/scalar_arithmetic.cc:734-781).
//
// Roofline: HBM-bound; algorithmic bytes/row = 3*sizeof(T) + 3/8 with two nullable
// inputs (Add f32: 12.375 B/row, SURVEY section 8d).
#include <limits>
#include <type_traits>

#include "bitmap.h"
#include "elementwise.cuh"

namespace b2 {

template <typename T>
using U = typename std::make_unsigned<T>::type;

// the integer-only ops: Power and the bit-wise ops are registered for integers alone
__host__ __device__ constexpr bool int_only_op(int op) {
  return (op >= B2_POWER && op <= B2_SHIFT_RIGHT) || op >= B2_POWER_CHECKED;
}

template <typename T, int OP>
struct ArithOp {
  BitmapReader valid;  // output validity (offset 0) -- only consulted on a failure
  LastErrorCell err;
  __device__ __forceinline__ T operator()(T l, T r, int64_t i) const {
    constexpr bool kInt = std::is_integral<T>::value;
    T res;
    bool bad = false;
    if constexpr (!kInt) {
      if constexpr (OP == B2_ADD || OP == B2_ADD_CHECKED) res = l + r;
      else if constexpr (OP == B2_SUBTRACT || OP == B2_SUBTRACT_CHECKED) res = l - r;
      else if constexpr (OP == B2_MULTIPLY || OP == B2_MULTIPLY_CHECKED) res = l * r;
      else if constexpr (OP == B2_DIVIDE) res = l / r;
      else {  // DivideChecked, base_arithmetic_internal.h:406-414
        bad = (r == 0);
        res = bad ? T(0) : l / r;
      }
    } else {
      using UT = U<T>;
      using W = typename std::conditional<(sizeof(T) < 4), uint32_t, UT>::type;
      if constexpr (OP == B2_ADD) {
        res = static_cast<T>(static_cast<W>(static_cast<UT>(l)) + static_cast<W>(static_cast<UT>(r)));
      } else if constexpr (OP == B2_SUBTRACT) {
        res = static_cast<T>(static_cast<W>(static_cast<UT>(l)) - static_cast<W>(static_cast<UT>(r)));
      } else if constexpr (OP == B2_MULTIPLY) {
        res = static_cast<T>(static_cast<W>(static_cast<UT>(l)) * static_cast<W>(static_cast<UT>(r)));
      } else if constexpr (OP == B2_ADD_CHECKED) {
        res = static_cast<T>(static_cast<W>(static_cast<UT>(l)) + static_cast<W>(static_cast<UT>(r)));
        if constexpr (std::is_signed<T>::value) bad = ((l ^ res) & (r ^ res)) < 0;
        else bad = res < l;
      } else if constexpr (OP == B2_SUBTRACT_CHECKED) {
        res = static_cast<T>(static_cast<W>(static_cast<UT>(l)) - static_cast<W>(static_cast<UT>(r)));
        if constexpr (std::is_signed<T>::value) bad = ((l ^ r) & (l ^ res)) < 0;
        else bad = l < r;
      } else if constexpr (OP == B2_MULTIPLY_CHECKED) {
        bad = mul_overflow(l, r, &res);
      } else if constexpr (OP == B2_POWER) {
        // IntegerPower: right to left over the operands sign-extended to uint64, wrapped back to T
        bad = r < T(0);
        uint64_t base = static_cast<uint64_t>(static_cast<int64_t>(l)), e = static_cast<uint64_t>(r), p = 1;
        if constexpr (!std::is_signed<T>::value) base = static_cast<uint64_t>(l);
#pragma unroll 1
        while (e) {
          p *= (e & 1) ? base : 1;
          base *= base;
          e >>= 1;
        }
        res = bad ? T(0) : static_cast<T>(p);
      } else if constexpr (OP == B2_POWER_CHECKED) {
        // left to right from the top set bit of the exponent, every step checked
        res = T(1);
        if (r < T(0)) {
          bad = true;
          res = T(0);
        } else if (r != T(0)) {
#pragma unroll 1
          for (uint64_t mask = 1ull << (63 - __clzll(static_cast<long long>(static_cast<uint64_t>(r)))); mask; mask >>= 1) {
            bad |= mul_overflow(res, res, &res);
            if (static_cast<uint64_t>(r) & mask) bad |= mul_overflow(res, l, &res);
          }
        }
      } else if constexpr (OP == B2_BIT_WISE_AND) {
        res = l & r;
      } else if constexpr (OP == B2_BIT_WISE_OR) {
        res = l | r;
      } else if constexpr (OP == B2_BIT_WISE_XOR) {
        res = l ^ r;
      } else if constexpr (OP == B2_SHIFT_LEFT || OP == B2_SHIFT_LEFT_CHECKED || OP == B2_SHIFT_RIGHT ||
                           OP == B2_SHIFT_RIGHT_CHECKED) {
        // an amount outside [0, digits) returns the left operand; digits excludes a signed type's sign bit
        const bool out_of_range = r < T(0) || r >= T(std::numeric_limits<T>::digits);
        bad = (OP == B2_SHIFT_LEFT_CHECKED || OP == B2_SHIFT_RIGHT_CHECKED) && out_of_range;
        if (out_of_range) res = l;
        else if constexpr (OP == B2_SHIFT_LEFT || OP == B2_SHIFT_LEFT_CHECKED)
          res = static_cast<T>(static_cast<W>(static_cast<UT>(l)) << static_cast<int>(r));
        else res = static_cast<T>(l >> static_cast<int>(r));  // arithmetic for a signed type
      } else {  // DIVIDE / DIVIDE_CHECKED, base_arithmetic_internal.h:364-400
        bool overflow = false;
        if constexpr (std::is_signed<T>::value)
          overflow = (l == std::numeric_limits<T>::min() && r == T(-1));
        if (r == 0) {
          bad = true;
          res = 0;
        } else if (overflow) {
          bad = (OP == B2_DIVIDE_CHECKED);
          res = (OP == B2_DIVIDE_CHECKED) ? l : T(0);
        } else {
          res = l / r;
        }
      }
    }
    if (bad && (OP == B2_POWER || valid.bit(i))) err.report(i);
    return res;
  }
};

template <typename T, int OP>
static int run_arith(const T* a, T sa, const T* b, T sb, T* out, int64_t n, const void* out_validity,
                     unsigned long long* d_err, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  bool vec_ok = aligned_to(out, 16) && (!a || aligned_to(a, 16)) && (!b || aligned_to(b, 16));
  ArithOp<T, OP> op;
  op.valid = BitmapReader(out_validity, 0, n);
  op.err.last_row1 = d_err;
  // the checked power loop keeps one access in flight per lane, so that its registers do not spill
  constexpr int U = OP == B2_POWER_CHECKED ? 1 : kUnroll;
  map2_kernel<T, T, V, ArithOp<T, OP>, T, U>
      <<<map_grid<T, T, V, U>(n), kBlock, 0, s>>>(a, sa, b, sb, out, n, vec_ok, op);
  B2_LAUNCHED();
  return B2_OK;
}

template <typename T>
static int run_arith_op(int op, const T* a, T sa, const T* b, T sb, T* out, int64_t n,
                        const void* v, unsigned long long* e, cudaStream_t s) {
  switch (op) {
    case B2_ADD: return run_arith<T, B2_ADD>(a, sa, b, sb, out, n, v, e, s);
    case B2_SUBTRACT: return run_arith<T, B2_SUBTRACT>(a, sa, b, sb, out, n, v, e, s);
    case B2_MULTIPLY: return run_arith<T, B2_MULTIPLY>(a, sa, b, sb, out, n, v, e, s);
    case B2_DIVIDE: return run_arith<T, B2_DIVIDE>(a, sa, b, sb, out, n, v, e, s);
    case B2_ADD_CHECKED: return run_arith<T, B2_ADD_CHECKED>(a, sa, b, sb, out, n, v, e, s);
    case B2_SUBTRACT_CHECKED: return run_arith<T, B2_SUBTRACT_CHECKED>(a, sa, b, sb, out, n, v, e, s);
    case B2_MULTIPLY_CHECKED: return run_arith<T, B2_MULTIPLY_CHECKED>(a, sa, b, sb, out, n, v, e, s);
    case B2_DIVIDE_CHECKED: return run_arith<T, B2_DIVIDE_CHECKED>(a, sa, b, sb, out, n, v, e, s);
    default: break;
  }
  if constexpr (std::is_integral<T>::value) {
    switch (op) {
      case B2_POWER: return run_arith<T, B2_POWER>(a, sa, b, sb, out, n, v, e, s);
      case B2_POWER_CHECKED: return run_arith<T, B2_POWER_CHECKED>(a, sa, b, sb, out, n, v, e, s);
      case B2_BIT_WISE_AND: return run_arith<T, B2_BIT_WISE_AND>(a, sa, b, sb, out, n, v, e, s);
      case B2_BIT_WISE_OR: return run_arith<T, B2_BIT_WISE_OR>(a, sa, b, sb, out, n, v, e, s);
      case B2_BIT_WISE_XOR: return run_arith<T, B2_BIT_WISE_XOR>(a, sa, b, sb, out, n, v, e, s);
      case B2_SHIFT_LEFT: return run_arith<T, B2_SHIFT_LEFT>(a, sa, b, sb, out, n, v, e, s);
      case B2_SHIFT_LEFT_CHECKED: return run_arith<T, B2_SHIFT_LEFT_CHECKED>(a, sa, b, sb, out, n, v, e, s);
      case B2_SHIFT_RIGHT: return run_arith<T, B2_SHIFT_RIGHT>(a, sa, b, sb, out, n, v, e, s);
      case B2_SHIFT_RIGHT_CHECKED: return run_arith<T, B2_SHIFT_RIGHT_CHECKED>(a, sa, b, sb, out, n, v, e, s);
      default: break;
    }
  }
  return set_error(B2_INVALID, "unknown arithmetic op %d", op);
}

}  // namespace b2

using namespace b2;

extern "C" int b2_binary_arith(B2Context* ctx, int op, const B2Value* left, const B2Value* right,
                               B2Array* out, void* stream) {
  if (!ctx || !out) return set_error(B2_INVALID, "b2_binary_arith: null argument");
  int type;
  int64_t n;
  bool null_scalar;
  B2_RETURN_NOT_OK(unpack_operands(left, right, &type, &n, &null_scalar));
  if (!type_is_numeric(type)) return set_error(B2_NOT_IMPLEMENTED, "arithmetic on type id %d", type);
  if (int_only_op(op) && (type == B2_FLOAT || type == B2_DOUBLE))
    return set_error(B2_NOT_IMPLEMENTED, "arithmetic op %d has no kernel matching input types (%s)", op,
                     type == B2_FLOAT ? "float" : "double");
  cudaStream_t s = ctx->pick(stream);
  B2_CUDA(cudaSetDevice(ctx->device));
  const B2Array* la = left->array;
  const B2Array* ra = right->array;
  const int w = type_width(type);

  Temp data(ctx, s);
  B2_RETURN_NOT_OK(data.alloc(static_cast<size_t>(n) * w));
  if (null_scalar) {
    // a null scalar operand nulls every slot (exec.cc:560-590 all-null propagation)
    Temp bits(ctx, s);
    B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(n)));
    B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bitmap_alloc_bytes(n), s));
    B2_CUDA(cudaMemsetAsync(data.ptr, 0, static_cast<size_t>(n) * w + (n == 0), s));
    fill_out(out, type, n, n, n ? bits.release() : nullptr, data.release());
    return B2_OK;
  }
  void* validity = nullptr;
  int64_t null_count = 0;
  B2_RETURN_NOT_OK(make_validity(ctx, la, ra, n, &validity, &null_count, s));
  Temp vguard(ctx, s);
  vguard.ptr = validity;
  if (n > 0) {
    // every checked op, and the two unchecked ones with an error: divide (by an integer zero) and power
    const bool can_fail = (op >= B2_ADD_CHECKED) || (op == B2_DIVIDE) || (op == B2_POWER);
    ScalarSlot slot(ctx);
    unsigned long long* d_err = nullptr;
    if (can_fail) {
      if (!slot.ok()) return set_error(B2_UNKNOWN_ERROR, "no free scalar slot");
      B2_CUDA(cudaMemsetAsync(slot.dev(), 0, 8, s));
      d_err = reinterpret_cast<unsigned long long*>(slot.dev());
    }
    B2_RETURN_NOT_OK(visit_type(NumericTypes{}, type, [&](auto tag) {
      using T = decltype(tag);
      const T* a = la ? static_cast<const T*>(la->data) + la->offset : nullptr;
      const T* b = ra ? static_cast<const T*>(ra->data) + ra->offset : nullptr;
      return run_arith_op<T>(op, a, scalar_bits<T>(left->scalar), b, scalar_bits<T>(right->scalar),
                             static_cast<T*>(data.ptr), n, validity, d_err, s);
    }));
    if (can_fail) {
      B2_RETURN_NOT_OK(slot.fetch(s));
      const uint64_t row1 = static_cast<uint64_t>(slot.host()[0]);
      if (row1 != 0) {
        const uint64_t row = row1 - 1;
        if (op == B2_SHIFT_LEFT_CHECKED || op == B2_SHIFT_RIGHT_CHECKED)
          return set_error(B2_INVALID, "shift amount must be >= 0 and less than precision of type");
        // classify from the right operand of that row: divide by zero vs overflow, negative exponent vs overflow
        uint64_t rv = 0;
        B2_RETURN_NOT_OK(operand_bits(right, static_cast<int64_t>(row), w, &rv, s));
        if (op == B2_POWER || op == B2_POWER_CHECKED) {
          const bool negative = type_is_signed_int(type) && ((rv >> (8 * w - 1)) & 1);
          return set_error(B2_INVALID, negative ? "integers to negative integer powers are not allowed" : "overflow");
        }
        bool zero = false;
        if (op == B2_DIVIDE || op == B2_DIVIDE_CHECKED) {
          if (type == B2_FLOAT) zero = (rv & 0x7fffffffull) == 0;
          else if (type == B2_DOUBLE) zero = (rv & 0x7fffffffffffffffull) == 0;
          else zero = rv == 0;
        }
        return set_error(B2_INVALID, zero ? "divide by zero" : "overflow");
      }
    }
  }
  fill_out(out, type, n, null_count, vguard.release(), data.release());
  return B2_OK;
}
