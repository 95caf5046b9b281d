/*
 * arrow_b200.h -- C-ABI of the GPU-native (H100) execution layer for arrow::compute's
 * ExecBatch hot path (Filter/Take, Cast, arithmetic/compare, SortIndices,
 * Grouper + hash aggregates).
 *
 * This is the drop-in boundary: every entry point below replaces one reference
 * kernel entry (an ArrayKernelExec, a Grouper method or a HashAggregateKernel
 * callback) and takes exactly the information the reference passes through an
 * ArraySpan (cpp/src/arrow/array/data.h:525-690): validity bitmap, data buffer(s),
 * length, offset, null_count, type id -- but with DEVICE addresses.  No torch, no
 * arrow C++ type appears in a signature; the C++ host plugin (arrow_b200/cpp) and
 * the Python ctypes mirror (arrow_b200/_cabi.py) both bind these symbols.
 *
 * Conventions
 *  - every function returns a B2Status (0 = OK); b2_last_error() gives the message
 *    for the calling thread.  Status codes map 1:1 to arrow::StatusCode
 *    (cpp/src/arrow/status.h:86-110) so the trampolines can rebuild the same Status.
 *  - all pointers inside B2Array are device pointers valid on ctx's device.
 *  - validity bitmaps and boolean data are LSB-first bit-packed
 *    (cpp/src/arrow/util/bit_util.h), addressed with `offset` in bits.
 *  - outputs are allocated through the context's allocator (built-in pool, or the
 *    callbacks the host installs with b2_context_set_allocator so memory stays in
 *    the host-side MemoryManager pool); ownership passes to the caller, who
 *    releases with b2_free().
 *  - calls are stream-ordered on `stream` (a cudaStream_t passed as void*; NULL =
 *    the context's own non-blocking stream).  Calls that return a length or a null
 *    count synchronise that stream once before returning (the one unavoidable
 *    read-back, SURVEY.md section 3.5).
 */
#ifndef ARROW_B200_H
#define ARROW_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2_API __attribute__((visibility("default")))

/* ---- status codes: values follow arrow::StatusCode (status.h:86-110) ---- */
typedef enum B2Status {
  B2_OK = 0,
  B2_OUT_OF_MEMORY = 1,
  B2_KEY_ERROR = 2,
  B2_TYPE_ERROR = 3,
  B2_INVALID = 4,
  B2_IO_ERROR = 5,
  B2_CAPACITY_ERROR = 6,
  B2_INDEX_ERROR = 7,
  B2_CANCELLED = 8,
  B2_UNKNOWN_ERROR = 9,
  B2_NOT_IMPLEMENTED = 10,
  B2_CUDA_ERROR = 100
} B2Status;

/* ---- type ids: values follow arrow::Type::type (type_fwd.h:328-460) ---- */
typedef enum B2Type {
  B2_NA = 0,
  B2_BOOL = 1,
  B2_UINT8 = 2,
  B2_INT8 = 3,
  B2_UINT16 = 4,
  B2_INT16 = 5,
  B2_UINT32 = 6,
  B2_INT32 = 7,
  B2_UINT64 = 8,
  B2_INT64 = 9,
  B2_HALF_FLOAT = 10,
  B2_FLOAT = 11,
  B2_DOUBLE = 12,
  B2_STRING = 13,
  B2_BINARY = 14,
  B2_FIXED_SIZE_BINARY = 15,
  B2_LIST = 25, /* list<T> with int32 offsets: only produced as offsets + child (b2_make_groupings,
                   b2_hashagg_finalize_list); no entry point takes it as an input */
  B2_LARGE_STRING = 34,
  B2_LARGE_BINARY = 35
} B2Type;

/* One ArraySpan with device addresses (array/data.h:525-690).
 *   fixed width : data  = values                       (data2 unused)
 *   bool        : data  = bit-packed values
 *   (large_)utf8/binary : data = int32/int64 offsets (length+1 entries, indexed
 *                 from `offset`), data2 = character bytes
 * byte_width is only read for B2_FIXED_SIZE_BINARY. */
typedef struct B2Array {
  const void* validity; /* NULL = no nulls */
  const void* data;
  const void* data2;
  int64_t length;
  int64_t offset;
  int64_t null_count; /* -1 = unknown (kUnknownNullCount) */
  int32_t type;       /* B2Type */
  int32_t byte_width;
} B2Array;

/* A Scalar operand (scalar.h): value bits in `bits` (little-endian, low bytes),
 * is_valid = 0 for a null scalar. */
typedef struct B2Scalar {
  uint64_t bits;
  int32_t type;
  int32_t is_valid;
} B2Scalar;

/* Binary-kernel operand: an array or a scalar (exec.h:275-330 ExecValue). */
typedef struct B2Value {
  const B2Array* array;   /* non-NULL => array operand */
  const B2Scalar* scalar; /* used when array == NULL */
} B2Value;

typedef struct B2Context B2Context;

/* ---------------------------------------------------------------------------
 * Context, device pool, streams.
 * Replaces: arrow::cuda::CudaContext / CudaMemoryManager allocation path
 * (cpp/src/arrow/gpu/cuda_context.cc:110-121 = one cuMemAlloc per buffer) with a
 * size-binned caching pool.
 * ------------------------------------------------------------------------- */
typedef void* (*B2AllocFn)(size_t nbytes, void* stream, void* user);
typedef void (*B2FreeFn)(void* ptr, size_t nbytes, void* stream, void* user);

B2_API int b2_context_create(int device, B2Context** out);
B2_API void b2_context_destroy(B2Context* ctx);
B2_API int b2_context_device(const B2Context* ctx);
B2_API void* b2_context_stream(const B2Context* ctx);
B2_API int b2_context_set_allocator(B2Context* ctx, B2AllocFn alloc, B2FreeFn free_fn,
                                    void* user);
B2_API int b2_alloc(B2Context* ctx, size_t nbytes, void** out);
B2_API int b2_free(B2Context* ctx, void* ptr);
B2_API int b2_pool_stats(const B2Context* ctx, int64_t* bytes_in_use,
                         int64_t* bytes_reserved, int64_t* max_in_use);
B2_API int b2_pool_trim(B2Context* ctx);
B2_API int b2_sync(B2Context* ctx, void* stream);
B2_API int b2_memcpy_h2d(B2Context* ctx, void* dst, const void* src, size_t n, void* stream);
B2_API int b2_memcpy_d2h(B2Context* ctx, void* dst, const void* src, size_t n, void* stream);
B2_API int b2_memset(B2Context* ctx, void* dst, int byte, size_t n, void* stream);
/* Events (cudaEvent_t as void*): the synchronisation object of the C Device Data Interface --
 * ArrowDeviceArray.sync_event is a cudaEvent_t* for ARROW_DEVICE_CUDA (c/abi.h:140-157); the producer
 * records it after the last kernel that writes the buffers, the consumer makes its stream wait on it
 * (arrow::Device::SyncEvent / Stream::WaitEvent, device.h:86-165). */
B2_API int b2_event_create(B2Context* ctx, void** out_event);
B2_API int b2_event_destroy(void* event);
B2_API int b2_event_record(B2Context* ctx, void* event, void* stream);
B2_API int b2_event_synchronize(void* event);
B2_API int b2_stream_wait_event(B2Context* ctx, void* stream, void* event);
/* pinned host staging (CudaHostBuffer, cuda_memory.h:113) */
B2_API int b2_host_alloc(size_t nbytes, void** out);
B2_API int b2_host_free(void* ptr);

B2_API const char* b2_last_error(void);
B2_API const char* b2_version(void);
/* number of kernels this library has launched in this process (bench.py's
 * gpu_launches claim) */
B2_API int64_t b2_launch_count(void);

/* ---------------------------------------------------------------------------
 * Bitmap utilities.  Replaces internal::CopyBitmap / BitmapAnd / CountSetBits
 * (cpp/src/arrow/util/bitmap_ops.cc) as used by NullPropagator
 * (cpp/src/arrow/compute/exec.cc:527-686).
 * ------------------------------------------------------------------------- */
/* number of set bits in bits[offset, offset+length) */
B2_API int b2_bitmap_count(B2Context* ctx, const void* bits, int64_t offset, int64_t length,
                           int64_t* out_count, void* stream);
/* dst[dst_offset..] = src[src_offset..]; dst must be a fresh buffer, padding zeroed */
B2_API int b2_bitmap_copy(B2Context* ctx, const void* src, int64_t src_offset, int64_t length,
                          void* dst, void* stream);
/* dst = a & b (either may be NULL = all ones); returns popcount if out_count != NULL */
B2_API int b2_bitmap_and(B2Context* ctx, const void* a, int64_t a_offset, const void* b,
                         int64_t b_offset, int64_t length, void* dst, int64_t* out_count,
                         void* stream);

/* ---------------------------------------------------------------------------
 * Cast.  Replaces CastNumberToNumberUnsafe + the safety checks
 * (kernels/scalar_cast_internal.cc:41-53,155; kernels/scalar_cast_numeric.cc:45-279).
 * out is allocated by the callee (data + validity copy at offset 0).
 * ------------------------------------------------------------------------- */
typedef struct B2CastOptions { /* compute/cast.h CastOptions */
  int32_t to_type;
  int32_t allow_int_overflow;
  int32_t allow_float_truncate;
  int32_t reserved;
} B2CastOptions;
B2_API int b2_cast_numeric(B2Context* ctx, const B2Array* in, const B2CastOptions* options,
                           B2Array* out, void* stream);

/* ---------------------------------------------------------------------------
 * Temporal types.  A temporal array keeps its storage type id in B2Array (B2_INT32 for date32 / time32, B2_INT64 for
 * date64 / time64 / timestamp / duration); a B2TemporalType says what the storage means.
 *   kind           : B2TemporalKind; B2_TEMPORAL_INT32 / INT64 are plain integers (the zero-copy relabels)
 *   unit           : B2TimeUnit for time32 (s, ms), time64 (us, ns), timestamp and duration; ignored for dates
 *   has_zone       : timestamp only: 1 for a zoned timestamp (UTC or a fixed offset), 0 for a naive one
 *   offset_minutes : the zone's fixed offset from UTC ("UTC" is 0, "+05:30" is 330, "-0800" is -480).  Named zones
 *                    with transitions have no descriptor: the caller refuses them.
 * ------------------------------------------------------------------------- */
typedef enum B2TemporalKind {
  B2_TEMPORAL_DATE32 = 0,
  B2_TEMPORAL_DATE64 = 1,
  B2_TEMPORAL_TIME32 = 2,
  B2_TEMPORAL_TIME64 = 3,
  B2_TEMPORAL_TIMESTAMP = 4,
  B2_TEMPORAL_DURATION = 5,
  B2_TEMPORAL_INT32 = 6,
  B2_TEMPORAL_INT64 = 7
} B2TemporalKind;
typedef enum B2TimeUnit { B2_SECOND = 0, B2_MILLI = 1, B2_MICRO = 2, B2_NANO = 3 } B2TimeUnit;
typedef struct B2TemporalType {
  int32_t kind;
  int32_t unit;
  int32_t has_zone;
  int32_t offset_minutes;
} B2TemporalType;

/* Cast between temporal types.  Replaces kernels/scalar_cast_temporal.cc: ShiftTime (:46-123) for timestamp ->
 * timestamp and duration -> duration across units (:149-175), time32 / time64 across units (:348-365), date32 <->
 * date64 (:370-384) and date -> timestamp (:389-414); the Date32 / Date64 / ExtractTime* functors for timestamp ->
 * date32 / date64 / time32 / time64 (:180-343), in local time for a zoned timestamp (ZonedLocalizer,
 * temporal_internal.h); and the zero-copy relabels of the same storage (GetDate32Cast ... GetTimestampCast :518-659,
 * scalar_cast_numeric.cc:1101-1111).  The accepted (from, to) pairs are exactly those; any other gives
 * B2_NOT_IMPLEMENTED "Unsupported cast from X to Y using function cast_Z".
 *   in : storage of `from`; out: storage of `to` (callee-allocated), validity = the input's re-based to offset 0.
 *   A multiplying unit change checks overflow unless allow_time_overflow (B2_INVALID "Casting from X to Y would result
 *   in out of bounds timestamp: V"); a dividing one checks for a remainder unless allow_time_truncate ("... would lose
 *   data: V", or "Cast would lose data: V" from timestamp to a time of day), and otherwise truncates toward zero.
 *   Only valid slots are checked; the error names the first offending row.  A zoned type is written in a message with
 *   its offset ("tz=+05:30"; "tz=UTC" for offset 0).  One kernel launch (plus one when the input has nulls).
 * ------------------------------------------------------------------------- */
B2_API int b2_cast_temporal(B2Context* ctx, const B2Array* in, const B2TemporalType* from, const B2TemporalType* to,
                            int allow_time_truncate, int allow_time_overflow, B2Array* out, void* stream);

/* Calendar and clock fields.  Replaces the Year / Month / Day / DayOfYear / DayOfWeek / Quarter / IsLeapYear / Hour /
 * Minute / Second / Millisecond / Microsecond / Nanosecond / Subsecond extractors of kernels/scalar_temporal_unary.cc
 * (:222-691) with DayOfWeekOptions (compute/api_scalar.h).  Date fields take date32 / date64 / timestamp, clock fields
 * time32 / time64 / timestamp; other types give B2_NOT_IMPLEMENTED.  A zoned timestamp's date fields, hour and minute
 * are those of its local time.  Far-out values wrap exactly as the reference's 32-bit day count and 16-bit year do.
 *   out: B2_INT64, B2_DOUBLE for subsecond, B2_BOOL (bit-packed) for is_leap_year; validity = the input's, re-based.
 *   week_start (1 = Monday .. 7 = Sunday, else B2_INVALID) and count_from_zero are read by day_of_week only.
 * One kernel launch (plus one when the input has nulls).
 * ------------------------------------------------------------------------- */
typedef enum B2TemporalField {
  B2_FIELD_YEAR = 0,
  B2_FIELD_MONTH = 1,
  B2_FIELD_DAY = 2,
  B2_FIELD_DAY_OF_YEAR = 3,
  B2_FIELD_DAY_OF_WEEK = 4,
  B2_FIELD_QUARTER = 5,
  B2_FIELD_IS_LEAP_YEAR = 6,
  B2_FIELD_HOUR = 7,
  B2_FIELD_MINUTE = 8,
  B2_FIELD_SECOND = 9,
  B2_FIELD_MILLISECOND = 10,
  B2_FIELD_MICROSECOND = 11,
  B2_FIELD_NANOSECOND = 12,
  B2_FIELD_SUBSECOND = 13
} B2TemporalField;
B2_API int b2_temporal_field(B2Context* ctx, const B2Array* in, const B2TemporalType* type, int field,
                             int week_start, int count_from_zero, B2Array* out, void* stream);

/* ---------------------------------------------------------------------------
 * Arithmetic.  Replaces ScalarBinary<..>::{ArrayArray,ArrayScalar,ScalarArray}
 * with the Add/Subtract/Multiply(+Checked)/Divide op functors
 * (kernels/codegen_internal.h:813-976, kernels/base_arithmetic_internal.h:44-330).
 * Both operands must already have the same (dispatched) type, as after
 * ArithmeticFunction::DispatchBest (kernels/scalar_arithmetic.cc:734-781).
 * ------------------------------------------------------------------------- */
typedef enum B2ArithOp {
  B2_ADD = 0,
  B2_SUBTRACT = 1,
  B2_MULTIPLY = 2,
  B2_DIVIDE = 3,
  /* integers only (B2_NOT_IMPLEMENTED on floats): Power, BitWiseAnd / Or / Xor, ShiftLeft, ShiftRight
   * (base_arithmetic_internal.h:558-584, scalar_arithmetic.cc:72-149).  power raises B2_INVALID "integers to negative
   * integer powers are not allowed" for a negative exponent in ANY slot, null slots included (it is a plain
   * ScalarBinary); otherwise it wraps.  A shift amount outside [0, digits) (digits = 7 / 15 / 31 / 63 for the signed
   * types, 8 / 16 / 32 / 64 for the unsigned ones) returns the left operand. */
  B2_POWER = 4,
  B2_BIT_WISE_AND = 5,
  B2_BIT_WISE_OR = 6,
  B2_BIT_WISE_XOR = 7,
  B2_SHIFT_LEFT = 8,
  B2_SHIFT_RIGHT = 9,
  B2_ADD_CHECKED = 16,
  B2_SUBTRACT_CHECKED = 17,
  B2_MULTIPLY_CHECKED = 18,
  B2_DIVIDE_CHECKED = 19,
  /* PowerChecked ("overflow", or the negative-exponent text) and ShiftLeftChecked / ShiftRightChecked ("shift amount
   * must be >= 0 and less than precision of type", nothing else checked): valid slots only
   * (base_arithmetic_internal.h:586-618, scalar_arithmetic.cc:106-161) */
  B2_POWER_CHECKED = 20,
  B2_SHIFT_LEFT_CHECKED = 21,
  B2_SHIFT_RIGHT_CHECKED = 22
} B2ArithOp;
B2_API int b2_binary_arith(B2Context* ctx, int op, const B2Value* left, const B2Value* right,
                           B2Array* out, void* stream);

/* ---------------------------------------------------------------------------
 * Unary numeric math.  Replaces ScalarUnary / ScalarUnaryNotNull over AbsoluteValue(Checked), Negate(Checked), Sign,
 * SquareRoot(Checked) (base_arithmetic_internal.h:126-170,471-530,620-660), BitWiseNot (scalar_arithmetic.cc:65-70)
 * and Floor / Ceil / Trunc (scalar_round.cc:1011-1036).
 *   in : abs, abs_checked, negate, sign: the eight integer types and float32 / float64; negate_checked: the signed
 *        integers and the floats; bit_wise_not: the integers; sqrt, sqrt_checked, floor, ceil, trunc: float32 /
 *        float64 (the caller casts an integer input to float64 first, as RoundIntegerToFloatingPointFunction /
 *        ArithmeticIntegerToFloatingPointFunction do).  Any other type gives B2_NOT_IMPLEMENTED "Function 'F' has no
 *        kernel matching input types (T)".
 *   out: the input's type, except sign over an integer: B2_INT8; validity = the input's, re-based.
 *   Unchecked integer ops wrap (abs(INT_MIN) = INT_MIN).  abs_checked / negate_checked raise B2_INVALID "overflow", and
 *   sqrt_checked "square root of negative number", for a valid slot only.  sign(-0.0) = +0.0; sign and abs keep a
 *   NaN's payload.  One kernel launch (plus one when the input has nulls).
 * ------------------------------------------------------------------------- */
typedef enum B2UnaryOp {
  B2_ABS = 0,
  B2_NEGATE = 1,
  B2_SIGN = 2,
  B2_SQRT = 3,
  B2_FLOOR = 4,
  B2_CEIL = 5,
  B2_TRUNC = 6,
  B2_BIT_WISE_NOT = 7,
  B2_ABS_CHECKED = 16,
  B2_NEGATE_CHECKED = 17,
  B2_SQRT_CHECKED = 18
} B2UnaryOp;
B2_API int b2_unary_arith(B2Context* ctx, int op, const B2Array* in, B2Array* out, void* stream);

/* ---------------------------------------------------------------------------
 * round, round_to_multiple and round_binary over the eight integer types and float32 / float64.  Replaces Round,
 * RoundToMultiple and RoundBinary with RoundImpl and RoundUtil::Pow10 (scalar_round.cc:89-102,141-418,527-565,
 * 725-765,865-911,960-1009) under RoundOptions / RoundToMultipleOptions / RoundBinaryOptions (compute/api_scalar.h).
 * The function is picked by which operand is given:
 *   digits != NULL  : round_binary(x, digits).  x: an array or scalar; digits: a B2_INT32 array or scalar (at least
 *                     one of the two is an array, arrays of one length); a null scalar nulls every row.
 *   multiple != NULL: round_to_multiple(x, multiple).  x: an array; multiple: a scalar of x's type (the caller applies
 *                     the safe cast); null gives B2_INVALID "Rounding multiple must be non-null and valid", <= 0
 *                     "Rounding multiple must be positive" (a float +0 is let through, -0.0 is not: the reference checks
 *                     the sign before its cast, which can turn a tiny positive float64 into float32 +0).
 *   else            : round(x, ndigits).  For an integer x, -ndigits above digits10 of its type gives B2_INVALID
 *                     "Rounding to N digits is out of range for type T" before any kernel runs.
 *   round_mode      : a B2RoundMode.
 * A float is rounded by the reference's sequence of IEEE operations: a non-finite value passes through, the value is
 * scaled by Pow10 (its table is float literals: 10^11 is 99999997952), a scaled value already on the grid returns the
 * input itself, a tie mode takes round-half-away unless the fraction is exactly 0.5, and a non-finite unscaled result
 * gives B2_INVALID "overflow occurred during rounding".  round scales a float32 in float32; round_binary in float64.
 * An integer is rounded to a multiple of 10^-ndigits, or of `multiple`; an overflow gives B2_INVALID "Rounding X up
 * to multiple of M would overflow" (or "down", or "multiples" from the nearest-value branch).  Only valid rows are
 * checked; when several fail, the message is the last one's.  out: x's type; validity = AND of the inputs', re-based.
 * One kernel launch (plus one when an input's validity is re-based).
 * ------------------------------------------------------------------------- */
typedef enum B2RoundMode { /* values follow arrow::compute::RoundMode (compute/api_scalar.h:58-100) */
  B2_ROUND_DOWN = 0,
  B2_ROUND_UP = 1,
  B2_ROUND_TOWARDS_ZERO = 2,
  B2_ROUND_TOWARDS_INFINITY = 3,
  B2_ROUND_HALF_DOWN = 4,
  B2_ROUND_HALF_UP = 5,
  B2_ROUND_HALF_TOWARDS_ZERO = 6,
  B2_ROUND_HALF_TOWARDS_INFINITY = 7,
  B2_ROUND_HALF_TO_EVEN = 8,
  B2_ROUND_HALF_TO_ODD = 9
} B2RoundMode;
B2_API int b2_round(B2Context* ctx, const B2Value* x, const B2Value* digits, int64_t ndigits, const B2Scalar* multiple,
                    int round_mode, B2Array* out, void* stream);

/* ---------------------------------------------------------------------------
 * Cumulative functions over one array or the chunks of one ChunkedArray.  Replaces CumulativeBinaryOp /
 * CumulativeMean, Accumulator, CumulativeKernel and CumulativeKernelChunked (kernels/vector_cumulative_ops.cc:67-203,
 * registered at :341-359) under CumulativeOptions{start, skip_nulls} (compute/api_vector.h:335-355).
 *   chunks  : n_chunks >= 1 arrays of one type, the eight integer types or float32 / float64 (any other type gives
 *             B2_NOT_IMPLEMENTED "Function 'F' has no kernel matching input types (T)"); any bit offset.
 *   start   : a scalar of the input's type (the caller applies the safe cast, CumulativeOptionsWrapper::Init :45-64), or
 *             NULL for the op's identity (Identity<Op>, base_arithmetic_internal.h:722-775): sum 0, prod 1, min
 *             numeric_limits<T>::max(), max numeric_limits<T>::min() -- for floats the largest finite value and the
 *             smallest positive normal.  A null scalar contributes the value bits it carries.  Mean ignores it.
 *   out     : ONE array over all chunks, the input's type (mean: B2_DOUBLE).  Row i is Op(x_i, Op(x_{i-1}, ... start)),
 *             integer sum / prod wrapping; float min / max ignore NaN and return the newer value on a tie, so
 *             cumulative_min([0.0, -0.0]) is [0.0, -0.0].  skip_nulls: a null row is null (value 0) and leaves the
 *             state alone.  Otherwise every row from the first null on is null, and an input without nulls gives an
 *             output without validity.  null_count is exact.
 *   checked : *_CHECKED over an integer type raise B2_INVALID "overflow" when a combined row overflows, the start's
 *             first step included; rows after the first null under skip_nulls = 0 are not combined and never raise.
 * Float sums, products and means are combined in tile order, not row by row, so they can differ from the sequential
 * fold in the last bits.  One kernel launch per non-empty chunk; a zero-length input launches nothing.
 * ------------------------------------------------------------------------- */
typedef enum B2CumulativeOp {
  B2_CUMULATIVE_SUM = 0,
  B2_CUMULATIVE_SUM_CHECKED = 1,
  B2_CUMULATIVE_PROD = 2,
  B2_CUMULATIVE_PROD_CHECKED = 3,
  B2_CUMULATIVE_MIN = 4,
  B2_CUMULATIVE_MAX = 5,
  B2_CUMULATIVE_MEAN = 6
} B2CumulativeOp;
B2_API int b2_cumulative(B2Context* ctx, int op, const B2Array* chunks, int32_t n_chunks,
                         const B2Scalar* start /* NULL: the op's identity */, int skip_nulls, B2Array* out,
                         void* stream);

/* ---------------------------------------------------------------------------
 * Compare -> bit-packed boolean.  Replaces CompareKernel::Exec
 * (kernels/scalar_compare.cc:164-303).  less/less_equal are the flipped
 * greater/greater_equal exactly as MakeFlippedCompare does (:910).
 * ------------------------------------------------------------------------- */
typedef enum B2CompareOp {
  B2_EQUAL = 0,
  B2_NOT_EQUAL = 1,
  B2_GREATER = 2,
  B2_GREATER_EQUAL = 3,
  B2_LESS = 4,
  B2_LESS_EQUAL = 5
} B2CompareOp;
B2_API int b2_compare(B2Context* ctx, int op, const B2Value* left, const B2Value* right,
                      B2Array* out, void* stream);

/* ---------------------------------------------------------------------------
 * Compare over utf8 / large_utf8 / binary / large_binary.  Replaces CompareKernel over BaseBinaryTypes and the
 * string_view ordering (kernels/scalar_compare.cc:42-72,431-433); CompareFunction::DispatchBest's cast of mixed
 * binary-like arguments to CommonBinary (:340-366) is not needed: any pair of the four types is read directly, each
 * side with its own offset width.
 *   left   : binary-like array
 *   right  : binary-like array of the same length, or NULL for a scalar: its host bytes [scalar, scalar + scalar_length)
 *            and scalar_valid (0: a null scalar, an all-null result).  A scalar-array call is the array-scalar call
 *            with the operator flipped (less <-> greater, less_equal <-> greater_equal).
 * out: B2_BOOL, validity = AND of the input validities; the data bits are computed on every slot, nulls included
 * (unsigned bytewise order, a proper prefix first; a null scalar compares as the empty string).  All six B2CompareOp.
 * Synchronises only to count the output's nulls, as b2_compare does.
 * ------------------------------------------------------------------------- */
B2_API int b2_compare_binary(B2Context* ctx, int op, const B2Array* left, const B2Array* right, const void* scalar,
                             int64_t scalar_length, int scalar_valid, B2Array* out, void* stream);

/* ---------------------------------------------------------------------------
 * match_substring / starts_with / ends_with / match_like over utf8 / large_utf8 / binary / large_binary.  Replaces
 * PlainSubstringMatcher, PlainStartsWithMatcher, PlainEndsWithMatcher (kernels/scalar_string_ascii.cc:1221-1307) and
 * MatchLike::Exec with its classifying regexes and MakeLikeRegex (:1456-1588); MatchSubstringOptions
 * compute/api_scalar.h.  ignore_case is not on the device (the reference folds case with RE2's Unicode tables).
 *   kind    : B2_MATCH_SUBSTRING / STARTS_WITH / ENDS_WITH (a byte match of the pattern; "" matches every row) or
 *             B2_MATCH_LIKE (SQL LIKE: `%`, `_`, `\` escapes).  Create classifies a LIKE pattern once, as MatchLike does:
 *             %lit% / lit% / %lit run as the substring / prefix / suffix match of lit, anything else as an anchored
 *             segment matcher where `_` is one code point (is_utf8) or one byte.
 *   is_utf8 : the input type the handle serves (utf8 / large_utf8 vs binary / large_binary); a LIKE pattern that is not
 *             valid UTF-8 gives B2_INVALID "Invalid regular expression: invalid UTF-8" when is_utf8 is set.
 * b2_string_match: out B2_BOOL, validity = the input's; data bits computed on every slot.  An input whose utf8-ness
 * differs from the handle's gives B2_TYPE_ERROR.  One kernel launch (two when the input has nulls).
 * b2_string_match_info: what the pattern runs as (a B2StringMatchKind; B2_MATCH_LIKE = the general matcher) and the
 * bytes of its literal (items of the general program).
 * ------------------------------------------------------------------------- */
typedef enum B2StringMatchKind {
  B2_MATCH_SUBSTRING = 0,
  B2_MATCH_STARTS_WITH = 1,
  B2_MATCH_ENDS_WITH = 2,
  B2_MATCH_LIKE = 3
} B2StringMatchKind;
typedef struct B2StringMatch B2StringMatch;
B2_API int b2_string_match_create(B2Context* ctx, int kind, const void* pattern, int64_t pattern_length, int is_utf8,
                                  B2StringMatch** out, void* stream);
B2_API void b2_string_match_destroy(B2StringMatch* h);
B2_API int b2_string_match_info(const B2StringMatch* h, int32_t* runs_as, int64_t* literal_bytes);
B2_API int b2_string_match(B2StringMatch* h, const B2Array* strings, B2Array* out, void* stream);

/* ---------------------------------------------------------------------------
 * String transforms over utf8 / large_utf8 / binary / large_binary.  Each output's validity is the input's, re-based,
 * except the join's.  A type the reference registers no kernel for gives B2_NOT_IMPLEMENTED.
 * b2_string_length: binary_length (is_utf8 = 0; BinaryLength, kernels/scalar_string_ascii.cc:852-880, any of the four
 *   types) or utf8_length (is_utf8 = 1; Utf8Length, kernels/scalar_string_utf8.cc:664-690, utf8 / large_utf8: the
 *   bytes that are not 10xxxxxx, util/utf8_internal.h:558, nothing validated).  out: B2_INT32 for int32 offsets,
 *   B2_INT64 for int64 offsets, computed on every slot.  One kernel launch (plus one when the input has nulls).
 * b2_ascii_case: ascii_upper (upper = 1) / ascii_lower over utf8 / large_utf8 (AsciiUpper / AsciiLower over
 *   StringDataTransform, kernels/scalar_string_ascii.cc:724-745,834-842).  out: the input's offsets re-based to 0 and
 *   its bytes [offsets[0], offsets[n]) with a..z / A..Z mapped, null slots included.  Synchronises once (for the byte
 *   count); one kernel launch (plus one when the input has nulls).
 * b2_string_slice: utf8_slice_codeunits (is_utf8 = 1, utf8 / large_utf8: start / stop / step count code points,
 *   SliceCodeunitsTransform kernels/scalar_string_utf8.cc:1157-1348) or binary_slice (is_utf8 = 0, binary /
 *   large_binary: bytes, SliceBytesTransform kernels/scalar_string_ascii.cc:2636-2800) under SliceOptions
 *   (compute/api_scalar.h).  step == 0 gives B2_INVALID "Slice step cannot be zero"; a UTF-8 decode error where a
 *   valid row is walked gives B2_INVALID "Invalid UTF8 sequence in input".  A null row is an empty value.  Synchronises
 *   once; three kernel launches (plus one when the input has nulls).
 * b2_binary_join_element_wise: BinaryJoinElementWise (kernels/scalar_string_ascii.cc:3298-3420) under JoinOptions.
 *   operands[0 .. n-2] are the values and operands[n-1] the separator; each is an array (every array of one type and
 *   one length, at least one array) or host bytes with a validity flag.  A row is null when its separator is, or, under
 *   B2_JOIN_EMIT_NULL, when any value is; B2_JOIN_SKIP drops a null value and its separator, B2_JOIN_REPLACE joins
 *   `replacement` in its place; with the separator alone every valid row is "".  Over int32 offsets an output of more
 *   than 2147483646 bytes gives B2_CAPACITY_ERROR "array cannot contain more than 2147483646 bytes, have N"
 *   (BaseBinaryBuilder::ReserveData).  Synchronises once; three kernel launches.
 * ------------------------------------------------------------------------- */
typedef enum B2JoinNullHandling { B2_JOIN_EMIT_NULL = 0, B2_JOIN_SKIP = 1, B2_JOIN_REPLACE = 2 } B2JoinNullHandling;
typedef struct B2JoinOperand {
  const B2Array* array; /* non-NULL: an array operand */
  const void* bytes;    /* otherwise a scalar: its host bytes [bytes, bytes + length) and validity */
  int64_t length;
  int32_t is_valid;
  int32_t reserved;
} B2JoinOperand;
B2_API int b2_string_length(B2Context* ctx, const B2Array* strings, int is_utf8, B2Array* out, void* stream);
B2_API int b2_ascii_case(B2Context* ctx, const B2Array* strings, int upper, B2Array* out, void* stream);
B2_API int b2_string_slice(B2Context* ctx, const B2Array* strings, int64_t start, int64_t stop, int64_t step, int is_utf8,
                           B2Array* out, void* stream);
B2_API int b2_binary_join_element_wise(B2Context* ctx, const B2JoinOperand* operands, int n_operands, int null_handling,
                                       const void* replacement, int64_t replacement_length, B2Array* out, void* stream);

/* ---------------------------------------------------------------------------
 * Boolean logic and validity predicates (what a filter Expression is made of; SURVEY.md 8f rank 3).
 * Replaces AndOp / OrOp / XorOp / AndNotOp / InvertOp and the Kleene variants
 * (kernels/scalar_boolean.cc:30-270) and IsValidExec / IsNullExec / TrueUnlessNullExec / is_nan
 * (kernels/scalar_validity.cc:35-311; NullOptions{nan_is_null} compute/api_scalar.h).
 * Operands are B2_BOOL arrays (or one B2_BOOL scalar); `right` is NULL for B2_BOOL_INVERT.
 * ------------------------------------------------------------------------- */
typedef enum B2BooleanOp {
  B2_BOOL_AND = 0,
  B2_BOOL_OR = 1,
  B2_BOOL_XOR = 2,
  B2_BOOL_AND_NOT = 3,
  B2_BOOL_AND_KLEENE = 4,
  B2_BOOL_OR_KLEENE = 5,
  B2_BOOL_AND_NOT_KLEENE = 6,
  B2_BOOL_INVERT = 7
} B2BooleanOp;
B2_API int b2_boolean(B2Context* ctx, int op, const B2Value* left, const B2Value* right, B2Array* out,
                      void* stream);
typedef enum B2ValidityOp {
  B2_IS_VALID = 0,
  B2_IS_NULL = 1,          /* nan_is_null != 0: NaN values of float arrays count as null too */
  B2_TRUE_UNLESS_NULL = 2,
  B2_IS_NAN = 3            /* float32 / float64 only; null in -> null out */
} B2ValidityOp;
B2_API int b2_validity(B2Context* ctx, int op, const B2Array* in, int nan_is_null, B2Array* out,
                       void* stream);

/* if_else(cond, left, right).  Replaces IfElseFunctor<Type>::Call and the AAA/ASA/AAS/ASS shapes
 * (kernels/scalar_if_else.cc:62-520): out = cond ? left : right; out is null where cond is null or the chosen side
 * is.  cond: boolean array or scalar; left / right: arrays or scalars of ONE fixed-width numeric or boolean type (the
 * caller applies DispatchBest's casts); at least one of the three is an array, arrays agree in length
 * (else B2_INVALID "Array arguments must all be the same length"). */
B2_API int b2_if_else(B2Context* ctx, const B2Value* cond, const B2Value* left, const B2Value* right,
                      B2Array* out, void* stream);

/* ---------------------------------------------------------------------------
 * Filter.  Replaces PrimitiveFilterExec / BinaryFilterExec /
 * DictionaryFilterExec (kernels/vector_selection_filter_internal.cc:445-510,
 * 806-856,871-881) and GetFilterOutputSize (:62-114).
 * null_selection: 0 = DROP, 1 = EMIT_NULL (compute/api_vector.h:37-51).
 * mask is a B2_BOOL array.
 * ------------------------------------------------------------------------- */
B2_API int b2_filter_output_size(B2Context* ctx, const B2Array* mask, int null_selection,
                                 int64_t* out_length, void* stream);
B2_API int b2_filter(B2Context* ctx, const B2Array* values, const B2Array* mask,
                     int null_selection, B2Array* out, void* stream);
/* mask -> selection indices (GetTakeIndices, vector_selection_take_internal.cc:62-305);
 * out type is B2_UINT32 if mask length <= UINT32_MAX else error as the reference. */
B2_API int b2_filter_indices(B2Context* ctx, const B2Array* mask, int null_selection,
                             B2Array* out, void* stream);

/* ---------------------------------------------------------------------------
 * Take.  Replaces FixedWidthTakeExec / Gather / VarBinaryTakeExec / DictionaryTake
 * (kernels/vector_selection_take_internal.cc:336-497, kernels/gather_internal.h:84-251)
 * and CheckIndexBounds (util/int_util.cc:452-560).
 * ------------------------------------------------------------------------- */
B2_API int b2_take(B2Context* ctx, const B2Array* values, const B2Array* indices,
                   int boundscheck, B2Array* out, void* stream);

/* Fused Take -> Cast -> arithmetic: out[i] = op(cast<to_type>(values[indices[i]]), other[i]) in one pass, i.e. the
 * Expression add(cast(take(values, indices), T), other) that ExecuteScalarExpression (compute/expression.cc:722-797) runs
 * as three kernels with two materialised intermediates.  Results are identical to b2_take + b2_cast_numeric(unsafe) +
 * b2_binary_arith: same validity (indices AND values-at-index AND other), same IndexError, one IEEE operation per slot.
 * values: float64 / float32 / int64 / int32; indices: 32- or 64-bit integers; to_type: B2_FLOAT or B2_DOUBLE;
 * op: B2_ADD / B2_SUBTRACT / B2_MULTIPLY; other: array (or valid scalar) of to_type. */
B2_API int b2_take_cast_arith(B2Context* ctx, const B2Array* values, const B2Array* indices, int32_t to_type, int op,
                              const B2Value* other, B2Array* out, void* stream);

/* Bytes of character data a (large_)utf8/binary array spans: offsets[offset+length] -
 * offsets[offset] (one D2H read).  Lets the host size the data buffer of an output the
 * way BufferSpan::size does (array/data.h:525-532). */
B2_API int b2_binary_data_size(B2Context* ctx, const B2Array* array, int64_t* out_bytes, void* stream);

/* ---------------------------------------------------------------------------
 * SortIndices.  Replaces ArraySortIndices::Exec + ArrayCompareSorter /
 * ArrayCountSorter (kernels/vector_array_sort.cc:144-446,524-540) and
 * PartitionNullsAndNans (kernels/vector_sort_internal.h:113-305).
 * order: 0 = Ascending, 1 = Descending; null_placement: 0 = AtStart, 1 = AtEnd
 * (compute/ordering.h:30-44).  out: B2_UINT64, length = values.length, no nulls.
 * values: numeric or (large_)utf8 / (large_)binary (byte-lexicographic on unsigned bytes, a
 * proper prefix first; ArrayCompareSorter, vector_array_sort.cc:144-178), < 2^32 - 8192 rows.
 * ------------------------------------------------------------------------- */
B2_API int b2_sort_indices(B2Context* ctx, const B2Array* values, int order,
                           int null_placement, B2Array* out, void* stream);
/* The same stable sort, but row i carries payload[i] (B2_UINT32, no nulls) instead of its row number i:
 * out[k] = payload of the k-th row in sorted order (B2_UINT64).  The owner GPU of the distributed SortIndices sorts the
 * received (key, global row) pairs with it, so the row numbers ride along the radix passes instead of being gathered
 * afterwards (b2_sort_indices + b2_take = a second, random-access-bound pass). */
B2_API int b2_sort_payload(B2Context* ctx, const B2Array* values, const B2Array* payload, int order,
                           int null_placement, B2Array* out, void* stream);
/* Multi-key SortIndices (record batch / table sort, kernels/vector_sort.cc:386-600,850-1027): rows ordered by keys[0],
 * ties by keys[1], ...; orders[k] = 0 ascending / 1 descending per key; one null placement (0 = AtStart, 1 = AtEnd); stable.  Every key column
 * is numeric or (large_)utf8 / (large_)binary, and all are of the same length (< 2^32 - 8192 rows).  out: B2_UINT64 row indices. */
B2_API int b2_sort_indices_multi(B2Context* ctx, const B2Array* keys, int n_keys, const int32_t* orders,
                                 int null_placement, B2Array* out, void* stream);

/* select_k_unstable over one numeric or (large_)utf8 / (large_)binary column (ArraySelector, kernels/vector_select_k.cc:157-232): out = the B2_UINT64
 * indices of the first min(k, length) rows in sort order = b2_sort_indices(...)[0:k] (ties in row order).  For k << n the
 * column is read once: a sampled threshold, one compare pass, a sort of the few candidates (csrc/select_k.cu). */
B2_API int b2_select_k(B2Context* ctx, const B2Array* values, int64_t k, int order, int null_placement,
                       B2Array* out, void* stream);

/* ---------------------------------------------------------------------------
 * Hash join: the matching row pairs of an equi-join.  Replaces the build / probe / match core of HashJoinNode
 * (acero/hash_join_node.cc, acero/swiss_join.cc; JoinType acero/options.h:365-374, JoinKeyCmp::EQ :384-392: a null key
 * matches nothing).  left_keys / right_keys: n_keys columns each, pairwise of equal type (anything the Grouper takes).
 *   INNER       out_left[k], out_right[k] (B2_UINT32, no nulls) = the k-th matching pair
 *   LEFT_OUTER  as INNER plus one pair per unmatched left row whose out_right slot is null
 *   FULL_OUTER  as LEFT_OUTER, followed by one pair per unmatched right row whose out_left slot is null
 *   LEFT_SEMI / LEFT_ANTI   out_left = the left rows with / without a match (out_right may be NULL)
 * Pairs come in left-row order, the matches of one left row in right-row order (the reference's order is unspecified).
 * The caller gathers the payload columns with b2_take, as HashJoinNode's materialize step does.
 * ------------------------------------------------------------------------- */
typedef enum B2JoinType {
  B2_JOIN_INNER = 0,
  B2_JOIN_LEFT_OUTER = 1,
  B2_JOIN_LEFT_SEMI = 2,
  B2_JOIN_LEFT_ANTI = 3,
  B2_JOIN_FULL_OUTER = 4
} B2JoinType;
B2_API int b2_hash_join(B2Context* ctx, const B2Array* left_keys, const B2Array* right_keys, int n_keys, int join_type,
                        B2Array* out_left, B2Array* out_right, void* stream);
/* b2_hash_join with a comparison per key column (JoinKeyCmp, acero/options.h:384-392): null_equal[j] != 0 is IS (a null
 * equals a null), 0 is EQ (a null matches nothing); null_equal = NULL is all EQ, i.e. b2_hash_join.  A row takes part in
 * matching unless one of its EQ columns is null. */
B2_API int b2_hash_join_ex(B2Context* ctx, const B2Array* left_keys, const B2Array* right_keys, int n_keys,
                           const uint8_t* null_equal, int join_type, B2Array* out_left, B2Array* out_right, void* stream);
/* The residual filter of a join (JoinResidualFilter, acero/swiss_join_internal.h): cand_left / cand_right are the INNER
 * pairs of b2_hash_join(_ex) (B2_UINT32, no nulls, cand_left non-decreasing), keep a B2_BOOL per pair -- the filter
 * evaluated on the pair; a null counts as false.  out = the join_type result over the surviving pairs, in b2_hash_join's
 * order and layout: a left row whose pairs all fail is unmatched (LEFT / FULL OUTER give it a null-extended row, ANTI keeps
 * it), FULL OUTER appends the right rows with no surviving pair.  n_left / n_right are the side lengths.  A candidate row
 * out of range, a decreasing cand_left or lengths that differ give B2_INVALID before anything is written through them. */
B2_API int b2_join_residual(B2Context* ctx, const B2Array* cand_left, const B2Array* cand_right, const B2Array* keep,
                            int64_t n_left, int64_t n_right, int join_type, B2Array* out_left, B2Array* out_right,
                            void* stream);

/* ---------------------------------------------------------------------------
 * Grouper.  Replaces Grouper::{Make,Consume,Lookup,GetUniques,num_groups,Reset}
 * (compute/row/grouper.h:104-196; GrouperFastImpl row/grouper.cc:555-963, GrouperImpl :300-553)
 * for 1..8 key columns, each fixed-width numeric (1/2/4/8 bytes) or utf8 / binary / large_utf8 /
 * large_binary.  Keys that pack into 64 bits use one table (csrc/grouper.cu); wider keys and string
 * keys are reduced part by part to 32-bit ids and folded (csrc/grouper_wide.cu; strings through a
 * 64-bit hash whose every row is verified against the stored key bytes).
 * Group ids are dense uint32 assigned in first-occurrence row order.
 * ------------------------------------------------------------------------- */
typedef struct B2Grouper B2Grouper;
B2_API int b2_grouper_create(B2Context* ctx, const int32_t* key_types, int n_keys,
                             B2Grouper** out);
B2_API void b2_grouper_destroy(B2Grouper* g);
/* keys: n_keys arrays of equal length; out_ids: B2_UINT32 array, no nulls */
B2_API int b2_grouper_consume(B2Grouper* g, const B2Array* keys, B2Array* out_ids,
                              void* stream);
/* as consume but never inserts; unknown keys give null ids */
B2_API int b2_grouper_lookup(B2Grouper* g, const B2Array* keys, B2Array* out_ids,
                             void* stream);
B2_API int b2_grouper_num_groups(const B2Grouper* g, uint32_t* out);
/* out_keys: n_keys arrays, each num_groups long, in group-id order */
B2_API int b2_grouper_uniques(B2Grouper* g, B2Array* out_keys, void* stream);
B2_API int b2_grouper_reset(B2Grouper* g);
/* Group-major order (Grouper::MakeGroupings, compute/row/grouper.h:141-167, row/grouper.cc:986-1025): the list<int32>
 * of length num_groups whose entry g holds the row numbers with id g, in row order; groups without rows are empty.
 *   ids        : B2_UINT32 without nulls (else B2_INVALID "MakeGroupings with null ids"), every id < num_groups
 *                (else B2_INDEX_ERROR), at most INT32_MAX of them (else B2_CAPACITY_ERROR, before any allocation)
 *   out_offsets: B2_INT32, num_groups + 1 entries, no nulls
 *   out_rows   : B2_INT32, ids.length row numbers in (id, row) order
 * Grouper::ApplyGroupings(groupings, values) is b2_take(values, out_rows) under the same offsets. */
B2_API int b2_make_groupings(B2Context* ctx, const B2Array* ids, int64_t num_groups, B2Array* out_offsets,
                             B2Array* out_rows, void* stream);

/* ---------------------------------------------------------------------------
 * Ungrouped sum / mean / min_max / count of one numeric column: everything the
 * reference's scalar-aggregate states keep, in one pass.  Replaces SumImpl / MeanImpl
 * (compute/kernels/aggregate_basic.inc.cc:49-107,227-290), MinMaxState / MinMaxImpl
 * (:657-701,776-860) and CountImpl (compute/kernels/aggregate_basic.cc:98-130); the
 * caller applies ScalarAggregateOptions{skip_nulls, min_count} (compute/api_aggregate.h:48-50)
 * the way their Finalize does.
 * ------------------------------------------------------------------------- */
typedef struct B2ReduceResult {
  int64_t count;      /* valid (non-null) rows */
  int64_t null_count; /* length - count */
  uint64_t sum_bits;  /* sum over valid rows in acc_type: int64 (wrapping) / uint64 / double bits */
  uint64_t min_bits;  /* min over valid rows widened to int64 / uint64 / double bits; the type's
                         anti-extremum (NaN for floats) when count == 0 or every value is NaN */
  uint64_t max_bits;
  uint64_t dsum_bits; /* the sum as a double for MeanImpl's sum / count (:263-283): floats = sum_bits,
                         integers = the exact 128-bit sum rounded once (never the int64 wrap-around) */
  int32_t acc_type;   /* B2_INT64, B2_UINT64 or B2_DOUBLE (FindAccumulatorType) */
  int32_t value_type;
} B2ReduceResult;
B2_API int b2_reduce(B2Context* ctx, const B2Array* values, B2ReduceResult* out, void* stream);

/* ---------------------------------------------------------------------------
 * unique / value_counts / dictionary_encode over one fixed-width numeric or utf8 / binary column.
 * Replaces UniqueAction / ValueCountsAction / DictEncodeAction + RegularHashKernel
 * (compute/kernels/vector_hash.cc:65-235,236-470; registration :782-830;
 * DictionaryEncodeOptions compute/api_vector.h:66-82).
 *   out_dictionary : the distinct values in first-occurrence order (required)
 *   out_indices    : int32 index of every row into the dictionary, or NULL if not wanted
 *   out_counts     : int64 occurrences of every dictionary entry, or NULL if not wanted
 *   null_encoding  : 0 = MASK  (null rows -> null index; no null in the dictionary)
 *                    1 = ENCODE (null is a dictionary entry; what unique / value_counts use)
 * unique = (ENCODE, NULL, &d, NULL); value_counts = (ENCODE, NULL, &d, &c);
 * dictionary_encode = (mode, &i, &d, NULL).
 * ------------------------------------------------------------------------- */
B2_API int b2_vector_hash(B2Context* ctx, const B2Array* values, int null_encoding,
                          B2Array* out_indices, B2Array* out_dictionary, B2Array* out_counts,
                          void* stream);

/* ---------------------------------------------------------------------------
 * is_in / index_in.  Replaces SetLookupState (kernels/scalar_set_lookup.cc:44-129), IndexInVisitor / ExecIndexIn
 * (:271-396) and IsInVisitor / ExecIsIn (:398-545); SetLookupOptions compute/api_scalar.h:279-324,
 * GetNullMatchingBehavior api_scalar.cc:604-612.
 *   value_set     : bool, numeric or (large_)utf8 / (large_)binary, of the values' type (casting is the caller's job;
 *                   other types give B2_NOT_IMPLEMENTED); at most INT32_MAX values (else B2_CAPACITY_ERROR).  Each
 *                   distinct value maps to its first position; numbers compare by bit pattern, strings by bytes.
 *   null_matching : 0 MATCH, 1 SKIP, 2 EMIT_NULL, 3 INCONCLUSIVE (SetLookupOptions::NullMatchingBehavior)
 * The table is built once by create and probed by every b2_is_in / b2_index_in call.
 *   b2_is_in    out: B2_BOOL; without validity under MATCH and SKIP
 *   b2_index_in out: B2_INT32, null where nothing matches; 0 under null slots
 * values of another type than the value set give B2_TYPE_ERROR.  A call synchronises only when its result can hold
 * a null (to return the null count).
 * b2_set_lookup_table reports the table's bytes and whether the probe stages it in shared memory (1) or reads it
 * from global memory (0); a boolean value set has no table.
 * ------------------------------------------------------------------------- */
typedef struct B2SetLookup B2SetLookup;
B2_API int b2_set_lookup_create(B2Context* ctx, const B2Array* value_set, int null_matching, B2SetLookup** out,
                                void* stream);
B2_API void b2_set_lookup_destroy(B2SetLookup* s);
B2_API int b2_set_lookup_table(const B2SetLookup* s, int64_t* table_bytes, int32_t* shared);
B2_API int b2_is_in(B2SetLookup* s, const B2Array* values, B2Array* out, void* stream);
B2_API int b2_index_in(B2SetLookup* s, const B2Array* values, B2Array* out, void* stream);

/* ---------------------------------------------------------------------------
 * Hash aggregates.  Replaces the HashAggregateKernel contract
 * {init,resize,consume,merge,finalize} (compute/kernel.h:720-769) for
 * GroupedSumImpl / GroupedCountImpl / GroupedCountAllImpl / GroupedMeanImpl /
 * GroupedMinMaxImpl (kernels/hash_aggregate_numeric.cc:44-295,330-,
 * kernels/hash_aggregate.cc:61-272).
 * ------------------------------------------------------------------------- */
typedef enum B2HashAggKind {
  B2_HASH_SUM = 0,
  B2_HASH_COUNT = 1,
  B2_HASH_COUNT_ALL = 2,
  B2_HASH_MEAN = 3,
  B2_HASH_MIN = 4,
  B2_HASH_MAX = 5,
  B2_HASH_PRODUCT = 6, /* GroupedProductImpl, hash_aggregate_numeric.cc:311-335 (integers wrap mod 2^64) */
  B2_HASH_ANY = 7,     /* GroupedAnyImpl / GroupedAllImpl over a B2_BOOL column, hash_aggregate.cc:1232-1397 */
  B2_HASH_ALL = 8,
  B2_HASH_COUNT_DISTINCT = 9, /* GroupedCountDistinctImpl, hash_aggregate.cc:1400-1478: distinct (value, group) pairs
                                through a Grouper, counted per group under CountOptions::mode; numeric and utf8 / binary values */
  /* GroupedStatisticImpl (hash_aggregate_numeric.cc:452-842) over numeric values, output B2_DOUBLE.  Defaults differ from
     the kinds above: min_count 0 (VarianceOptions / SkewOptions, api_aggregate.h:103-134).  These four also take
     ids == NULL in b2_hashagg_consume when the state has exactly one group: the ungrouped variance / stddev / skew /
     kurtosis (aggregate_var_std.cc:40-235), bitwise reproducible for a given input and batch split. */
  B2_HASH_VARIANCE = 10,
  B2_HASH_STDDEV = 11,
  B2_HASH_SKEW = 12,
  B2_HASH_KURTOSIS = 13,
  /* list outputs (b2_hashagg_out_type = B2_LIST), finalized with b2_hashagg_finalize_list.
     hash_list (GroupedListImpl, hash_aggregate.cc:1858-2047): every value of the group, nulls included, in consume
     order then merge order; numeric, bool, (large_)utf8 / binary and fixed_size_binary(1/2/4/8/16) values; at most
     INT32_MAX values in all (else B2_CAPACITY_ERROR).
     hash_distinct (GroupedDistinctImpl, :1400-1539): the distinct values of the group in first-occurrence order, under
     CountOptions::mode (count_mode); the value types of hash_count_distinct. */
  B2_HASH_LIST = 14,
  B2_HASH_DISTINCT = 15
} B2HashAggKind;
typedef struct B2HashAggOptions {
  int32_t skip_nulls;  /* ScalarAggregateOptions (api_aggregate.h:48-50), default 1 */
  uint32_t min_count;  /* default 1 */
  int32_t count_mode;  /* CountOptions: 0 ONLY_VALID, 1 ONLY_NULL, 2 ALL (api_aggregate.h:64-78) */
  int32_t stat_param;  /* variance / stddev: ddof (>= 0); skew / kurtosis: 1 = unbiased (0 = biased, the default); else 0 */
} B2HashAggOptions;
typedef struct B2HashAgg B2HashAgg;
B2_API int b2_hashagg_create(B2Context* ctx, int kind, int32_t value_type,
                             const B2HashAggOptions* options, B2HashAgg** out);
B2_API void b2_hashagg_destroy(B2HashAgg* a);
B2_API int b2_hashagg_resize(B2HashAgg* a, int64_t num_groups, void* stream);
/* values may be NULL for count_all; ids: B2_UINT32 array of the same length, or NULL for the four moment kinds
   when num_groups == 1 (every row is in group 0) */
B2_API int b2_hashagg_consume(B2HashAgg* a, const B2Array* values, const B2Array* ids,
                              void* stream);
/* state[mapping[i]] (+)= other.state[i]; mapping: B2_UINT32, length = other groups */
B2_API int b2_hashagg_merge(B2HashAgg* a, B2HashAgg* other, const B2Array* group_id_mapping,
                            void* stream);
B2_API int b2_hashagg_finalize(B2HashAgg* a, B2Array* out, void* stream);
/* The list<value type> of a B2_HASH_LIST / B2_HASH_DISTINCT state as two flat arrays: out_offsets (B2_INT32,
 * num_groups + 1 entries) and out_values (the child, of the value type).  List slots are never null. */
B2_API int b2_hashagg_finalize_list(B2HashAgg* a, B2Array* out_offsets, B2Array* out_values, void* stream);
B2_API int32_t b2_hashagg_out_type(const B2HashAgg* a);

/* Fused group-by for the Acero aggregate node (acero/groupby_aggregate_node.cc:210-253
 * Consume = grouper->Consume + kernel->consume per aggregate): one pass over
 * (key, value) rows updating an on-device table, no uint32 id column materialised.
 * Semantically identical to b2_grouper_consume followed by b2_hashagg_consume of a
 * sum and a count(ONLY_VALID) aggregator over the same value column. */
/* expected_groups: cardinality hint (like reserving a builder).  0 = unknown: the table grows batch by
 * batch and large batches are processed in 64M-row chunks.  > 0: the table is sized for it and a batch is
 * processed in one chunk (fastest: rows of a key meet in shared memory); if the true number of groups
 * exceeds the hint by more than the table slack + 64M inside one batch, consume fails with
 * B2_CAPACITY_ERROR (nothing is silently dropped). */
typedef struct B2GroupBySumCount B2GroupBySumCount;
B2_API int b2_groupby_sumcount_create(B2Context* ctx, int32_t key_type, int32_t value_type,
                                      int64_t expected_groups, B2GroupBySumCount** out);
B2_API void b2_groupby_sumcount_destroy(B2GroupBySumCount* g);
B2_API int b2_groupby_sumcount_consume(B2GroupBySumCount* g, const B2Array* keys,
                                       const B2Array* values, void* stream);
/* Adds partial states into the table: keys / sums (the accumulator type b2_groupby_sumcount_finalize returns) /
 * counts (int64) of ANOTHER group-by over the same key and value types -- a peer GPU's groups after the exchange, or
 * another thread's.  The fused twin of HashAggregateKernel::merge (compute/kernel.h:720-725) as GroupByNode::Merge uses
 * it (acero/groupby_aggregate_node.cc:255-298).  A partial with count 0 only asserts the group exists. */
B2_API int b2_groupby_sumcount_merge(B2GroupBySumCount* g, const B2Array* keys, const B2Array* sums,
                                     const B2Array* counts, void* stream);
/* how many consume() chunks ran on each internal path (diagnostics for tests / bench):
 *   dense   : direct-addressed packed state in L2, one reduction per row (dense key range, narrow verified value window)
 *   compact : 8-byte tuples + bulk-async partition passes (key range + value window fit 63 bits)
 *   general : 17-byte tuples, any key / value
 *   atomic  : small batches, one global-table update per row */
B2_API int b2_groupby_sumcount_path_counts(const B2GroupBySumCount* g, int64_t* dense, int64_t* compact,
                                           int64_t* general, int64_t* atomic);
/* out_keys / out_sums / out_counts: num_groups long, group order unspecified */
B2_API int b2_groupby_sumcount_finalize(B2GroupBySumCount* g, B2Array* out_keys,
                                        B2Array* out_sums, B2Array* out_counts, void* stream);

/* ---------------------------------------------------------------------------
 * Multi-GPU exchange helpers (no reference counterpart: the reference is single-process;
 * its per-thread analogue is GroupByNode::Merge, acero/groupby_aggregate_node.cc:255-298).
 * out_ids: B2_UINT32, one destination id per row.
 *   hash : id = hash64(key) % n_parts, null keys -> 0          (hash-aggregate shuffle)
 *   range: id = #splitters <= value in SortIndices' total order; nulls -> n_splitters + 1
 *          (SortIndices shuffle; order as in b2_sort_indices)
 * ------------------------------------------------------------------------- */
B2_API int b2_hash_partition(B2Context* ctx, const B2Array* keys, int n_parts, B2Array* out_ids,
                             void* stream);
B2_API int b2_range_partition(B2Context* ctx, const B2Array* values, const B2Array* splitters,
                              int order, B2Array* out_ids, void* stream);
/* Sender side of the distributed SortIndices in one call: a STABLE split of (value, row number) pairs by range id
 * (bin b = #splitters <= value in SortIndices' order, b = 0 .. n_splitters; rows with a null value form the last bin).
 *   out_values : values regrouped bin by bin (row order kept inside a bin), no validity
 *   out_rows   : B2_UINT32 row_base + original row, regrouped the same way (the payload of b2_sort_payload at the owner)
 *   out_counts : HOST array of n_splitters + 2 int64 = rows per bin
 * count -> scan -> scatter: two streaming passes instead of ids + sort_indices(ids) + two takes + an offset add. */
B2_API int b2_range_split(B2Context* ctx, const B2Array* values, const B2Array* splitters, int order,
                          uint64_t row_base, B2Array* out_values, B2Array* out_rows, int64_t* out_counts,
                          void* stream);
/* out_counts[b] (HOST array of n_bins int64) = rows whose id == b: the send counts of the exchange.
 * ids: B2_UINT32 without nulls, every id < n_bins (else B2_INDEX_ERROR); n_bins <= 8192. */
B2_API int b2_bincount(B2Context* ctx, const B2Array* ids, int n_bins, int64_t* out_counts, void* stream);

/* The exchange itself: one process per GPU, NCCL over NVLink / NVSwitch (resolved with dlopen at the
 * first call; libarrow_b200.so does not link NCCL).  Rank 0 creates the 128-byte id, the host
 * application distributes it (MPI, a torch.distributed store, a file) and every rank calls
 * b2_comm_init with the same id.  All calls are stream-ordered on `stream` like every other entry.
 *   all_gather    : recv[r * bytes_per_rank ..] = rank r's `send` (the P x P count matrix)
 *   all_reduce_i64: element-wise sum / max / min of `count` int64 values
 *   all_to_all_v  : rank p receives send[send_offsets[p] .. + send_bytes[p]) of every rank q at
 *                   recv[recv_offsets[q] ..]; the P-1 sends and receives are one NCCL group
 *                   (host arrays of `world` entries, in bytes; recv_bytes must match the peers' send_bytes) */
#define B2_COMM_ID_BYTES 128
typedef struct B2Comm B2Comm;
typedef enum B2CommOp { B2_COMM_SUM = 0, B2_COMM_MAX = 1, B2_COMM_MIN = 2 } B2CommOp;
B2_API int b2_comm_unique_id(uint8_t* out_id /* [B2_COMM_ID_BYTES] */);
B2_API int b2_comm_init(B2Context* ctx, int rank, int world, const uint8_t* id, B2Comm** out);
B2_API void b2_comm_destroy(B2Comm* comm);
B2_API int b2_comm_rank(const B2Comm* comm);
B2_API int b2_comm_world(const B2Comm* comm);
B2_API int b2_comm_nccl_version(int* out);
/* all_to_all_v calls between group_start and group_end (one per column) are issued as ONE NCCL launch */
B2_API int b2_comm_group_start(B2Comm* comm);
B2_API int b2_comm_group_end(B2Comm* comm);
B2_API int b2_comm_all_gather(B2Comm* comm, const void* send, void* recv, int64_t bytes_per_rank, void* stream);
B2_API int b2_comm_all_reduce_i64(B2Comm* comm, const void* send, void* recv, int64_t count, int op, void* stream);
B2_API int b2_comm_all_to_all_v(B2Comm* comm, const void* send, const int64_t* send_offsets,
                                const int64_t* send_bytes, void* recv, const int64_t* recv_offsets,
                                const int64_t* recv_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ARROW_B200_H */
