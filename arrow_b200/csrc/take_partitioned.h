// take_partitioned.h -- the partitioned path of a large random fixed-width Take (take_partitioned.cu), called by
// b2_take and b2_take_cast_arith (selection_take.cu) when take_partition_plan picks it.
#pragma once
#include "common.cuh"
#include "context.h"

namespace b2 {

template <typename OT>
__device__ __forceinline__ OT fused_apply(int op, OT x, OT y) {
  return op == B2_ADD ? x + y : (op == B2_SUBTRACT ? x - y : x * y);
}

struct PartTakeArgs {
  const void* values;  // advanced by offset
  BitmapReader values_valid;
  int64_t values_length;  // 1 .. 2^32
  const void* indices;    // advanced by offset
  BitmapReader idx_valid;
  int64_t n;              // < 2^30
  // fused take + cast + arithmetic only (b2_take_cast_arith)
  const void* other;  // NULL: broadcast `other_scalar`
  double other_scalar;
  BitmapReader other_valid;
  int op;
  void* out;
  uint32_t* out_validity;  // NULL when no validity is produced
  int64_t* valid_count;
  unsigned long long* first_bad;  // ~0 initially; the first out-of-range valid index's row, as the direct kernels report it
  unsigned long long* stalled;    // 0 initially; set when the folded gather gave up waiting for a fold item: the result is void
  int shift;                      // bucket of index j = j >> shift, < 256
  bool fold;            // gather from a float32 copy of the values with the nulls folded in (see kFoldMinShift)
  int64_t value_nulls;  // values->null_count when `fold`: the size of the table of the null rows' casts
};

// The folded gather of b2_take_cast_arith to float32 from 8-byte values with nulls: a null row's slot in the folded copy
// holds a signalling NaN naming the row's rank among its band's nulls (2^23 - 2 codes), so a band may hold at most 2^22
// rows (shift <= 22).  The null counts are taken over tiles of at most 4096 rows that are whole 64-bit bitmap words
// (shift >= 6).  The caller sets `fold` only within these bounds and only when values->null_count > 0.
constexpr int kFoldMinShift = 6;
constexpr int kFoldMaxShift = 22;

// out_type < 0: plain take of `vw`-byte values (4 or 8); else out = op(static_cast<out_type>(values[idx]), other) for
// value_type float64 / float32 / int64 / int32.  *ran = false (and nothing launched) when the temporaries cannot be had.
int take_partitioned(B2Context* ctx, const PartTakeArgs& a, int vw, int value_type, int idx_type, int out_type,
                     cudaStream_t s, bool* ran);

}  // namespace b2
