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
  int shift;                      // bucket of index j = j >> shift, < 256
};

// out_type < 0: plain take of `vw`-byte values (4 or 8); else out = op(static_cast<out_type>(values[idx]), other) for
// value_type float64 / float32 / int64 / int32.  *ran = false (and nothing launched) when the temporaries cannot be had.
int take_partitioned(B2Context* ctx, const PartTakeArgs& a, int vw, int value_type, int idx_type, int out_type,
                     cudaStream_t s, bool* ran);

}  // namespace b2
