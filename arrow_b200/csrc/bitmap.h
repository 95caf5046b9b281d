// bitmap.h -- internal launchers for validity bitmaps (see bitmap.cu)
#pragma once
#include "common.cuh"
#include "context.h"

namespace b2 {

// dst (64-bit words, may be NULL) = a & b re-based to bit 0; *d_count (device, may be
// NULL) += popcount.
int launch_bitmap_and(const void* a, int64_t a_off, const void* b, int64_t b_off, int64_t length,
                      void* dst, int64_t* d_count, cudaStream_t s);

// Output validity of a scalar kernel over inputs a (and optionally b): allocates the
// intersection bitmap from the pool, returns NULL validity when the result has no
// nulls.  Mirrors PropagateNullsSpans (cpp/src/arrow/compute/exec.cc:1222-1281).
int make_validity(B2Context* ctx, const B2Array* a, const B2Array* b, int64_t length,
                  void** out_validity, int64_t* out_null_count, cudaStream_t s);

// out[i] = in[0] + ... + in[i-1] for i < n (out[n] is not written); *total (device, may be NULL) = the sum of all n.
// Runs as one 1024-thread block: meant for per-tile counts.
int launch_exclusive_scan_i64(const int64_t* in, int64_t n, int64_t* out, int64_t* total, cudaStream_t s);

}  // namespace b2
