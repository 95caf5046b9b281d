// hash_moments.h -- the state behind B2_HASH_VARIANCE / STDDEV / SKEW / KURTOSIS (hash_moments.cu); b2_hashagg_*
// forwards those four kinds here.
#pragma once

#include "context.h"

// B2_HASHAGG_BAND_MB: bytes of state one consume launch applies (hash_aggregate.cu)
int64_t hashagg_band_bytes();

namespace b2 {

struct MomentAgg;

inline bool is_moment_kind(int kind) { return kind >= B2_HASH_VARIANCE && kind <= B2_HASH_KURTOSIS; }

int moments_create(B2Context* ctx, int kind, int32_t value_type, const B2HashAggOptions& opt, MomentAgg** out);
void moments_destroy(MomentAgg* m);
int moments_resize(MomentAgg* m, int64_t num_groups, cudaStream_t s);
// ids == nullptr: every row is in group 0 (the state must have exactly one group)
int moments_consume(MomentAgg* m, const B2Array* values, const B2Array* ids, cudaStream_t s);
int moments_merge(MomentAgg* m, const MomentAgg* other, const B2Array* group_id_mapping, cudaStream_t s);
int moments_finalize(MomentAgg* m, B2Array* out, cudaStream_t s);

}  // namespace b2
