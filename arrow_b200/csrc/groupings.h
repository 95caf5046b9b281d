// groupings.h -- group-major order (b2_make_groupings, groupings.cu) and the states behind B2_HASH_LIST /
// B2_HASH_DISTINCT; b2_hashagg_* forwards those two kinds here.
#pragma once

#include "context.h"

namespace b2 {

// Stable LSD radix sort of n uint32 group ids on the onesweep passes of sort_indices.cu: rows[k] = the row number of the
// k-th id in (id, row) order.  Only the digits that vary are sorted.  When at least one pass runs, the sorted ids are
// written to sorted_ids and *ids_sorted is set; otherwise every id is equal and `ids` itself is in order.  n < 2^31.
int radix_sort_ids(B2Context* ctx, const uint32_t* ids, int64_t n, int32_t* rows, uint32_t* sorted_ids, bool* ids_sorted,
                   cudaStream_t s);

struct ListAgg;

inline bool is_list_kind(int kind) { return kind == B2_HASH_LIST || kind == B2_HASH_DISTINCT; }

int list_create(B2Context* ctx, int32_t value_type, ListAgg** out);
void list_destroy(ListAgg* l);
int list_resize(ListAgg* l, int64_t num_groups);
int list_consume(ListAgg* l, const B2Array* values, const B2Array* ids, cudaStream_t s);
int list_merge(ListAgg* l, const ListAgg* other, const B2Array* group_id_mapping, cudaStream_t s);
int list_finalize(ListAgg* l, B2Array* out_offsets, B2Array* out_values, cudaStream_t s);

// hash_distinct's finalize over the (value, group id) pair Grouper of hash_count_distinct: the pairs CountOptions mode
// admits (0 ONLY_VALID, 1 ONLY_NULL, 2 ALL), grouped in first-occurrence order
int distinct_finalize(B2Context* ctx, B2Grouper* pairs, int count_mode, int64_t num_groups, B2Array* out_offsets,
                      B2Array* out_values, cudaStream_t s);

}  // namespace b2
