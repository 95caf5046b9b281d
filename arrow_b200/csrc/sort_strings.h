// sort_strings.h -- the string rank behind every sort by a (large_)utf8 / (large_)binary key (sort_strings.cu).
#pragma once
#include "context.h"

namespace b2 {

// One uint32 per row of a string column such that rank(a) < rank(b) iff a sorts before b (unsigned byte order, a
// proper prefix first) and equal strings get equal ranks.  *out becomes a B2_UINT32 array over `rank` (allocated here
// from the context pool, owned by the caller) that carries the input's validity by pointing at the input's own bitmap,
// so both `rank` and the input must outlive every use of *out.  Rows: < 2^32 - 8192, as the numeric sorts.
// Stream-ordered on s; one device-to-host read of a count per refinement round.
int string_rank(B2Context* ctx, const B2Array* values, Temp* rank, B2Array* out, cudaStream_t s);

}  // namespace b2
