// string_predicates.cu -- predicates over utf8 / large_utf8 / binary / large_binary columns: the six comparisons,
// match_substring, starts_with, ends_with and match_like, producing Arrow's bit-packed boolean layout.
//
// Replaces:
//   CompareKernel over BaseBinaryTypes, string_view ordering     kernels/scalar_compare.cc:42-72,340-366,431-433
//   StringBoolTransform, PlainSubstringMatcher (KMP),
//     PlainStartsWithMatcher, PlainEndsWithMatcher               kernels/scalar_string_ascii.cc:1207-1307
//   MatchLike::Exec and its three classifying regexes,
//     MakeLikeRegex                                              :1456-1588
// Semantics kept: every slot is evaluated, nulls included, over the bytes its offsets span (the data bits under a null
// are those of that slot's bytes); the output validity is the AND of the input validities; a null scalar gives an
// all-null result whose data bits are the comparison with the empty string (UnboxScalar of a null binary scalar).
// Strings order by unsigned bytes, a proper prefix first.  Matching is by bytes; for match_like `_` is one code point
// over utf8 and one byte over binary, and `%` skips code points / bytes.
//
// Design.  One streaming pass: warp w owns 32-row groups, lane l evaluates row 32w + l, and the result leaves as one
// 32-bit word from one ballot, without atomics.  Offsets are read coalesced (lane l reads offsets l and l + 1), character
// bytes through aligned 8-byte loads (load_bytes8), so neither the data buffer nor a row needs any alignment.  Equality
// checks lengths before it reads a byte.  A row whose work (bytes to compare or to search) exceeds kLongRow is not
// evaluated by its lane: the warp takes such rows one at a time and all 32 lanes cooperate on it (a first-difference
// scan 256 bytes per step, or substring windows of kWindow starts that overlap by m - 1 bytes, then __any_sync), so one
// 1 MiB row does not serialise a warp.  The general LIKE matcher (a pattern the classifying regexes do not take) runs
// one lane per row: the pattern is compiled on the host into anchored segments of literal bytes and `_` slots split at
// `%`, and each row is matched by a leftmost greedy segment search, which is exact because segments hold no `%`.
#include <string>
#include <vector>

#include "bitmap.h"
#include "common.cuh"
#include "context.h"

namespace b2 {

constexpr int kPredBlock = 256;
constexpr int kPredBlocksPerSM = 4;  // the register budget of __launch_bounds__: up to 64 per thread
constexpr int64_t kLongRow = 1024;  // bytes of work above which the warp cooperates on the row
constexpr int kWindow = 64;         // substring start positions per lane per cooperative step

struct View {
  const uint8_t* p;
  int64_t len;
};

template <typename OffT>
__device__ __forceinline__ View row_view(const OffT* offs, const uint8_t* bytes, int64_t i) {
  const int64_t o0 = static_cast<int64_t>(offs[i]);
  return View{bytes + o0, static_cast<int64_t>(offs[i + 1]) - o0};
}

__device__ __forceinline__ uint32_t byte_at(const uint8_t* p) { return static_cast<uint32_t>(load_bytes8(p, 1)); }

// index of the first byte where a and b differ in [0, n), or n
__device__ __forceinline__ int64_t first_diff(const uint8_t* a, const uint8_t* b, int64_t n) {
  for (int64_t o = 0; o < n; o += 8) {
    const int nb = n - o >= 8 ? 8 : static_cast<int>(n - o);
    const uint64_t x = load_bytes8(a + o, nb) ^ load_bytes8(b + o, nb);
    if (x) return o + (__ffsll(static_cast<long long>(x)) - 1) / 8;
  }
  return n;
}

// the same with all 32 lanes of the warp: 256 bytes per step, the lowest differing chunk wins
__device__ __forceinline__ int64_t warp_first_diff(const uint8_t* a, const uint8_t* b, int64_t n) {
  const unsigned lane = lane_id();
  for (int64_t base = 0; base < n; base += 32 * 8) {
    const int64_t o = base + lane * 8;
    uint64_t x = 0;
    if (o < n) {
      const int nb = n - o >= 8 ? 8 : static_cast<int>(n - o);
      x = load_bytes8(a + o, nb) ^ load_bytes8(b + o, nb);
    }
    const unsigned hit = __ballot_sync(0xffffffffu, x != 0);
    if (hit) {
      const int src = __ffs(hit) - 1;
      const unsigned long long xs = __shfl_sync(0xffffffffu, static_cast<unsigned long long>(x), src);
      return base + src * 8 + (__ffsll(static_cast<long long>(xs)) - 1) / 8;
    }
  }
  return n;
}

// -1 / 0 / 1 as a < b, a == b, a > b, from their first difference d over min(len) bytes
__device__ __forceinline__ int order_from(View a, View b, int64_t d) {
  const int64_t m = a.len < b.len ? a.len : b.len;
  if (d < m) return byte_at(a.p + d) < byte_at(b.p + d) ? -1 : 1;
  return a.len < b.len ? -1 : (a.len > b.len ? 1 : 0);
}

__device__ __forceinline__ bool op_result(int op, int c) {
  switch (op) {
    case B2_EQUAL: return c == 0;
    case B2_NOT_EQUAL: return c != 0;
    case B2_GREATER: return c > 0;
    case B2_GREATER_EQUAL: return c >= 0;
    case B2_LESS: return c < 0;
    default: return c <= 0;
  }
}

// Whether pattern pat (m >= 1 bytes, head = its first min(m, 8) bytes) occurs in t[0, len): a 64-bit window slides
// over the text one byte at a time (bytes fetched 8 at a time), its top k bytes are compared with the head, and a head
// hit of a pattern longer than 8 bytes is verified against the rest.
__device__ __forceinline__ bool find_in(const uint8_t* t, int64_t len, const uint8_t* pat, int64_t m, uint64_t head) {
  if (len < m) return false;
  const int k = m < 8 ? static_cast<int>(m) : 8;
  const int sh = 64 - 8 * k;
  uint64_t win = 0;
  const int64_t last_end = len - m + k;  // the head of the last candidate start ends at byte last_end - 1
  for (int64_t o = 0; o < last_end; o += 8) {
    const int nb = last_end - o >= 8 ? 8 : static_cast<int>(last_end - o);
    uint64_t c = load_bytes8(t + o, nb);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (j < nb) {
        win = (win >> 8) | (c << 56);
        c >>= 8;
        const int64_t end = o + j + 1;  // bytes [end - k, end) are in the window's top k bytes
        if (end >= k && (win >> sh) == head) {
          if (m <= 8 || first_diff(t + end, pat + 8, m - 8) == m - 8) return true;
        }
      }
    }
  }
  return false;
}

// the same with all 32 lanes: lane l of step s searches the starts [(32s + l) W, (32s + l + 1) W), i.e. the bytes of
// that range plus the m - 1 that follow
__device__ __forceinline__ bool warp_find_in(const uint8_t* t, int64_t len, const uint8_t* pat, int64_t m, uint64_t head) {
  const unsigned lane = lane_id();
  const int64_t n_starts = len - m + 1;
  for (int64_t base = 0; base < n_starts; base += 32 * kWindow) {
    const int64_t s0 = base + lane * kWindow;
    bool hit = false;
    if (s0 < n_starts) {
      const int64_t starts = n_starts - s0 < kWindow ? n_starts - s0 : kWindow;
      hit = find_in(t + s0, starts + m - 1, pat, m, head);
    }
    if (__any_sync(0xffffffffu, hit)) return true;
  }
  return false;
}

// ---------------------------------------------------------------------------------------------------------------------
// comparisons: left array against a right array (OffB = its offsets) or a scalar (OffB = void)
// ---------------------------------------------------------------------------------------------------------------------
struct CompareArgs {
  const void* a_offs;  // at the left array's offset
  const uint8_t* a_bytes;
  const void* b_offs;  // at the right array's offset; NULL: the scalar
  const uint8_t* b_bytes;
  const uint8_t* scalar;
  int64_t scalar_len;
  int64_t n;
  int64_t n_words;
  int op;
  uint32_t* out;
};

template <typename OffA, typename OffB>
__global__ void __launch_bounds__(kPredBlock, kPredBlocksPerSM) compare_binary_kernel(const CompareArgs a) {
  const unsigned lane = lane_id();
  const int64_t warp = (blockIdx.x * (int64_t)kPredBlock + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * kPredBlock) >> 5;
  const bool eq = a.op == B2_EQUAL || a.op == B2_NOT_EQUAL;
  for (int64_t w = warp; w < a.n_words; w += n_warps) {
    const int64_t i = (w << 5) + lane;
    const bool in = i < a.n;
    View x{a.a_bytes, 0}, y{a.scalar, a.scalar_len};
    if (in) {
      x = row_view(static_cast<const OffA*>(a.a_offs), a.a_bytes, i);
      if constexpr (!std::is_void_v<OffB>) y = row_view(static_cast<const OffB*>(a.b_offs), a.b_bytes, i);
    }
    const int64_t m = x.len < y.len ? x.len : y.len;
    // equality of rows whose lengths differ reads no byte
    const int64_t work = eq && x.len != y.len ? 0 : m;
    const bool lng = in && work > kLongRow;
    bool res = false;
    if (in && !lng) res = op_result(a.op, eq && x.len != y.len ? 1 : order_from(x, y, first_diff(x.p, y.p, work)));
    for (unsigned longs = __ballot_sync(0xffffffffu, lng); longs; longs &= longs - 1) {
      const int src = __ffs(longs) - 1;
      const View xs{reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(x.p), src)),
                    static_cast<int64_t>(__shfl_sync(0xffffffffu, static_cast<long long>(x.len), src))};
      const View ys{reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(y.p), src)),
                    static_cast<int64_t>(__shfl_sync(0xffffffffu, static_cast<long long>(y.len), src))};
      const int64_t ms = xs.len < ys.len ? xs.len : ys.len;
      const bool r = op_result(a.op, order_from(xs, ys, warp_first_diff(xs.p, ys.p, ms)));
      if (lane == src) res = r;
    }
    const unsigned word = __ballot_sync(0xffffffffu, res);
    if (lane == 0) st_stream(a.out + w, word);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// match_substring / starts_with / ends_with (and match_like patterns the classifying regexes turn into one of them)
// ---------------------------------------------------------------------------------------------------------------------
struct MatchArgs {
  const void* offs;  // at the input's offset
  const uint8_t* bytes;
  int64_t n;
  int64_t n_words;
  int kind;  // B2_MATCH_SUBSTRING / STARTS_WITH / ENDS_WITH
  const uint8_t* pat;
  int64_t m;
  uint64_t head;  // the pattern's first min(m, 8) bytes
  // general LIKE program (kind == B2_MATCH_LIKE)
  const uint8_t* lit;      // the literal byte of every item
  const uint8_t* any;      // 1 where the item is a `_` slot
  const int64_t* seg;      // segment k holds items [seg[k], seg[k + 1])
  int n_seg;               // segments: the prefix, the middles, the suffix (n_seg == 1: no `%`, the whole row)
  bool utf8;
  uint32_t* out;
};

// end of segment [i0, i1) matched at t[s, len), or -1
__device__ __forceinline__ int64_t match_segment(const MatchArgs& a, int64_t i0, int64_t i1, const uint8_t* t, int64_t len, int64_t s) {
  for (int64_t j = i0; j < i1; ++j) {
    if (s >= len) return -1;
    const uint32_t c = byte_at(t + s);
    if (a.any[j]) {
      s += !a.utf8 || c < 0xc0 ? 1 : (c < 0xe0 ? 2 : (c < 0xf0 ? 3 : 4));  // one code point over utf8
      if (s > len) return -1;
    } else {
      if (c != a.lit[j]) return -1;
      ++s;
    }
  }
  return s;
}

// the leftmost start >= s of segment [i0, i1) in t (at a code point boundary over utf8) whose match ends at `need_end`
// (or anywhere when need_end < 0); returns the match's end, or -1
__device__ __forceinline__ int64_t search_segment(const MatchArgs& a, int64_t i0, int64_t i1, const uint8_t* t, int64_t len,
                                                  int64_t s, int64_t need_end) {
  for (; s <= len; ++s) {
    if (a.utf8 && s < len && (byte_at(t + s) & 0xc0) == 0x80) continue;
    const int64_t e = match_segment(a, i0, i1, t, len, s);
    if (e >= 0 && (need_end < 0 || e == need_end)) return e;
  }
  return -1;
}

__device__ __forceinline__ bool like_general(const MatchArgs& a, View v) {
  const int64_t e0 = match_segment(a, a.seg[0], a.seg[1], v.p, v.len, 0);
  if (e0 < 0) return false;
  if (a.n_seg == 1) return e0 == v.len;
  int64_t pos = e0;
  for (int k = 1; k + 1 < a.n_seg; ++k) {
    pos = search_segment(a, a.seg[k], a.seg[k + 1], v.p, v.len, pos, -1);
    if (pos < 0) return false;
  }
  return search_segment(a, a.seg[a.n_seg - 1], a.seg[a.n_seg], v.p, v.len, pos, v.len) >= 0;
}

template <typename OffT, bool LIKE>
__global__ void __launch_bounds__(kPredBlock, kPredBlocksPerSM) match_kernel(const MatchArgs a) {
  const unsigned lane = lane_id();
  const int64_t warp = (blockIdx.x * (int64_t)kPredBlock + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * kPredBlock) >> 5;
  for (int64_t w = warp; w < a.n_words; w += n_warps) {
    const int64_t i = (w << 5) + lane;
    const bool in = i < a.n;
    View v{a.bytes, 0};
    if (in) v = row_view(static_cast<const OffT*>(a.offs), a.bytes, i);
    bool res = false;
    if constexpr (LIKE) {
      if (in) res = like_general(a, v);
    } else {
      const bool fits = v.len >= a.m;
      // substring search reads the row; starts_with / ends_with read m bytes of it
      const int64_t work = !fits || a.m == 0 ? 0 : (a.kind == B2_MATCH_SUBSTRING ? v.len : a.m);
      const bool lng = in && work > kLongRow;
      if (in && !lng && fits) {
        if (a.kind == B2_MATCH_SUBSTRING) res = a.m == 0 || find_in(v.p, v.len, a.pat, a.m, a.head);
        else res = first_diff(a.kind == B2_MATCH_STARTS_WITH ? v.p : v.p + v.len - a.m, a.pat, a.m) == a.m;
      }
      for (unsigned longs = __ballot_sync(0xffffffffu, lng); longs; longs &= longs - 1) {
        const int src = __ffs(longs) - 1;
        const uint8_t* p = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(v.p), src));
        const int64_t len = __shfl_sync(0xffffffffu, static_cast<long long>(v.len), src);
        bool r;
        if (a.kind == B2_MATCH_SUBSTRING) r = warp_find_in(p, len, a.pat, a.m, a.head);
        else r = warp_first_diff(a.kind == B2_MATCH_STARTS_WITH ? p : p + len - a.m, a.pat, a.m) == a.m;
        if (lane == src) res = r;
      }
    }
    const unsigned word = __ballot_sync(0xffffffffu, res);
    if (lane == 0) st_stream(a.out + w, word);
  }
}

inline int pred_grid(B2Context* ctx, int64_t n_words) {
  return grid_for(n_words, kPredBlock / 32, ctx->sm_count * (2048 / kPredBlock));
}

// the bits of a result of n rows, padding words zeroed
inline int alloc_bits(B2Context* ctx, int64_t n, Temp* data, cudaStream_t s) {
  B2_RETURN_NOT_OK(data->alloc(bitmap_alloc_bytes(n)));
  const int64_t written = ((n + 31) >> 5) * 4;
  B2_CUDA(cudaMemsetAsync(data->as<char>() + written, 0, bitmap_alloc_bytes(n) - written, s));
  return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// host: the LIKE pattern's classification and compilation
// ---------------------------------------------------------------------------------------------------------------------
bool valid_utf8(const std::string& s) {
  size_t i = 0;
  while (i < s.size()) {
    const unsigned char c = s[i];
    int n;
    uint32_t cp;
    if (c < 0x80) { ++i; continue; }
    if (c >= 0xc2 && c <= 0xdf) { n = 1; cp = c & 0x1f; }
    else if (c >= 0xe0 && c <= 0xef) { n = 2; cp = c & 0x0f; }
    else if (c >= 0xf0 && c <= 0xf4) { n = 3; cp = c & 0x07; }
    else return false;
    for (int k = 1; k <= n; ++k) {
      if (i + k >= s.size()) return false;
      const unsigned char d = s[i + k];
      if ((d & 0xc0) != 0x80) return false;
      cp = (cp << 6) | (d & 0x3f);
    }
    if ((n == 2 && cp < 0x800) || (n == 3 && (cp < 0x10000 || cp > 0x10ffff)) || (cp >= 0xd800 && cp <= 0xdfff)) return false;
    i += n + 1;
  }
  return true;
}

bool no_wildcards(const std::string& s) { return s.find_first_of("%_") == std::string::npos; }

// MatchLike::Exec's dispatch (scalar_string_ascii.cc:1533-1588) without ignore_case: the three regexes, in order
//   substring  %+([^%_]*[^\\%_])?%+      prefix  ([^%_]*[^\\%_])?%+      suffix  %+([^%_]*)
// Their character classes exclude only ASCII bytes, so over valid UTF-8 (utf8) and Latin-1 (binary) alike they are
// decided on bytes.  Returns the kind and sets *lit to the captured text, or returns B2_MATCH_LIKE.
int classify_like(const std::string& p, std::string* lit) {
  const size_t n = p.size();
  size_t lead = 0, trail = 0;
  while (lead < n && p[lead] == '%') ++lead;
  while (trail < n && p[n - 1 - trail] == '%') ++trail;
  auto capture_ok = [](const std::string& x) { return no_wildcards(x) && (x.empty() || x.back() != '\\'); };
  if (n > 0 && lead == n) {  // only '%': two or more are a substring search of "", one is a prefix search of ""
    lit->clear();
    return n >= 2 ? B2_MATCH_SUBSTRING : B2_MATCH_STARTS_WITH;
  }
  if (lead >= 1 && trail >= 1) {
    const std::string x = p.substr(lead, n - lead - trail);
    if (capture_ok(x)) { *lit = x; return B2_MATCH_SUBSTRING; }
  }
  if (trail >= 1) {
    const std::string x = p.substr(0, n - trail);
    if (capture_ok(x)) { *lit = x; return B2_MATCH_STARTS_WITH; }
  }
  if (lead >= 1) {
    const std::string x = p.substr(lead);
    if (no_wildcards(x)) { *lit = x; return B2_MATCH_ENDS_WITH; }
  }
  return B2_MATCH_LIKE;  // "" included: it matches only the empty string
}

// MakeLikeRegex (:1456-1497) as segments: `\` makes the next byte literal (a trailing lone `\` is dropped), `_` is a
// slot, `%` ends a segment.  Segment 0 is anchored at the start, the last at the end; empty middle segments are dropped.
struct LikeProgram {
  std::vector<uint8_t> lit, any;
  std::vector<int64_t> seg;
};
LikeProgram compile_like(const std::string& p) {
  LikeProgram g;
  std::vector<std::vector<std::pair<uint8_t, uint8_t>>> segs(1);
  bool escaped = false;
  for (const char ch : p) {
    const uint8_t c = static_cast<uint8_t>(ch);
    if (!escaped && c == '%') segs.emplace_back();
    else if (!escaped && c == '_') segs.back().push_back({0, 1});
    else if (!escaped && c == '\\') escaped = true;
    else {
      segs.back().push_back({c, 0});
      escaped = false;
    }
  }
  std::vector<std::vector<std::pair<uint8_t, uint8_t>>> kept;
  for (size_t k = 0; k < segs.size(); ++k)
    if (k == 0 || k + 1 == segs.size() || !segs[k].empty()) kept.push_back(segs[k]);
  g.seg.push_back(0);
  for (const auto& s : kept) {
    for (const auto& it : s) {
      g.lit.push_back(it.first);
      g.any.push_back(it.second);
    }
    g.seg.push_back(static_cast<int64_t>(g.lit.size()));
  }
  return g;
}

}  // namespace b2

using namespace b2;

struct B2StringMatch {
  B2Context* ctx = nullptr;
  int kind = 0;       // what runs: SUBSTRING / STARTS_WITH / ENDS_WITH, or LIKE for the general matcher
  bool utf8 = false;
  int64_t m = 0;      // literal bytes
  uint64_t head = 0;
  int n_seg = 0;
  void* buf = nullptr;  // the literal, or the program: lit[items] any[items] (padded to 8) seg[n_seg + 1]
  int64_t items = 0;
};

namespace {

template <typename OffA>
int launch_compare(B2Context* ctx, const B2Array* right, const CompareArgs& a, cudaStream_t s) {
  const int grid = pred_grid(ctx, a.n_words);
  if (!right) compare_binary_kernel<OffA, void><<<grid, kPredBlock, 0, s>>>(a);
  else if (offset_width(right->type) == 8) compare_binary_kernel<OffA, int64_t><<<grid, kPredBlock, 0, s>>>(a);
  else compare_binary_kernel<OffA, int32_t><<<grid, kPredBlock, 0, s>>>(a);
  B2_LAUNCHED();
  return B2_OK;
}

const void* offsets_at(const B2Array* x) {
  return static_cast<const uint8_t*>(x->data) + x->offset * offset_width(x->type);
}

}  // namespace

extern "C" int b2_compare_binary(B2Context* ctx, int op, const B2Array* left, const B2Array* right, const void* scalar,
                                 int64_t scalar_length, int scalar_valid, B2Array* out, void* stream) {
  if (!ctx || !left || !out) return set_error(B2_INVALID, "b2_compare_binary: null argument");
  if (op < B2_EQUAL || op > B2_LESS_EQUAL) return set_error(B2_INVALID, "unknown compare op %d", op);
  if (!type_is_binary_like(left->type) || (right && !type_is_binary_like(right->type)))
    return set_error(B2_NOT_IMPLEMENTED, "compare: no binary kernel for type ids %d and %d", left->type,
                     right ? right->type : left->type);
  if (right && right->length != left->length) return set_error(B2_INVALID, "Array arguments must all be the same length");
  if (!right && scalar_valid && scalar_length > 0 && !scalar) return set_error(B2_INVALID, "b2_compare_binary: null scalar bytes");
  if (scalar_length < 0) return set_error(B2_INVALID, "b2_compare_binary: negative scalar length");
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->pick(stream);
  const int64_t n = left->length;
  const bool null_scalar = !right && !scalar_valid;
  Temp data(ctx, s), sbytes(ctx, s);
  B2_RETURN_NOT_OK(alloc_bits(ctx, n, &data, s));
  const int64_t m = right || null_scalar ? 0 : scalar_length;  // a null scalar compares as "" (UnboxScalar of a null)
  if (m > 0) {
    B2_RETURN_NOT_OK(sbytes.alloc(m));
    B2_CUDA(cudaMemcpyAsync(sbytes.ptr, scalar, m, cudaMemcpyHostToDevice, s));
  }
  void* validity = nullptr;
  int64_t null_count = 0;
  if (null_scalar) {
    Temp bits(ctx, s);
    B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(n)));
    B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bitmap_alloc_bytes(n), s));
    validity = n ? bits.release() : nullptr;
    null_count = n;
  } else {
    B2_RETURN_NOT_OK(make_validity(ctx, left, right, n, &validity, &null_count, s));
  }
  Temp vguard(ctx, s);
  vguard.ptr = validity;
  if (n > 0) {
    CompareArgs a{};
    a.a_offs = offsets_at(left);
    a.a_bytes = static_cast<const uint8_t*>(left->data2);
    a.b_offs = right ? offsets_at(right) : nullptr;
    a.b_bytes = right ? static_cast<const uint8_t*>(right->data2) : nullptr;
    a.scalar = sbytes.as<uint8_t>();
    a.scalar_len = m;
    a.n = n;
    a.n_words = (n + 31) >> 5;
    a.op = op;
    a.out = data.as<uint32_t>();
    if (offset_width(left->type) == 8) B2_RETURN_NOT_OK(launch_compare<int64_t>(ctx, right, a, s));
    else B2_RETURN_NOT_OK(launch_compare<int32_t>(ctx, right, a, s));
  }
  fill_out(out, B2_BOOL, n, null_count, vguard.release(), data.release());
  return B2_OK;
}

namespace {
void free_match(B2StringMatch* h) {
  if (h->buf) h->ctx->free(h->buf, h->ctx->stream);
  delete h;
}
}  // namespace

extern "C" int b2_string_match_create(B2Context* ctx, int kind, const void* pattern, int64_t pattern_length, int is_utf8,
                                      B2StringMatch** out, void* stream) {
  if (!ctx || !out || (pattern_length > 0 && !pattern)) return set_error(B2_INVALID, "b2_string_match_create: null argument");
  if (kind < B2_MATCH_SUBSTRING || kind > B2_MATCH_LIKE) return set_error(B2_INVALID, "b2_string_match_create: unknown kind %d", kind);
  if (pattern_length < 0) return set_error(B2_INVALID, "b2_string_match_create: negative pattern length");
  const std::string p(static_cast<const char*>(pattern), static_cast<size_t>(pattern_length));
  // a LIKE pattern over utf8 becomes a UTF-8 regex (or is classified by UTF-8 regexes), which RE2 refuses to compile
  // from invalid UTF-8, even when the pattern looks like %...%
  if (kind == B2_MATCH_LIKE && is_utf8 && !valid_utf8(p)) return set_error(B2_INVALID, "Invalid regular expression: invalid UTF-8");
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->pick(stream);
  auto* h = new B2StringMatch();
  h->ctx = ctx;
  h->utf8 = is_utf8 != 0;
  std::string lit = p;
  h->kind = kind == B2_MATCH_LIKE ? classify_like(p, &lit) : kind;
  std::vector<uint8_t> host;
  if (h->kind == B2_MATCH_LIKE) {
    const LikeProgram g = compile_like(p);
    h->items = static_cast<int64_t>(g.lit.size());
    h->n_seg = static_cast<int>(g.seg.size()) - 1;
    const size_t padded = (g.lit.size() + 7) & ~size_t(7);
    host.assign(2 * padded + g.seg.size() * sizeof(int64_t), 0);
    memcpy(host.data(), g.lit.data(), g.lit.size());
    memcpy(host.data() + padded, g.any.data(), g.any.size());
    memcpy(host.data() + 2 * padded, g.seg.data(), g.seg.size() * sizeof(int64_t));
  } else {
    h->m = static_cast<int64_t>(lit.size());
    for (int k = 0; k < 8 && k < h->m; ++k) h->head |= static_cast<uint64_t>(static_cast<uint8_t>(lit[k])) << (8 * k);
    host.assign(lit.begin(), lit.end());
  }
  if (!host.empty()) {
    int st = ctx->alloc(host.size(), &h->buf, s);
    if (st == B2_OK && cudaMemcpyAsync(h->buf, host.data(), host.size(), cudaMemcpyHostToDevice, s) != cudaSuccess)
      st = set_error(B2_CUDA_ERROR, "b2_string_match_create: pattern upload failed");
    if (st == B2_OK && cudaStreamSynchronize(s) != cudaSuccess)  // `host` goes out of scope
      st = set_error(B2_CUDA_ERROR, "b2_string_match_create: pattern upload failed");
    if (st != B2_OK) {
      free_match(h);
      return st;
    }
  }
  *out = h;
  return B2_OK;
}

extern "C" void b2_string_match_destroy(B2StringMatch* h) {
  if (!h) return;
  cudaSetDevice(h->ctx->device);
  free_match(h);
}

extern "C" int b2_string_match_info(const B2StringMatch* h, int32_t* runs_as, int64_t* literal_bytes) {
  if (!h) return set_error(B2_INVALID, "b2_string_match_info: null argument");
  if (runs_as) *runs_as = h->kind;
  if (literal_bytes) *literal_bytes = h->kind == B2_MATCH_LIKE ? h->items : h->m;
  return B2_OK;
}

extern "C" int b2_string_match(B2StringMatch* h, const B2Array* strings, B2Array* out, void* stream) {
  if (!h || !strings || !out) return set_error(B2_INVALID, "b2_string_match: null argument");
  if (!type_is_binary_like(strings->type))
    return set_error(B2_NOT_IMPLEMENTED, "string match: no kernel for type id %d", strings->type);
  const bool utf8 = strings->type == B2_STRING || strings->type == B2_LARGE_STRING;
  if (utf8 != h->utf8)
    return set_error(B2_TYPE_ERROR, "string match: the pattern was compiled for %s input, got type id %d",
                     h->utf8 ? "utf8" : "binary", strings->type);
  B2Context* ctx = h->ctx;
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->pick(stream);
  const int64_t n = strings->length;
  Temp data(ctx, s);
  B2_RETURN_NOT_OK(alloc_bits(ctx, n, &data, s));
  void* validity = nullptr;
  int64_t null_count = 0;
  B2_RETURN_NOT_OK(make_validity(ctx, strings, nullptr, n, &validity, &null_count, s));
  Temp vguard(ctx, s);
  vguard.ptr = validity;
  if (n > 0) {
    MatchArgs a{};
    a.offs = offsets_at(strings);
    a.bytes = static_cast<const uint8_t*>(strings->data2);
    a.n = n;
    a.n_words = (n + 31) >> 5;
    a.kind = h->kind;
    a.utf8 = h->utf8;
    a.out = data.as<uint32_t>();
    const bool like = h->kind == B2_MATCH_LIKE;
    if (like) {
      const size_t padded = (static_cast<size_t>(h->items) + 7) & ~size_t(7);
      a.lit = static_cast<const uint8_t*>(h->buf);
      a.any = a.lit + padded;
      a.seg = reinterpret_cast<const int64_t*>(a.lit + 2 * padded);
      a.n_seg = h->n_seg;
    } else {
      a.pat = static_cast<const uint8_t*>(h->buf);
      a.m = h->m;
      a.head = h->head;
    }
    const int grid = pred_grid(ctx, a.n_words);
    const bool wide = offset_width(strings->type) == 8;
    if (like) {
      if (wide) match_kernel<int64_t, true><<<grid, kPredBlock, 0, s>>>(a);
      else match_kernel<int32_t, true><<<grid, kPredBlock, 0, s>>>(a);
    } else {
      if (wide) match_kernel<int64_t, false><<<grid, kPredBlock, 0, s>>>(a);
      else match_kernel<int32_t, false><<<grid, kPredBlock, 0, s>>>(a);
    }
    B2_LAUNCHED();
  }
  fill_out(out, B2_BOOL, n, null_count, vguard.release(), data.release());
  return B2_OK;
}
