// string_transform.cu -- functions that compute from utf8 / large_utf8 / binary / large_binary columns: binary_length,
// utf8_length, ascii_upper, ascii_lower, utf8_slice_codeunits, binary_slice and binary_join_element_wise.
//
// Replaces:
//   BinaryLength (ScalarUnaryNotNull)                               kernels/scalar_string_ascii.cc:852-880
//   Utf8Length, util::UTF8Length                                    kernels/scalar_string_utf8.cc:664-690, util/utf8_internal.h:558
//   AsciiUpper / AsciiLower over StringDataTransform                kernels/scalar_string_ascii.cc:724-745,834-842
//   SliceCodeunitsTransform (UTF8AdvanceCodepoints[Reverse],
//     UTF8Decode[Reverse], UTF8Encode)                              kernels/scalar_string_utf8.cc:1157-1348, util/utf8_internal.h:330-520
//   SliceBytesTransform                                             kernels/scalar_string_ascii.cc:2636-2800
//   StringTransformExecBase::Execute, StringSliceTransformBase      kernels/scalar_string_internal.h:80-117,259-273
//   BinaryJoinElementWise with JoinOptions                          kernels/scalar_string_ascii.cc:3298-3420
// Semantics kept: lengths and case maps compute every slot, the slices write an empty value for a null row, and the
// output validity of all of these is the input's.  The join's validity is its own: a row is null when its separator
// is, or (EMIT_NULL) when any value is; SKIP drops a null value with its separator, REPLACE puts null_replacement in
// its place, and a call with only the separator gives "" on every valid row.  An int32-offset join whose output
// exceeds 2^31 - 2 bytes fails like BaseBinaryBuilder::ReserveData.  step == 0 is "Slice step cannot be zero"; a UTF-8
// decode error in the part of a valid row the slice walks is "Invalid UTF8 sequence in input".
//
// Design.
//   lengths: one streaming pass.  Warp w owns 32-row groups and lane l row 32w + l: binary_length is a difference of
//     offsets, utf8_length counts the bytes that are not 10xxxxxx with one popcount per 8-byte word.  A row longer than
//     kLongRow bytes is counted by the whole warp (256 bytes per step, then a warp sum), as string_predicates.cu does.
//   ascii case: one streaming pass.  The offsets are rebased to 0 and the contiguous span [offsets[0], offsets[n]) is
//     mapped 8 bytes at a time with a SWAR test for a..z / A..Z; every aligned output word is written once.  Null rows
//     keep their mapped bytes, as they do in the reference.
//   slices and join: sizes pass -> tile scan (launch_exclusive_scan_i64) -> write pass.  A CTA owns kTile rows, each
//     thread 8 consecutive ones.  Both passes evaluate each row from its inputs (a slice range, a code-point walk, or
//     the join's pieces); the write pass block-scans the row sizes into output offsets, stages them in shared memory
//     and then, for step-1 slices and the join, every thread produces aligned 8-byte words of the tile's contiguous
//     output range, gathering each from the row pieces that cover it.  A slice with |step| > 1 or step < 0 is written
//     by the lane that owns the row, a binary one of more than kLongRow bytes by the whole warp.  The utf8 code-point
//     walks stay one lane per row (DESIGN, string transforms: the decoder's position is sequential).
// Bytes outside a row are never read: a code point cut off by the row's end (or, walking backwards, by its start) is
// a decode error here, where the reference's decoder reads on into the neighbouring row.
#include <string>
#include <vector>

#include "bitmap.h"
#include "common.cuh"
#include "context.h"

namespace b2 {

constexpr int kStrBlock = 256;
constexpr int64_t kLongRow = 1024;  // bytes above which the warp counts a row's code points together
constexpr int kTile = 2048;         // rows per CTA of the slice / join builder
constexpr int kRowsPerThread = kTile / kStrBlock;
constexpr int kBuildBlocksPerSM = 4;  // the builder's register budget: up to 64 per thread, no spills
constexpr int64_t kI64Max = INT64_MAX;

__device__ __forceinline__ uint32_t byte_at(const uint8_t* p) { return static_cast<uint32_t>(load_bytes8(p, 1)); }

// bytes of an 8-byte word (nb valid) that are not UTF-8 continuation bytes
__device__ __forceinline__ int lead_bytes(uint64_t w, int nb) {
  const uint64_t cont = w & ~(w << 1) & 0x8080808080808080ull;  // bit 7 set, bit 6 clear
  return nb - __popcll(cont);
}

// ---------------------------------------------------------------------------------------------------------------------
// lengths
// ---------------------------------------------------------------------------------------------------------------------
template <typename OffT, typename OutT, bool UTF8>
__global__ void __launch_bounds__(kStrBlock) length_kernel(const OffT* __restrict__ offs, const uint8_t* bytes, int64_t n,
                                                           int64_t n_groups, OutT* __restrict__ out) {
  const unsigned lane = lane_id();
  const int64_t warp = (blockIdx.x * (int64_t)kStrBlock + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * kStrBlock) >> 5;
  for (int64_t w = warp; w < n_groups; w += n_warps) {
    const int64_t i = (w << 5) + lane;
    const bool in = i < n;
    int64_t o0 = 0, len = 0;
    if (in) {
      o0 = static_cast<int64_t>(offs[i]);
      len = static_cast<int64_t>(offs[i + 1]) - o0;
    }
    if constexpr (!UTF8) {
      if (in) st_stream(out + i, static_cast<OutT>(len));
    } else {
      const bool lng = in && len > kLongRow;
      int64_t count = 0;
      if (in && !lng) {
        const uint8_t* p = bytes + o0;
        for (int64_t o = 0; o < len; o += 8) {
          const int nb = len - o >= 8 ? 8 : static_cast<int>(len - o);
          count += lead_bytes(load_bytes8(p + o, nb), nb);
        }
      }
      for (unsigned longs = __ballot_sync(0xffffffffu, lng); longs; longs &= longs - 1) {
        const int src = __ffs(longs) - 1;
        const uint8_t* p = bytes + __shfl_sync(0xffffffffu, static_cast<long long>(o0), src);
        const int64_t ln = __shfl_sync(0xffffffffu, static_cast<long long>(len), src);
        int64_t c = 0;
        for (int64_t o = lane * 8; o < ln; o += 32 * 8) {
          const int nb = ln - o >= 8 ? 8 : static_cast<int>(ln - o);
          c += lead_bytes(load_bytes8(p + o, nb), nb);
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
        if (lane == src) count = c;
      }
      if (in) st_stream(out + i, static_cast<OutT>(count));
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// ascii_upper / ascii_lower
// ---------------------------------------------------------------------------------------------------------------------
// flips bit 5 of every byte in A..Z (upper == false) or a..z (upper == true)
__device__ __forceinline__ uint64_t ascii_case_word(uint64_t w, bool upper) {
  const uint64_t hept = w & 0x7f7f7f7f7f7f7f7full;
  const uint64_t lo = upper ? 0x1f1f1f1f1f1f1f1full : 0x3f3f3f3f3f3f3f3full;  // 0x80 - 'a'   / 0x80 - 'A'
  const uint64_t hi = upper ? 0x0505050505050505ull : 0x2525252525252525ull;  // 0x80 - 'z' - 1 / 0x80 - 'Z' - 1
  const uint64_t in_range = (hept + lo) & ~(hept + hi) & ~w & 0x8080808080808080ull;
  return w ^ (in_range >> 2);
}

template <typename OffT>
__global__ void __launch_bounds__(kStrBlock) ascii_case_kernel(const OffT* __restrict__ offs, const uint8_t* src, int64_t n,
                                                               int64_t nbytes, bool upper, OffT* __restrict__ out_offs,
                                                               uint64_t* __restrict__ out_words) {
  const OffT base = offs[0];
  const int64_t stride = (int64_t)gridDim.x * kStrBlock;
  const int64_t t0 = blockIdx.x * (int64_t)kStrBlock + threadIdx.x;
  for (int64_t i = t0; i <= n; i += stride) st_stream(out_offs + i, static_cast<OffT>(offs[i] - base));
  const uint8_t* p = src + static_cast<int64_t>(base);
  const int64_t n_words = (nbytes + 7) >> 3;
  for (int64_t k = t0; k < n_words; k += stride) {
    const int nb = nbytes - 8 * k >= 8 ? 8 : static_cast<int>(nbytes - 8 * k);
    st_stream(out_words + k, ascii_case_word(load_bytes8(p + 8 * k, nb), upper));
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// slices: the reference's index arithmetic, per row
// ---------------------------------------------------------------------------------------------------------------------
struct Row {
  const uint8_t* p;
  int64_t len;
};

// UTF8Decode at byte i of the row: the code point's bytes (1..4), or 0 on a decode error.  Overlong forms decode as
// the reference's decoder decodes them.
__device__ __forceinline__ int decode_fwd(Row r, int64_t i, uint32_t* cp) {
  const uint32_t c = byte_at(r.p + i);
  if (c < 0x80) {
    *cp = c;
    return 1;
  }
  const int n = c < 0xc0 ? 0 : c < 0xe0 ? 2 : c < 0xf0 ? 3 : c < 0xf8 ? 4 : 0;
  if (n == 0) return 0;
  uint32_t v = c & (0x7fu >> n);
  for (int k = 1; k < n; ++k) {
    if (i + k >= r.len) return 0;
    const uint32_t d = byte_at(r.p + i + k);
    if ((d & 0xc0) != 0x80) return 0;
    v = (v << 6) | (d & 0x3f);
  }
  *cp = v;
  return n;
}

// UTF8DecodeReverse with byte i of the row the code point's last byte: its bytes (1..4), or 0
__device__ __forceinline__ int decode_rev(Row r, int64_t i, uint32_t* cp) {
  const uint32_t c = byte_at(r.p + i);
  if (c < 0x80) {
    *cp = c;
    return 1;
  }
  if ((c & 0xc0) != 0x80) return 0;
  uint32_t v = c & 0x3f;
  for (int k = 1; k < 4; ++k) {
    if (i - k < 0) return 0;
    const uint32_t d = byte_at(r.p + i - k);
    const uint32_t lead_mask = k == 1 ? 0xe0 : k == 2 ? 0xf0 : 0xf8;
    if ((d & lead_mask) == ((lead_mask << 1) & 0xff)) {
      *cp = ((d & (0x7fu >> (k + 1))) << (6 * k)) | v;
      return k + 1;
    }
    if (k == 3 || (d & 0xc0) != 0x80) return 0;
    v |= (d & 0x3f) << (6 * k);
  }
  return 0;
}

__device__ __forceinline__ int encoded_len(uint32_t cp) { return cp < 0x80 ? 1 : cp < 0x800 ? 2 : cp < 0x10000 ? 3 : 4; }

__device__ __forceinline__ uint32_t encode(uint32_t cp, uint8_t* out) {
  if (cp < 0x80) {
    out[0] = static_cast<uint8_t>(cp);
    return 1;
  }
  if (cp < 0x800) {
    out[0] = static_cast<uint8_t>(0xc0 + (cp >> 6));
    out[1] = static_cast<uint8_t>(0x80 + (cp & 0x3f));
    return 2;
  }
  if (cp < 0x10000) {
    out[0] = static_cast<uint8_t>(0xe0 + (cp >> 12));
    out[1] = static_cast<uint8_t>(0x80 + ((cp >> 6) & 0x3f));
    out[2] = static_cast<uint8_t>(0x80 + (cp & 0x3f));
    return 3;
  }
  out[0] = static_cast<uint8_t>(0xf0 + (cp >> 18));
  out[1] = static_cast<uint8_t>(0x80 + ((cp >> 12) & 0x3f));
  out[2] = static_cast<uint8_t>(0x80 + ((cp >> 6) & 0x3f));
  out[3] = static_cast<uint8_t>(0x80 + (cp & 0x3f));
  return 4;
}

// UTF8AdvanceCodepoints from byte `from`: the start of code point n (counting from 0), or the row's end; -1 on a decode
// error.  n counts down and stops at 0 only, so a negative n (the reference's wrapped start + 1) walks to the end.
__device__ __forceinline__ int64_t advance(Row r, int64_t from, int64_t n) {
  int64_t i = from;
  while (i < r.len) {
    uint32_t cp;
    const int k = decode_fwd(r, i, &cp);
    if (!k) return -1;
    if (n == 0) return i;
    n = static_cast<int64_t>(static_cast<uint64_t>(n) - 1);
    i += k;
  }
  return r.len;
}

// UTF8AdvanceCodepointsReverse over [first, len): the end of the n-th code point counted from the row's end, or first
__device__ __forceinline__ int64_t advance_rev(Row r, int64_t first, int64_t n) {
  int64_t i = r.len - 1;
  while (i >= first) {
    uint32_t cp;
    const int k = decode_rev(r, i, &cp);
    if (!k) return -1;
    if (n == 0) return i + 1;
    n = static_cast<int64_t>(static_cast<uint64_t>(n) - 1);
    i -= k;
  }
  return first;
}

__device__ __forceinline__ int64_t negate_sat(int64_t v) { return v < -kI64Max ? kI64Max : -v; }
// the reference's int64 arithmetic where it can wrap (two's complement)
__device__ __forceinline__ int64_t wrap_add(int64_t a, int64_t b) {
  return static_cast<int64_t>(static_cast<uint64_t>(a) + static_cast<uint64_t>(b));
}
__device__ __forceinline__ int64_t wrap_neg(int64_t a) { return static_cast<int64_t>(0 - static_cast<uint64_t>(a)); }

struct SliceSpec {
  int64_t start, stop, step;
};

// A slice of one row: the byte range it reads ([b, e) forward, (e, b] backward; b == e: a zero-length slice), or a
// decode error (bad).
struct Range {
  int64_t b, e;
  bool bad;
};
constexpr Range kBadRange{0, 0, true};

// SliceCodeunitsTransform::SliceForward / SliceBackward's ranges, in code points
__device__ __forceinline__ Range utf8_range(Row r, const SliceSpec& o) {
  if (o.step >= 1) {
    int64_t b, e;
    if (o.start >= 0) {
      b = advance(r, 0, o.start);
      if (b < 0) return kBadRange;
      if (o.stop > o.start) e = advance(r, b, o.stop - o.start);
      else if (o.stop < 0) e = advance_rev(r, b, negate_sat(o.stop));
      else return {0, 0, false};
    } else {
      b = advance_rev(r, 0, wrap_neg(o.start));
      if (b < 0) return kBadRange;
      if (o.stop > 0) {
        e = advance(r, 0, o.stop);
        if (e >= 0 && e <= b) return {0, 0, false};
      } else if (o.stop < 0 && o.stop > o.start) {
        e = advance_rev(r, b, negate_sat(o.stop));
      } else {
        return {0, 0, false};
      }
    }
    if (e < 0) return kBadRange;
    return {b, e, false};
  }
  const int64_t b = o.start >= 0 ? advance(r, 0, wrap_add(o.start, 1)) : advance_rev(r, 0, wrap_add(wrap_neg(o.start), -1));
  if (b < 0) return kBadRange;
  const int64_t stop1 = (o.stop < kI64Max - 1 ? o.stop : kI64Max - 1) + 1;
  const int64_t e = o.stop >= 0 ? advance(r, 0, stop1) : advance_rev(r, 0, negate_sat(o.stop) - 1);
  if (e < 0) return kBadRange;
  return {b - 1, e - 1, false};
}

// SliceBytesTransform::SliceForwardRange / SliceBackwardRange, without the reference's int64 overflow at start or
// stop == INT64_MAX
__device__ __forceinline__ Range binary_range(int64_t len, const SliceSpec& o) {
  if (len == 0) return {0, 0, false};
  if (o.step >= 1) {
    int64_t b, e;
    if (o.start >= 0) {
      b = o.start < len ? o.start : len;
      if (o.stop > o.start) {
        const int64_t length = o.stop - o.start;
        e = length < len - b ? b + length : len;
      } else if (o.stop < 0) {
        e = len + o.stop > b ? len + o.stop : b;
      } else {
        return {0, 0, false};
      }
    } else {
      b = len + o.start > 0 ? len + o.start : 0;
      if (o.stop > 0) {
        e = o.stop < len ? o.stop : len;
        if (e <= b) return {0, 0, false};
      } else if (o.stop < 0 && o.stop > o.start) {
        e = len + o.stop > b ? len + o.stop : b;
      } else {
        return {0, 0, false};
      }
    }
    return {b, e, false};
  }
  int64_t b = o.start >= 0 ? (o.start < len ? o.start + 1 : len) : (len + o.start + 1 > 0 ? len + o.start + 1 : 0);
  int64_t e = o.stop >= 0 ? (o.stop < len ? o.stop + 1 : len) : (len + o.stop + 1 > 0 ? len + o.stop + 1 : 0);
  --b;
  --e;
  if (b <= e) return {0, 0, false};
  return {b, e, false};
}

// items of a strided walk over (e, b] or [b, e) with |step| >= 1: ceil(|b - e| / |step|)
// (span > 0).  The rare quotient of a row of 4 GiB or more is a shift-subtract division, so no kernel calls the 64-bit
// division routine.
__device__ __forceinline__ int64_t strided_count(int64_t span, int64_t step) {
  const uint64_t a = step < 0 ? 0 - static_cast<uint64_t>(step) : static_cast<uint64_t>(step);
  const uint64_t m = static_cast<uint64_t>(span) - 1;  // ceil(span / a) = floor((span - 1) / a) + 1
  if (a > m) return 1;
  uint64_t q = 0;
  if ((m >> 32) == 0) {
    q = static_cast<uint32_t>(m) / static_cast<uint32_t>(a);
  } else {
    uint64_t r = 0;
    for (int b = 63; b >= 0; --b) {
      r = (r << 1) | ((m >> b) & 1);
      if (r >= a) {
        r -= a;
        q |= 1ull << b;
      }
    }
  }
  return static_cast<int64_t>(q) + 1;
}

// the utf8 slice of a row with step != 1: its output bytes, written to out unless it is null; -1 on a decode error
__device__ __forceinline__ int64_t utf8_strided(Row r, Range g, int64_t step, uint8_t* out) {
  int64_t n = 0;
  uint32_t cp;
  if (step > 0) {
    const uint64_t skips = static_cast<uint64_t>(step) - 1;
    int64_t i = g.b;
    while (i < g.e) {
      const int k = decode_fwd(r, i, &cp);
      if (!k) return -1;
      i += k;
      n += out ? encode(cp, out + n) : encoded_len(cp);
      for (uint64_t s = 0; s < skips && i < g.e; ++s) {
        const int k2 = decode_fwd(r, i, &cp);
        if (!k2) return -1;
        i += k2;
      }
    }
  } else {
    const uint64_t skips = (0 - static_cast<uint64_t>(step)) - 1;
    int64_t i = g.b;
    while (i > g.e) {
      const int k = decode_rev(r, i, &cp);
      if (!k) return -1;
      i -= k;
      n += out ? encode(cp, out + n) : encoded_len(cp);
      for (uint64_t s = 0; s < skips && i > g.e; ++s) {
        const int k2 = decode_rev(r, i, &cp);
        if (!k2) return -1;
        i -= k2;
      }
    }
  }
  return n;
}

// ---------------------------------------------------------------------------------------------------------------------
// the slice / join builder
// ---------------------------------------------------------------------------------------------------------------------
enum BuildMode { kSpan = 0, kStrided = 1, kJoin = 2 };

struct JoinOp {
  const void* offs;  // array: its offsets at its offset; NULL for a scalar
  const uint8_t* bytes;
  BitmapReader valid;
  int64_t len;  // scalar: its byte length
  int32_t scalar_valid;
  int32_t pad;
};

struct BuildArgs {
  const void* offs;  // slice input at its offset
  const uint8_t* bytes;
  BitmapReader valid;
  SliceSpec sl;
  bool utf8;
  const JoinOp* ops;  // join: the values, then the separator
  int n_ops;
  int null_handling;
  const uint8_t* repl;
  int64_t repl_len;
  int64_t n;
  int64_t* tile_bytes;  // sizes pass: per-tile bytes; write pass: their exclusive prefix
  void* out_offs;
  uint8_t* out_bytes;
  uint32_t* out_valid;  // join only
  unsigned long long* first_bad;  // sizes pass: the first row with a decode error
  unsigned long long* valid_count;  // sizes pass, join: valid rows
  int64_t* oversize;  // sizes pass: a tile's output reaches 4 GiB
};

template <typename OffT>
__device__ __forceinline__ Row row_of(const void* offs, const uint8_t* bytes, int64_t i) {
  const OffT* o = static_cast<const OffT*>(offs);
  const int64_t o0 = static_cast<int64_t>(o[i]);
  return Row{bytes + o0, static_cast<int64_t>(o[i + 1]) - o0};
}

template <typename OffT>
__device__ __forceinline__ bool join_operand(const JoinOp& op, int64_t i, Row* r) {
  if (!op.offs) {
    *r = Row{op.bytes, op.len};
    return op.scalar_valid != 0;
  }
  *r = row_of<OffT>(op.offs, op.bytes, i);
  return op.valid.bit(i);
}

// the join of row i: whether it is valid and its bytes (CalculateRowSize)
template <typename OffT>
__device__ __forceinline__ bool join_size(const BuildArgs& a, int64_t i, int64_t* size) {
  Row sep;
  if (!join_operand<OffT>(a.ops[a.n_ops - 1], i, &sep)) return false;
  int64_t total = 0, emitted = 0;
  for (int c = 0; c + 1 < a.n_ops; ++c) {
    Row v;
    if (!join_operand<OffT>(a.ops[c], i, &v)) {
      if (a.null_handling == B2_JOIN_EMIT_NULL) return false;
      if (a.null_handling == B2_JOIN_SKIP) continue;
      v.len = a.repl_len;
    }
    total += v.len;
    ++emitted;
  }
  if (emitted > 1) total += (emitted - 1) * sep.len;
  *size = total;
  return true;
}

// up to `want` bytes of row i's join output from byte `pos`, all from the one piece that holds pos; *took = how many
template <typename OffT>
__device__ __forceinline__ uint64_t join_bytes(const BuildArgs& a, int64_t i, int64_t pos, int want, int* took) {
  Row sep;
  join_operand<OffT>(a.ops[a.n_ops - 1], i, &sep);
  int64_t at = 0;
  bool first = true;
  Row piece{nullptr, 0};
  for (int c = 0; c + 1 < a.n_ops; ++c) {
    Row v;
    if (!join_operand<OffT>(a.ops[c], i, &v)) {
      if (a.null_handling == B2_JOIN_SKIP) continue;
      v = Row{a.repl, a.repl_len};
    }
    if (!first) {
      if (pos < at + sep.len) {
        piece = Row{sep.p + (pos - at), sep.len - (pos - at)};
        break;
      }
      at += sep.len;
    }
    first = false;
    if (pos < at + v.len) {
      piece = Row{v.p + (pos - at), v.len - (pos - at)};
      break;
    }
    at += v.len;
  }
  const int t = piece.len < want ? static_cast<int>(piece.len) : want;
  *took = t;
  return load_bytes8(piece.p, t);
}

// what the sizes and write passes know of one row
struct RowOut {
  int64_t len;   // output bytes
  int64_t src;   // kSpan: the byte the slice starts at, relative to the input's data buffer
  bool valid;
  bool bad;      // a decode error
};

template <typename OffT, int MODE>
__device__ __forceinline__ RowOut row_out(const BuildArgs& a, int64_t i) {
  RowOut o{0, 0, true, false};
  if constexpr (MODE == kJoin) {
    o.valid = join_size<OffT>(a, i, &o.len);
    if (!o.valid) o.len = 0;
    return o;
  } else {
    if (!a.valid.bit(i)) return o;  // a null row: an empty value, nothing walked
    const Row r = row_of<OffT>(a.offs, a.bytes, i);
    const Range g = a.utf8 ? utf8_range(r, a.sl) : binary_range(r.len, a.sl);
    if (g.bad) {
      o.bad = true;
      return o;
    }
    if (g.b == g.e) return o;
    if constexpr (MODE == kSpan) {
      o.len = g.e - g.b;
      o.src = (r.p - a.bytes) + g.b;
    } else if (a.utf8) {
      o.len = utf8_strided(r, g, a.sl.step, nullptr);
      if (o.len < 0) {
        o.bad = true;
        o.len = 0;
      }
    } else {
      o.len = strided_count(a.sl.step > 0 ? g.e - g.b : g.b - g.e, a.sl.step);
    }
    return o;
  }
}

// exclusive block scan of one int64 per thread; *total = the block's sum
__device__ __forceinline__ int64_t block_scan(int64_t v, int64_t* total) {
  __shared__ int64_t s_w[kStrBlock / 32];
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  int64_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) s_w[warp] = incl;
  __syncthreads();
  int64_t woff = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kStrBlock / 32; ++w) {
    const int64_t x = s_w[w];
    if (w < static_cast<int>(warp)) woff += x;
    tot += x;
  }
  *total = tot;
  return woff + incl - v;
}

template <typename OffT, int MODE, bool WRITE>
__global__ void __launch_bounds__(kStrBlock, kBuildBlocksPerSM) build_kernel(const BuildArgs a) {
  __shared__ uint32_t s_out[WRITE ? kTile + 1 : 1];
  __shared__ int64_t s_src[(WRITE && MODE == kSpan) ? kTile : 1];
  __shared__ uint32_t s_bits[(WRITE && MODE == kJoin) ? kTile / 32 : 1];
  const int64_t tile = blockIdx.x;
  const int64_t row0 = tile * kTile + threadIdx.x * kRowsPerThread;
  if constexpr (WRITE && MODE == kJoin) {
    for (int k = threadIdx.x; k < kTile / 32; k += kStrBlock) s_bits[k] = 0;
    __syncthreads();
  }
  // each row's size (and span start) is staged at its tile row in s_out (s_src) and turned into its output offset after
  // the block scan, by the thread that owns it
  unsigned vb = 0;
  int64_t local = 0;
#pragma unroll 1
  for (int k = 0; k < kRowsPerThread; ++k) {
    const int64_t i = row0 + k;
    if (i >= a.n) break;
    const RowOut r = row_out<OffT, MODE>(a, i);
    if (!WRITE && r.bad) atomicMin(a.first_bad, static_cast<unsigned long long>(i));
    if constexpr (WRITE) {
      s_out[threadIdx.x * kRowsPerThread + k] = static_cast<uint32_t>(r.len);
      if constexpr (MODE == kSpan) s_src[threadIdx.x * kRowsPerThread + k] = r.src;
    }
    local += r.len;
    if (r.valid) vb |= 1u << k;
  }
  int64_t total;
  const int64_t excl = block_scan(local, &total);
  if constexpr (!WRITE) {
    if (MODE == kJoin) {
      const int64_t cnt = block_sum<kStrBlock>(__popc(vb));
      if (threadIdx.x == 0 && cnt) atomicAdd(a.valid_count, static_cast<unsigned long long>(cnt));
    }
    if (threadIdx.x == 0) {
      a.tile_bytes[tile] = total;
      if (total >= (1ll << 32)) *a.oversize = 1;
    }
    return;
  } else {
    OffT* out_offs = static_cast<OffT*>(a.out_offs);
    const int64_t byte_base = a.tile_bytes[tile];
    const int64_t tile_left = a.n - tile * kTile;
    const int tile_n = tile_left < kTile ? static_cast<int>(tile_left) : kTile;
    uint32_t run = static_cast<uint32_t>(excl);
#pragma unroll
    for (int k = 0; k < kRowsPerThread; ++k) {
      const int lr = threadIdx.x * kRowsPerThread + k;
      if (lr < tile_n) {
        const uint32_t len = s_out[lr];
        s_out[lr] = run;
        out_offs[row0 + k] = static_cast<OffT>(byte_base + run);
        run += len;
      }
    }
    if constexpr (MODE == kJoin) {
      if (vb) atomicOr(&s_bits[(threadIdx.x * kRowsPerThread) >> 5], vb << ((threadIdx.x * kRowsPerThread) & 31));
    }
    if (threadIdx.x == 0) {
      s_out[tile_n] = static_cast<uint32_t>(total);
      if (tile == gridDim.x - 1) out_offs[a.n] = static_cast<OffT>(byte_base + total);
    }
    __syncthreads();
    if constexpr (MODE == kJoin) {
      if (threadIdx.x < kTile / 32 && static_cast<int>(threadIdx.x) * 32 < tile_n)
        a.out_valid[tile * (kTile / 32) + threadIdx.x] = s_bits[threadIdx.x];
    }
    uint8_t* d0 = a.out_bytes + byte_base;
    if constexpr (MODE == kStrided) {
      // the lane that owns a row writes it; a binary row of more than kLongRow output bytes is written by the whole warp
      // (lane l writes bytes l, l + 32, ...), so one long row does not serialise its warp
#pragma unroll 1
      for (int k = 0; k < kRowsPerThread; ++k) {
        const int lr = threadIdx.x * kRowsPerThread + k;
        const uint32_t bytes = lr < tile_n ? s_out[lr + 1] - s_out[lr] : 0;
        const bool lng = !a.utf8 && bytes > kLongRow;
        const uint8_t* src = nullptr;
        if (bytes) {
          const Row r = row_of<OffT>(a.offs, a.bytes, row0 + k);
          const Range g = a.utf8 ? utf8_range(r, a.sl) : binary_range(r.len, a.sl);
          uint8_t* out = d0 + s_out[lr];
          src = r.p + g.b;
          if (a.utf8) {
            utf8_strided(r, g, a.sl.step, out);
          } else if (!lng) {
            int64_t j = g.b;
            for (uint32_t q = 0; q < bytes; ++q, j = wrap_add(j, a.sl.step)) out[q] = static_cast<uint8_t>(byte_at(r.p + j));
          }
        }
        for (unsigned longs = __ballot_sync(0xffffffffu, lng); longs; longs &= longs - 1) {
          const int owner = __ffs(longs) - 1;
          const uint8_t* p = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(src), owner));
          const uint32_t nb = __shfl_sync(0xffffffffu, bytes, owner);
          uint8_t* out = d0 + s_out[__shfl_sync(0xffffffffu, lr, owner)];
          for (uint32_t q = lane_id(); q < nb; q += 32) out[q] = static_cast<uint8_t>(byte_at(p + static_cast<int64_t>(q) * a.sl.step));
        }
      }
    } else {
      // every thread produces aligned 8-byte words of the tile's output [0, total): the rows (and, for the join, the
      // pieces) that cover a word are found from the staged offsets; head and tail bytes are written one at a time
      const int64_t tile_bytes = total;
      if (tile_bytes == 0) return;
      int64_t head = static_cast<int64_t>((8 - (reinterpret_cast<uintptr_t>(d0) & 7)) & 7);
      if (head > tile_bytes) head = tile_bytes;
      const int64_t words = (tile_bytes - head) >> 3;
      const int64_t tail_start = head + (words << 3);
      auto find_row = [&](uint32_t pos) {  // the largest j with s_out[j] <= pos
        int lo = 0, hi = tile_n;
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (s_out[mid] <= pos) lo = mid;
          else hi = mid;
        }
        return lo;
      };
      auto gather = [&](uint32_t pos, int nb) {
        int j = find_row(pos);
        uint64_t w = 0;
        int filled = 0;
        while (filled < nb) {
          while (pos >= s_out[j + 1]) ++j;  // skips empty rows; s_out[tile_n] = tile_bytes > pos
          const uint32_t avail = s_out[j + 1] - pos;
          const int want = avail < static_cast<uint32_t>(nb - filled) ? static_cast<int>(avail) : nb - filled;
          int took = want;
          uint64_t v;
          if constexpr (MODE == kSpan) v = load_bytes8(a.bytes + s_src[j] + (pos - s_out[j]), want);
          else v = join_bytes<OffT>(a, tile * kTile + j, pos - s_out[j], want, &took);
          w |= v << (8 * filled);
          filled += took;
          pos += took;
        }
        return w;
      };
      for (int64_t c = threadIdx.x; c < words; c += kStrBlock) {
        const uint32_t pos = static_cast<uint32_t>(head + (c << 3));
        st_stream(reinterpret_cast<uint64_t*>(d0 + pos), gather(pos, 8));
      }
      const int64_t edge = head + (tile_bytes - tail_start);
      for (int64_t e = threadIdx.x; e < edge; e += kStrBlock) {
        const uint32_t pos = static_cast<uint32_t>(e < head ? e : tail_start + (e - head));
        d0[pos] = static_cast<uint8_t>(gather(pos, 1));
      }
    }
  }
}

inline int stream_grid(B2Context* ctx, int64_t items, int64_t per_block) {
  return grid_for(items, per_block, ctx->sm_count * (2048 / kStrBlock));
}

const void* offsets_at(const B2Array* x) {
  return static_cast<const uint8_t*>(x->data) + x->offset * offset_width(x->type);
}

bool is_utf8_type(int t) { return t == B2_STRING || t == B2_LARGE_STRING; }

// an empty binary-like output of type t (one zero offset)
int empty_binary(B2Context* ctx, int type, B2Array* out, cudaStream_t s) {
  Temp offs(ctx, s);
  B2_RETURN_NOT_OK(offs.alloc(offset_width(type)));
  B2_CUDA(cudaMemsetAsync(offs.ptr, 0, offset_width(type), s));
  fill_out(out, type, 0, 0, nullptr, offs.release(), nullptr);
  return B2_OK;
}

// The sizes -> scan -> write builder over n rows of output type `type`.  validity / null_count: the output's, for a
// slice (the input's); the join computes its own.
template <typename OffT, int MODE>
int build(B2Context* ctx, BuildArgs a, int type, void* validity, int64_t null_count, B2Array* out, cudaStream_t s) {
  Temp vguard(ctx, s);
  vguard.ptr = validity;
  const int64_t n = a.n;
  const int64_t n_tiles = (n + kTile - 1) / kTile;
  Temp tile_bytes(ctx, s), byte_offsets(ctx, s);
  B2_RETURN_NOT_OK(tile_bytes.alloc(sizeof(int64_t) * n_tiles));
  B2_RETURN_NOT_OK(byte_offsets.alloc(sizeof(int64_t) * n_tiles));
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  B2_CUDA(cudaMemsetAsync(slot.dev() + 1, 0xff, 8, s));
  a.tile_bytes = tile_bytes.as<int64_t>();
  a.first_bad = reinterpret_cast<unsigned long long*>(slot.dev() + 1);
  a.valid_count = reinterpret_cast<unsigned long long*>(slot.dev() + 2);
  a.oversize = slot.dev() + 3;
  build_kernel<OffT, MODE, false><<<(unsigned)n_tiles, kStrBlock, 0, s>>>(a);
  B2_LAUNCHED();
  B2_RETURN_NOT_OK(launch_exclusive_scan_i64(tile_bytes.as<int64_t>(), n_tiles, byte_offsets.as<int64_t>(), slot.dev(), s));
  B2_RETURN_NOT_OK(slot.fetch(s));
  if (static_cast<uint64_t>(slot.host()[1]) != ~0ull) return set_error(B2_INVALID, "Invalid UTF8 sequence in input");
  const int64_t total = slot.host()[0];
  if (sizeof(OffT) == 4 && total > 2147483646ll)  // BaseBinaryBuilder::ReserveData (builder_binary.h:312-333)
    return set_error(B2_CAPACITY_ERROR, "array cannot contain more than 2147483646 bytes, have %lld", static_cast<long long>(total));
  if (slot.host()[3] != 0)
    return set_error(B2_NOT_IMPLEMENTED, "string transform: %d rows of this output hold 4 GiB or more of bytes", kTile);
  Temp offs(ctx, s), data(ctx, s), bits(ctx, s);
  B2_RETURN_NOT_OK(offs.alloc(sizeof(OffT) * (size_t)(n + 1)));
  B2_RETURN_NOT_OK(data.alloc((size_t)total + 8));
  if (MODE == kJoin) {
    null_count = n - slot.host()[2];
    B2_RETURN_NOT_OK(bits.alloc(bitmap_alloc_bytes(n) + kTile / 8));
    B2_CUDA(cudaMemsetAsync(bits.ptr, 0, bitmap_alloc_bytes(n) + kTile / 8, s));
  }
  a.tile_bytes = byte_offsets.as<int64_t>();
  a.out_offs = offs.ptr;
  a.out_bytes = data.as<uint8_t>();
  a.out_valid = bits.as<uint32_t>();
  build_kernel<OffT, MODE, true><<<(unsigned)n_tiles, kStrBlock, 0, s>>>(a);
  B2_LAUNCHED();
  if (MODE == kJoin && null_count) vguard.ptr = bits.release();
  fill_out(out, type, n, null_count, vguard.release(), offs.release(), data.release());
  return B2_OK;
}

}  // namespace b2

using namespace b2;

extern "C" int b2_string_length(B2Context* ctx, const B2Array* strings, int is_utf8, B2Array* out, void* stream) {
  if (!ctx || !strings || !out) return set_error(B2_INVALID, "b2_string_length: null argument");
  const char* fn = is_utf8 ? "utf8_length" : "binary_length";
  if (is_utf8 ? !is_utf8_type(strings->type) : !type_is_binary_like(strings->type))
    return set_error(B2_NOT_IMPLEMENTED, "%s: no kernel for type id %d", fn, strings->type);
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->pick(stream);
  const int64_t n = strings->length;
  const bool wide = offset_width(strings->type) == 8;
  const int out_type = wide ? B2_INT64 : B2_INT32;
  Temp data(ctx, s);
  B2_RETURN_NOT_OK(data.alloc((wide ? 8 : 4) * (size_t)n));
  void* validity = nullptr;
  int64_t null_count = 0;
  B2_RETURN_NOT_OK(make_validity(ctx, strings, nullptr, n, &validity, &null_count, s));
  Temp vguard(ctx, s);
  vguard.ptr = validity;
  if (n > 0) {
    const int64_t groups = (n + 31) >> 5;
    const int grid = stream_grid(ctx, groups, kStrBlock / 32);
    const uint8_t* bytes = static_cast<const uint8_t*>(strings->data2);
    const void* offs = offsets_at(strings);
    if (wide) {
      if (is_utf8) length_kernel<int64_t, int64_t, true><<<grid, kStrBlock, 0, s>>>(static_cast<const int64_t*>(offs), bytes, n, groups, data.as<int64_t>());
      else length_kernel<int64_t, int64_t, false><<<grid, kStrBlock, 0, s>>>(static_cast<const int64_t*>(offs), bytes, n, groups, data.as<int64_t>());
    } else {
      if (is_utf8) length_kernel<int32_t, int32_t, true><<<grid, kStrBlock, 0, s>>>(static_cast<const int32_t*>(offs), bytes, n, groups, data.as<int32_t>());
      else length_kernel<int32_t, int32_t, false><<<grid, kStrBlock, 0, s>>>(static_cast<const int32_t*>(offs), bytes, n, groups, data.as<int32_t>());
    }
    B2_LAUNCHED();
  }
  fill_out(out, out_type, n, null_count, vguard.release(), data.release());
  return B2_OK;
}

namespace {
template <typename OffT>
int ascii_case_typed(B2Context* ctx, const B2Array* strings, bool upper, void* validity, int64_t null_count, B2Array* out,
                     cudaStream_t s) {
  Temp vguard(ctx, s);
  vguard.ptr = validity;
  const int64_t n = strings->length;
  const OffT* offs = static_cast<const OffT*>(offsets_at(strings));
  ScalarSlot slot(ctx);
  B2_RETURN_NOT_OK(slot.zero(s));
  B2_CUDA(cudaMemcpyAsync(slot.dev(), offs, sizeof(OffT), cudaMemcpyDeviceToDevice, s));
  B2_CUDA(cudaMemcpyAsync(slot.dev() + 1, offs + n, sizeof(OffT), cudaMemcpyDeviceToDevice, s));
  B2_RETURN_NOT_OK(slot.fetch(s));
  OffT first, last;
  memcpy(&first, const_cast<int64_t*>(slot.host()), sizeof(OffT));
  memcpy(&last, const_cast<int64_t*>(slot.host() + 1), sizeof(OffT));
  const int64_t nbytes = static_cast<int64_t>(last) - static_cast<int64_t>(first);
  Temp o(ctx, s), data(ctx, s);
  B2_RETURN_NOT_OK(o.alloc(sizeof(OffT) * (size_t)(n + 1)));
  B2_RETURN_NOT_OK(data.alloc((size_t)((nbytes + 7) & ~int64_t(7))));
  const int64_t items = n + 1 > (nbytes + 7) / 8 ? n + 1 : (nbytes + 7) / 8;
  ascii_case_kernel<OffT><<<stream_grid(ctx, items, kStrBlock), kStrBlock, 0, s>>>(
      offs, static_cast<const uint8_t*>(strings->data2), n, nbytes, upper, o.as<OffT>(), data.as<uint64_t>());
  B2_LAUNCHED();
  fill_out(out, strings->type, n, null_count, vguard.release(), o.release(), data.release());
  return B2_OK;
}
}  // namespace

extern "C" int b2_ascii_case(B2Context* ctx, const B2Array* strings, int upper, B2Array* out, void* stream) {
  if (!ctx || !strings || !out) return set_error(B2_INVALID, "b2_ascii_case: null argument");
  if (!is_utf8_type(strings->type))
    return set_error(B2_NOT_IMPLEMENTED, "%s: no kernel for type id %d", upper ? "ascii_upper" : "ascii_lower", strings->type);
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->pick(stream);
  const int64_t n = strings->length;
  if (n == 0) return empty_binary(ctx, strings->type, out, s);
  void* validity = nullptr;
  int64_t null_count = 0;
  B2_RETURN_NOT_OK(make_validity(ctx, strings, nullptr, n, &validity, &null_count, s));
  if (offset_width(strings->type) == 8) return ascii_case_typed<int64_t>(ctx, strings, upper != 0, validity, null_count, out, s);
  return ascii_case_typed<int32_t>(ctx, strings, upper != 0, validity, null_count, out, s);
}

extern "C" int b2_string_slice(B2Context* ctx, const B2Array* strings, int64_t start, int64_t stop, int64_t step, int is_utf8,
                               B2Array* out, void* stream) {
  if (!ctx || !strings || !out) return set_error(B2_INVALID, "b2_string_slice: null argument");
  const bool utf8_in = is_utf8_type(strings->type);
  if (!type_is_binary_like(strings->type) || utf8_in != (is_utf8 != 0))
    return set_error(B2_NOT_IMPLEMENTED, "%s: no kernel for type id %d", is_utf8 ? "utf8_slice_codeunits" : "binary_slice",
                     strings->type);
  if (step == 0) return set_error(B2_INVALID, "Slice step cannot be zero");
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->pick(stream);
  const int64_t n = strings->length;
  if (n == 0) return empty_binary(ctx, strings->type, out, s);
  void* validity = nullptr;
  int64_t null_count = 0;
  B2_RETURN_NOT_OK(make_validity(ctx, strings, nullptr, n, &validity, &null_count, s));
  BuildArgs a{};
  a.offs = offsets_at(strings);
  a.bytes = static_cast<const uint8_t*>(strings->data2);
  a.valid = BitmapReader(strings->null_count == 0 ? nullptr : strings->validity, strings->offset, n);
  a.sl = SliceSpec{start, stop, step};
  a.utf8 = is_utf8 != 0;
  a.n = n;
  const bool span = step == 1;
  if (offset_width(strings->type) == 8) {
    return span ? build<int64_t, kSpan>(ctx, a, strings->type, validity, null_count, out, s)
                : build<int64_t, kStrided>(ctx, a, strings->type, validity, null_count, out, s);
  }
  return span ? build<int32_t, kSpan>(ctx, a, strings->type, validity, null_count, out, s)
              : build<int32_t, kStrided>(ctx, a, strings->type, validity, null_count, out, s);
}

extern "C" int b2_binary_join_element_wise(B2Context* ctx, const B2JoinOperand* operands, int n_operands, int null_handling,
                                           const void* replacement, int64_t replacement_length, B2Array* out, void* stream) {
  if (!ctx || !operands || !out || n_operands < 1) return set_error(B2_INVALID, "b2_binary_join_element_wise: null argument");
  if (null_handling < B2_JOIN_EMIT_NULL || null_handling > B2_JOIN_REPLACE)
    return set_error(B2_INVALID, "b2_binary_join_element_wise: unknown null handling %d", null_handling);
  if (replacement_length < 0 || (replacement_length > 0 && !replacement))
    return set_error(B2_INVALID, "b2_binary_join_element_wise: bad null replacement");
  const B2Array* first = nullptr;
  for (int c = 0; c < n_operands; ++c) {
    const B2JoinOperand& op = operands[c];
    if (op.array) {
      if (!type_is_binary_like(op.array->type))
        return set_error(B2_NOT_IMPLEMENTED, "binary_join_element_wise: no kernel for type id %d", op.array->type);
      if (!first) first = op.array;
      if (op.array->type != first->type)
        return set_error(B2_NOT_IMPLEMENTED, "binary_join_element_wise: no kernel for type ids %d and %d", first->type, op.array->type);
      if (op.array->length != first->length) return set_error(B2_INVALID, "Array arguments must all be the same length");
    } else if (op.length < 0 || (op.length > 0 && !op.bytes)) {
      return set_error(B2_INVALID, "b2_binary_join_element_wise: bad scalar operand %d", c);
    }
  }
  if (!first) return set_error(B2_INVALID, "b2_binary_join_element_wise: at least one operand must be an array");
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->pick(stream);
  const int64_t n = first->length;
  if (n == 0) return empty_binary(ctx, first->type, out, s);
  // one upload: the operand table, then every scalar's bytes and the replacement, each at an 8-byte boundary
  std::vector<JoinOp> ops(n_operands);
  size_t table = sizeof(JoinOp) * n_operands, at = table;
  std::vector<size_t> where(n_operands + 1);
  for (int c = 0; c <= n_operands; ++c) {
    where[c] = at;
    const int64_t len = c == n_operands ? replacement_length : (operands[c].array ? 0 : operands[c].length);
    at += (static_cast<size_t>(len) + 7) & ~size_t(7);
  }
  Temp dev(ctx, s);
  B2_RETURN_NOT_OK(dev.alloc(at));
  uint8_t* d = dev.as<uint8_t>();
  std::vector<uint8_t> host(at, 0);
  for (int c = 0; c < n_operands; ++c) {
    const B2JoinOperand& op = operands[c];
    JoinOp j{};
    if (op.array) {
      j.offs = offsets_at(op.array);
      j.bytes = static_cast<const uint8_t*>(op.array->data2);
      j.valid = BitmapReader(op.array->null_count == 0 ? nullptr : op.array->validity, op.array->offset, n);
    } else {
      j.bytes = d + where[c];
      j.len = op.length;
      j.scalar_valid = op.is_valid ? 1 : 0;
      if (op.length) memcpy(host.data() + where[c], op.bytes, op.length);
    }
    ops[c] = j;
  }
  memcpy(host.data(), ops.data(), table);
  if (replacement_length) memcpy(host.data() + where[n_operands], replacement, replacement_length);
  B2_CUDA(cudaMemcpyAsync(d, host.data(), at, cudaMemcpyHostToDevice, s));
  BuildArgs a{};
  a.ops = reinterpret_cast<const JoinOp*>(d);
  a.n_ops = n_operands;
  a.null_handling = null_handling;
  a.repl = d + where[n_operands];
  a.repl_len = replacement_length;
  a.n = n;
  // `host` outlives the upload: build() synchronises the stream before it returns
  if (offset_width(first->type) == 8) return build<int64_t, kJoin>(ctx, a, first->type, nullptr, 0, out, s);
  return build<int32_t, kJoin>(ctx, a, first->type, nullptr, 0, out, s);
}
