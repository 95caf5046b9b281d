"""A host restatement, without pyarrow.compute, of the string transforms the device runs (csrc/string_transform.cu):

  * binary_length / utf8_length: the bytes of a slot / its bytes that are not 10xxxxxx (util/utf8_internal.h:558);
  * ascii_upper / ascii_lower: a..z <-> A..Z, every other byte kept, offsets re-based to 0 (StringDataTransform);
  * utf8_slice_codeunits: SliceCodeunitsTransform (kernels/scalar_string_utf8.cc:1157-1348) line for line, with
    UTF8Decode / UTF8DecodeReverse / UTF8AdvanceCodepoints[Reverse] (util/utf8_internal.h:345-520) and the re-encoding of
    each code point a |step| > 1 or backward slice emits;
  * binary_slice: SliceBytesTransform's ranges (kernels/scalar_string_ascii.cc:2656-2770), in exact integers;
  * binary_join_element_wise: BinaryJoinElementWise (:3298-3420) with JoinOptions.

Python integers do not overflow: where the reference's int64 arithmetic wraps (start + 1 at INT64_MAX, -start at
INT64_MIN) the restatement follows the reference's result, which is what exact arithmetic gives for any real row.
A decode never reads outside its row: a sequence cut off by the row's end (or, backwards, its start) is invalid."""
import numpy as np
import pyarrow as pa

INT64_MAX = (1 << 63) - 1
INT64_MIN = -(1 << 63)
UTF8_TYPES = (pa.string(), pa.large_string())
BINARY_TYPES = (pa.binary(), pa.large_binary())
BINARY_LIKE = UTF8_TYPES + BINARY_TYPES
INVALID_UTF8 = "Invalid UTF8 sequence in input"


class InvalidUtf8(ValueError):
    """the reference's `Invalid: Invalid UTF8 sequence in input`"""


def slots(arr: pa.Array):
    """the bytes of every slot of a binary-like array, null slots included"""
    wide = arr.type in (pa.large_string(), pa.large_binary())
    bufs = arr.buffers()
    offs = np.frombuffer(bufs[1], np.int64 if wide else np.int32, count=arr.offset + len(arr) + 1)[arr.offset:]
    data = bufs[2].to_pybytes() if bufs[2] is not None else b""
    return [data[int(offs[i]):int(offs[i + 1])] for i in range(len(arr))]


def values(arr: pa.Array):
    """the bytes of each valid slot, None for a null"""
    valid = arr.is_valid().to_pylist() if arr.null_count else [True] * len(arr)
    return [s if v else None for s, v in zip(slots(arr), valid)]


def to_array(vals, type_) -> pa.Array:
    """an array of `type_` from bytes / None: offsets from 0, empty null slots (what the reference's builders write)"""
    if type_ in UTF8_TYPES:
        binary = pa.large_binary() if type_ == pa.large_string() else pa.binary()
        return pa.array(vals, binary).view(type_)
    return pa.array(vals, type_)


# ------------------------------------------------------------------------------------------------------------------
# lengths and ascii case
# ------------------------------------------------------------------------------------------------------------------
def binary_length(arr: pa.Array) -> pa.Array:
    out = pa.int64() if arr.type in (pa.large_string(), pa.large_binary()) else pa.int32()
    return pa.array([None if v is None else len(v) for v in values(arr)], out)


def utf8_length(arr: pa.Array) -> pa.Array:
    out = pa.int64() if arr.type == pa.large_string() else pa.int32()
    return pa.array([None if v is None else sum((c & 0xC0) != 0x80 for c in v) for v in values(arr)], out)


_UPPER = bytes.maketrans(bytes(range(97, 123)), bytes(range(65, 91)))
_LOWER = bytes.maketrans(bytes(range(65, 91)), bytes(range(97, 123)))


def ascii_case(arr: pa.Array, upper: bool) -> pa.Array:
    """the mapped values; the device also maps the bytes under null slots, as the reference does"""
    table = _UPPER if upper else _LOWER
    return to_array([None if v is None else v.translate(table) for v in values(arr)], arr.type)


# ------------------------------------------------------------------------------------------------------------------
# UTF-8 walk (util/utf8_internal.h)
# ------------------------------------------------------------------------------------------------------------------
def _decode(r: bytes, i: int):
    """UTF8Decode at byte i: (bytes, code point); raises on a bad sequence"""
    c = r[i]
    if c < 0x80:
        return 1, c
    n = 0 if c < 0xC0 else 2 if c < 0xE0 else 3 if c < 0xF0 else 4 if c < 0xF8 else 0
    if not n:
        raise InvalidUtf8(INVALID_UTF8)
    v = c & (0x7F >> n)
    for k in range(1, n):
        if i + k >= len(r) or (r[i + k] & 0xC0) != 0x80:
            raise InvalidUtf8(INVALID_UTF8)
        v = (v << 6) | (r[i + k] & 0x3F)
    return n, v


def _decode_rev(r: bytes, i: int):
    """UTF8DecodeReverse with byte i the code point's last byte: (bytes, code point)"""
    c = r[i]
    if c < 0x80:
        return 1, c
    if (c & 0xC0) != 0x80:
        raise InvalidUtf8(INVALID_UTF8)
    v = c & 0x3F
    for k, (mask, lead) in enumerate(((0xE0, 0xC0), (0xF0, 0xE0), (0xF8, 0xF0)), start=1):
        if i - k < 0:
            raise InvalidUtf8(INVALID_UTF8)
        d = r[i - k]
        if (d & mask) == lead:
            return k + 1, ((d & (0x7F >> (k + 1))) << (6 * k)) | v
        if k == 3 or (d & 0xC0) != 0x80:
            raise InvalidUtf8(INVALID_UTF8)
        v |= (d & 0x3F) << (6 * k)
    raise InvalidUtf8(INVALID_UTF8)


def _encode(cp: int) -> bytes:
    if cp < 0x80:
        return bytes([cp])
    if cp < 0x800:
        return bytes([0xC0 + (cp >> 6), 0x80 + (cp & 0x3F)])
    if cp < 0x10000:
        return bytes([0xE0 + (cp >> 12), 0x80 + ((cp >> 6) & 0x3F), 0x80 + (cp & 0x3F)])
    return bytes([0xF0 + (cp >> 18), 0x80 + ((cp >> 12) & 0x3F), 0x80 + ((cp >> 6) & 0x3F), 0x80 + (cp & 0x3F)])


def _advance(r: bytes, frm: int, n: int) -> int:
    """UTF8AdvanceCodepoints: where code point n starts (each one walked is decoded), or the end"""
    i = frm
    while i < len(r):
        k, _ = _decode(r, i)
        if n == 0:
            return i
        n -= 1
        i += k
    return len(r)


def _advance_rev(r: bytes, first: int, n: int) -> int:
    """UTF8AdvanceCodepointsReverse over [first, len)"""
    i = len(r) - 1
    while i >= first:
        k, _ = _decode_rev(r, i)
        if n == 0:
            return i + 1
        n -= 1
        i -= k
    return first


def _negate(v: int) -> int:
    return INT64_MAX if v < -INT64_MAX else -v


def utf8_slice_row(r: bytes, start: int, stop: int, step: int) -> bytes:
    if step >= 1:
        if start >= 0:
            b = _advance(r, 0, start)
            if stop > start:
                e = _advance(r, b, stop - start)
            elif stop < 0:
                e = _advance_rev(r, b, _negate(stop))
            else:
                return b""
        else:
            b = _advance_rev(r, 0, -start)
            if stop > 0:
                e = _advance(r, 0, stop)
                if e <= b:
                    return b""
            elif stop < 0 and stop > start:
                e = _advance_rev(r, b, _negate(stop))
            else:
                return b""
        if step == 1:
            return r[b:e]
        out, i = bytearray(), b
        while i < e:
            k, cp = _decode(r, i)
            i += k
            out += _encode(cp)
            skips = step - 1
            while skips and i < e:
                i += _decode(r, i)[0]
                skips -= 1
        return bytes(out)
    b = (_advance(r, 0, start + 1) if start >= 0 else _advance_rev(r, 0, -start - 1)) - 1
    e = (_advance(r, 0, min(stop, INT64_MAX - 1) + 1) if stop >= 0 else _advance_rev(r, 0, _negate(stop) - 1)) - 1
    out, i = bytearray(), b
    while i > e:
        k, cp = _decode_rev(r, i)
        i -= k
        out += _encode(cp)
        skips = -step - 1
        while skips and i > e:
            i -= _decode_rev(r, i)[0]
            skips -= 1
    return bytes(out)


def binary_slice_row(r: bytes, start: int, stop: int, step: int) -> bytes:
    n = len(r)
    if n == 0:
        return b""
    if step >= 1:
        if start >= 0:
            b = min(start, n)
            if stop > start:
                e = min(b + (stop - start), n)
            elif stop < 0:
                e = max(n + stop, b)
            else:
                return b""
        else:
            b = max(n + start, 0)
            if stop > 0:
                e = min(stop, n)
                if e <= b:
                    return b""
            elif stop < 0 and stop > start:
                e = max(n + stop, b)
            else:
                return b""
        return r[b:e:step]
    b = (min(start + 1, n) if start >= 0 else max(n + start + 1, 0)) - 1
    e = (min(stop + 1, n) if stop >= 0 else max(n + stop + 1, 0)) - 1
    if b <= e:
        return b""
    return bytes(r[j] for j in range(b, e, step))


def _check_step(step):
    if step == 0:
        raise ValueError("Slice step cannot be zero")


def utf8_slice_codeunits(arr: pa.Array, start: int, stop: int = INT64_MAX, step: int = 1) -> pa.Array:
    """null rows are empty and never walked; raises InvalidUtf8 on a decode error in a valid row"""
    _check_step(step)
    return to_array([None if v is None else utf8_slice_row(v, start, stop, step) for v in values(arr)], arr.type)


def binary_slice(arr: pa.Array, start: int, stop: int = INT64_MAX, step: int = 1) -> pa.Array:
    _check_step(step)
    return pa.array([None if v is None else binary_slice_row(v, start, stop, step) for v in values(arr)], arr.type)


# ------------------------------------------------------------------------------------------------------------------
# the reference's output estimates (StringTransform::MaxCodeunits), in its wrapping int64 arithmetic
# ------------------------------------------------------------------------------------------------------------------
def _wrap(x: int) -> int:
    return (x + (1 << 63)) % (1 << 64) - (1 << 63)


def _cdiv(a: int, b: int) -> int:
    """C++ integer division (toward zero)"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def reference_max_codeunits(utf8: bool, n_rows: int, input_bytes: int, start: int, stop: int, step: int) -> int:
    """the byte count the reference allocates for a slice: below 0 it fails with "Negative buffer resize", below the
    output's real size it writes past its allocation"""
    if (start >= 0) != (stop >= 0):
        return input_bytes
    if utf8:
        stop = max(-input_bytes, min(stop, input_bytes))
        m = _cdiv(_wrap(_wrap(_wrap(stop - start) + step) - 1), step)
        return min(input_bytes, _wrap(_wrap(4 * n_rows) * max(0, m)))
    m = _cdiv(_wrap(_wrap(_wrap(stop - start) + step) - 1), step)
    return min(input_bytes, _wrap(n_rows * max(0, m)))


# ------------------------------------------------------------------------------------------------------------------
# binary_join_element_wise
# ------------------------------------------------------------------------------------------------------------------
NULL_HANDLING = ("emit_null", "skip", "replace")


def join_row(vals, sep, null_handling: str, replacement: bytes):
    """one row: vals a list of bytes / None, sep bytes / None; returns bytes or None"""
    if sep is None:
        return None
    if null_handling == "emit_null" and any(v is None for v in vals):
        return None
    kept = []
    for v in vals:
        if v is None:
            if null_handling == "skip":
                continue
            v = replacement
        kept.append(v)
    return sep.join(kept)


def binary_join_element_wise(operands, type_, null_handling="emit_null", null_replacement=b""):
    """operands: pa.Arrays and pa.Scalars (the separator last), at least one array"""
    n = next(len(o) for o in operands if isinstance(o, pa.Array))
    cols = []
    for o in operands:
        if isinstance(o, pa.Array):
            cols.append(values(o))
        else:
            cols.append([o.as_buffer().to_pybytes() if o.is_valid else None] * n)
    repl = null_replacement.encode() if isinstance(null_replacement, str) else null_replacement
    out = [join_row([c[i] for c in cols[:-1]], cols[-1][i], null_handling, repl) for i in range(n)]
    return to_array(out, type_)


def join_capacity_error(total: int) -> str:
    """BaseBinaryBuilder::ReserveData's text for an int32-offset output of `total` bytes"""
    return f"array cannot contain more than 2147483646 bytes, have {total}"


def reference_slice_defined(utf8: bool, n_rows: int, input_bytes: int, start: int, stop: int, step: int,
                            output_bytes: int) -> bool:
    """Whether pyarrow 24's slice is safe to call here: it either answers or fails cleanly.  It is not where its output
    estimate wraps to a size below the output (it writes past its buffer), where the estimate divides INT64_MIN by -1
    (SIGFPE), and, for binary_slice backwards, where start + 1 wraps at INT64_MAX or a step below -2^31 walks the
    pointer out of the address space."""
    if not utf8 and step < 0 and (start == INT64_MAX or step < -(1 << 31)):
        return False
    if (start >= 0) == (stop >= 0):
        s = max(-input_bytes, min(stop, input_bytes)) if utf8 else stop
        if step == -1 and _wrap(_wrap(_wrap(s - start) + step) - 1) == INT64_MIN:
            return False
    m = reference_max_codeunits(utf8, n_rows, input_bytes, start, stop, step)
    return m < 0 or m >= output_bytes
