"""String sort-key inputs shared by the CPU oracle test and the GPU test of sorting by utf8 / binary keys: random bytes
(NUL and bytes >= 0x80 included) at sizes around the 4096-row tiles, heavy ties and prefixes, strings ending at the
7-byte chunk boundaries, degenerate columns, and the long-shared-prefix inputs that bound the refinement rounds."""
import numpy as np
import pyarrow as pa

from tests.util import SEED

STRING_TYPES = [pa.string(), pa.binary(), pa.large_string(), pa.large_binary()]


def strings_array(t, vals, null_p=0.0, seed=SEED, offset=0):
    """pa array of type t from a list of bytes; rows turn null with probability null_p; `offset` leading rows are added
    and sliced away, so offsets[offset] != 0 and the validity starts mid-byte."""
    rng = np.random.default_rng(seed)
    pad = [bytes(rng.integers(0, 256, int(rng.integers(0, 12)), dtype=np.uint8)) for _ in range(offset)]
    vals = pad + list(vals)
    mask = rng.random(len(vals)) < null_p if null_p > 0 else None
    if pa.types.is_string(t) or pa.types.is_large_string(t):  # any bytes: build as binary, reinterpret the buffers
        arr = pa.array(vals, pa.large_binary() if pa.types.is_large_string(t) else pa.binary(), mask=mask)
        arr = pa.Array.from_buffers(t, len(arr), arr.buffers(), null_count=arr.null_count)
    else:
        arr = pa.array(vals, t, mask=mask)
    return arr.slice(offset) if offset else arr


def random_bytes(n, seed, max_len=24, alphabet=None):
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, max_len, n, endpoint=True)
    if alphabet is None:
        data = rng.integers(0, 256, int(lens.sum()), dtype=np.uint8)
    else:
        data = np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), int(lens.sum()))]
    offs = np.concatenate([[0], np.cumsum(lens)])
    out = [data[offs[i]:offs[i + 1]].tobytes() for i in range(n)]
    # duplicates: every 7th row repeats an earlier one
    for i in range(7, n, 7):
        out[i] = out[int(rng.integers(0, i))]
    return out


def chunk_boundary_strings(seed):
    """prefixes of one string at every length around the 7-byte chunks (6, 7, 8, 14, 15 ...), with NUL-extended variants"""
    rng = np.random.default_rng(seed)
    base = bytes(rng.integers(1, 256, 24, dtype=np.uint8))
    vals = [base[:k] for k in range(0, 25)] + [base[:k] + b"\x00" for k in (5, 6, 7, 13, 14, 15)]
    vals = vals * 5
    return [vals[i] for i in rng.permutation(len(vals))]


def cases(n_big=(0, 1, 2, 4095, 4097, 70_000)):
    """(name, list of bytes, null_p) of the functional inputs"""
    out = [(f"random n={n}", random_bytes(n, SEED + n), 0.1) for n in n_big]
    out.append(("two letters 0-20", random_bytes(5000, SEED + 1, max_len=20, alphabet=b"ab"), 0.05))
    out.append(("nul and high bytes", random_bytes(3000, SEED + 2, max_len=10, alphabet=b"\x00\x01\x7f\x80\xff"), 0.1))
    out.append(("chunk boundaries", chunk_boundary_strings(SEED + 3), 0.0))
    out.append(("all identical", [b"identical value, longer than a chunk"] * 5000, 0.0))
    out.append(("all null", [b"x"] * 3000, 1.0))
    out.append(("issue example", [b"\x80", b"a", b"", None, b"a\x00", b"a", b"\xff\x01"], 0.0))
    return out


def shared_prefix_strings(seed, n=1000, prefix_len=64 << 10):
    """n strings sharing one 64 KiB prefix, then a short random tail (some tails empty, some repeated)"""
    rng = np.random.default_rng(seed)
    prefix = bytes(rng.integers(0, 256, prefix_len, dtype=np.uint8))
    tails = random_bytes(n, seed + 1, max_len=6)
    return [prefix + t for t in tails] + [prefix[:prefix_len // 2], b"", b"short"]


def two_long_identical(seed, n_short=2000, long_len=1 << 20):
    """two identical 1 MiB strings among short ones (and one that differs from them in its last byte)"""
    rng = np.random.default_rng(seed)
    big = bytes(rng.integers(0, 256, long_len, dtype=np.uint8))
    vals = random_bytes(n_short, seed + 1, max_len=16)
    vals[17] = big
    vals[1234] = big
    vals[999] = big[:-1] + bytes([(big[-1] + 1) % 256])
    return vals
