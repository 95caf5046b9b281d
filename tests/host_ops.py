"""Host stand-in for arrow_b200.distributed.DeviceOps, used only by the world_size-2 gloo tests:
the same `ops` interface over pyarrow host arrays, the oracle and CPU tensors, so the exchange
logic (partition, splits, all-to-all, merge, ordering) is exercised without a GPU."""
import contextlib

import numpy as np
import pyarrow as pa
import torch

from arrow_b200.distributed import partial_sum_bits
from oracle import arrow_oracle as ora

_MIX = (0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53)


def hash64(k: np.ndarray) -> np.ndarray:
    """murmur3 fmix64 -- must equal hash64() in arrow_b200/csrc/hash_table.cuh"""
    k = k.astype(np.uint64)
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33)
        k *= np.uint64(_MIX[0])
        k ^= k >> np.uint64(33)
        k *= np.uint64(_MIX[1])
        k ^= k >> np.uint64(33)
    return k


class HostOps:
    """same method set as arrow_b200.distributed.DeviceOps"""

    @contextlib.contextmanager
    def stream_guard(self):
        yield

    def type_of(self, arr):
        return arr.type

    def length(self, arr):
        return len(arr)

    def null_count(self, arr):
        return arr.null_count

    def raw_tensor(self, arr):
        v = ora.values(arr)
        if v.dtype in (np.uint16, np.uint32, np.uint64):
            v = v.view({2: np.int16, 4: np.int32, 8: np.int64}[v.dtype.itemsize])
        t = torch.from_numpy(v.copy())
        return t if len(v) else torch.empty(0, dtype=t.dtype)   # an empty numpy array maps to stride 0, which .view(dtype) refuses

    def from_raw_tensor(self, t, typ):
        return pa.array(t.numpy().view(ora.np_dtype(typ)), typ)

    def meta_tensor(self, ints):
        return torch.tensor([int(x) for x in ints], dtype=torch.int64)

    def mark(self):
        return None

    def note_exchange(self, t0, xchg):
        pass

    def local_group_by(self, keys, values, expected_groups=0):
        uniq, (s, c) = ora.group_by([keys], [("hash_sum", values, None), ("hash_count", values, None)])
        return uniq[0], s, c

    def split_null_group(self, k, s, c):
        if k.null_count == 0:
            return k, s, c, (0, 0, 0)
        valid = ora.validity(k)
        pos = int(np.flatnonzero(~valid)[0])
        keep = pa.array(valid)
        return ora.filter(k, keep), ora.filter(s, keep), ora.filter(c, keep), (1, partial_sum_bits(s.slice(pos, 1)), c[pos].as_py())

    def hash_partition(self, keys, n_parts):
        v, valid = ora.values(keys), ora.validity(keys)
        raw = v.view(f"u{v.dtype.itemsize}").astype(np.uint64)     # the key's bits, zero-extended (load_key_bits)
        ids = (hash64(raw) % np.uint64(n_parts)).astype(np.uint32)
        return pa.array(np.where(valid, ids, 0).astype(np.uint32))

    def range_partition(self, values, splitters):
        v, valid = ora.values(values), ora.validity(values)
        sp = ora.values(splitters)
        ids = np.searchsorted(sp, v, side="right").astype(np.uint32)
        return pa.array(np.where(valid, ids, len(sp) + 1).astype(np.uint32))

    def partition_plan(self, dest, n_bins):
        counts = [int(x) for x in np.bincount(ora.values(dest), minlength=n_bins)[:n_bins]]
        return ora.sort_indices(dest), counts

    def stable_sort_indices(self, arr):
        return ora.sort_indices(arr)

    def take(self, arr, idx):
        return ora.take(arr, idx)

    def slice(self, arr, off, length):
        return arr.slice(off, length)

    def add_offset(self, idx_arr, off):
        return pa.array(ora.values(idx_arr).astype(np.uint64) + np.uint64(off), pa.uint64())

    def range_split(self, values, splitters, row0):
        v, valid = ora.values(values), ora.validity(values)
        sp = ora.values(splitters)
        ids = np.where(valid, np.searchsorted(sp, v, side="right"), len(sp) + 1)
        order = np.argsort(ids, kind="stable")
        counts = [int(x) for x in np.bincount(ids, minlength=len(sp) + 2)]
        return (ora.make_array(values.type, v[order]), pa.array((order + row0).astype(np.uint32), pa.uint32()), counts)

    def to_uint32(self, arr):
        return pa.array(ora.values(arr).astype(np.uint32), pa.uint32())

    def sort_payload(self, arr, payload):
        return pa.array(ora.values(ora.take(payload, ora.sort_indices(arr))).astype(np.uint64), pa.uint64())

    def sample_valid(self, values, k):
        s = values.drop_null()
        step = max(1, -(-len(s) // k))
        return self.raw_tensor(s.take(pa.array(np.arange(0, len(s), step))))

    def pick_splitters(self, gathered, world, typ):
        g, _ = torch.sort(gathered)
        if g.numel() == 0 or world == 1:
            return pa.array(g[:0].numpy(), typ)
        pos = (torch.arange(1, world) * g.numel()) // world
        return pa.array(g[pos.clamp(max=g.numel() - 1)].numpy(), typ)

    def merge_partials(self, rk, rs, rc, keys_type, sum_type, null_group):
        kv, sv, cv = rk.numpy(), rs.numpy().view(ora.np_dtype(sum_type)), rc.numpy()
        mask = np.zeros(len(kv), dtype=bool)
        if null_group is not None:
            kv = np.concatenate([kv, np.zeros(1, kv.dtype)])
            sv = np.concatenate([sv, np.array([null_group[0]], dtype=np.int64).view(sv.dtype)])
            cv = np.concatenate([cv, np.array([null_group[1]], dtype=cv.dtype)])
            mask = np.concatenate([mask, [True]])
        keys = pa.array(kv.view(ora.np_dtype(keys_type)), keys_type, mask=mask)
        uniq, (s, c) = ora.group_by([keys], [("hash_sum", pa.array(sv, sum_type), None),
                                              ("hash_sum", pa.array(cv, pa.int64()), None)])
        cnt = ora.values(c)
        s = ora.make_array(sum_type, ora.values(s), cnt != 0)
        return uniq[0], s, c
