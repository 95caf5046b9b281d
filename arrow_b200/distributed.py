"""Multi-GPU execution of the two hot-path operators that need an exchange step.

One process per GPU.  Filter / Cast / arithmetic / compare / Take shard by row range with no
collective (bench.py does exactly that); hash-aggregate and SortIndices do one local pass, ONE
exchange and one local merge -- the shape of the reference's own per-thread scheme
(GroupByNode: per-thread Grouper + aggregators, then Merge by re-consuming uniques,
acero/groupby_aggregate_node.cc:211-218,255-298), with GPUs in place of threads:

  group_by_sum_count : local fused group-by -> partial groups (key, sum, count) -> the null-key
                       group is split off (it travels in the metadata) -> destination =
                       hash(key) % P (b2_hash_partition) -> stable partition (b2_sort_indices on
                       the destination id + b2_take, send counts from b2_bincount) -> exchange
                       -> the owner merges partials with Grouper + hash_sum (sum of sums, sum of
                       counts); a merged count of 0 makes the sum null (min_count = 1).
  sort_indices       : sample -> all-gather -> P-1 splitters -> destination = range id
                       (b2_range_partition) -> stable partition of (key, global row) ->
                       exchange -> local stable sort; nulls never move.
                       Result = rank-ordered concatenation of the value segments, then of the
                       null segments (AtEnd) -- identical to the single-GPU answer.

The exchange is ONE metadata all-gather (the P x P send counts + the null-group partials) followed
by ONE all-to-all-v of the partitioned columns:
  * B2CommExchange  -- the C-ABI path (b2_comm_*, csrc/comm.cu): every column's sends and receives
                       are issued inside a single NCCL group, i.e. one fused NCCL launch over
                       NVLink / NVSwitch, with no pack / unpack copies;
  * TorchExchange   -- torch.distributed (gloo for the CPU tests, nccl otherwise): the columns are
                       packed into one byte buffer and moved by one all_to_all_single.

All compute steps are C-ABI kernels (b2_*); torch appears only as tensor plumbing (zero-copy views,
slices, copies) and, in TorchExchange, as the transport.  The algorithms are written against a small
`ops` interface so the same code runs on device (DeviceOps) and, for the world_size-2 gloo tests, on
host arrays (tests/host_ops.py: the oracle + CPU tensors).
"""
from __future__ import annotations

import contextlib
import ctypes as C
from typing import List, Optional, Sequence

import numpy as np
import pyarrow as pa
import torch
import torch.distributed as dist

from . import _cabi as cabi
from .device import NativeHandle, check

_META_EXTRA = 3  # has_null, null_sum, null_count


# ------------------------------------------------------------------------------------------------
# transports
# ------------------------------------------------------------------------------------------------
def _pad8(nbytes: int) -> int:
    return (nbytes + 7) // 8 * 8


class TorchExchange:
    """torch.distributed transport: one all_gather_into_tensor for the metadata, one packed
    all_to_all_single for the data."""

    def __init__(self, group=None):
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.stats = {}

    def all_gather_i64(self, row: torch.Tensor) -> torch.Tensor:
        """row: int64[m] -> int64[world, m]"""
        out = torch.empty(self.world * row.numel(), dtype=torch.int64, device=row.device)
        if self.world == 1:
            out.copy_(row)
        else:
            dist.all_gather_into_tensor(out, row.contiguous(), group=self.group)
        return out.view(self.world, row.numel())

    def all_gather_bytes(self, buf: torch.Tensor) -> torch.Tensor:
        out = torch.empty(self.world * buf.numel(), dtype=torch.uint8, device=buf.device)
        if self.world == 1:
            out.copy_(buf)
        else:
            dist.all_gather_into_tensor(out, buf.contiguous(), group=self.group)
        return out.view(self.world, buf.numel())

    def all_to_all_columns(self, columns: Sequence[torch.Tensor], send_rows: Sequence[int], recv_rows: Sequence[int]):
        """columns: 1-D tensors, rows already grouped by destination (send_rows[d] rows for rank d).
        Returns the received columns, grouped by source rank in rank order."""
        widths = [c.element_size() for c in columns]
        dev = columns[0].device
        s_chunk = [sum(_pad8(w * n) for w in widths) for n in send_rows]
        r_chunk = [sum(_pad8(w * n) for w in widths) for n in recv_rows]
        send = torch.empty(sum(s_chunk), dtype=torch.uint8, device=dev)
        off, row0 = 0, 0
        for d, n in enumerate(send_rows):               # pack: chunk d = [col0 rows | col1 rows | ...]
            for c, w in zip(columns, widths):
                send[off: off + w * n] = c[row0: row0 + n].contiguous().view(torch.uint8)
                off += _pad8(w * n)
            row0 += n
        recv = torch.empty(sum(r_chunk), dtype=torch.uint8, device=dev)
        if self.world == 1:
            recv.copy_(send)
        else:
            dist.all_to_all_single(recv, send, output_split_sizes=r_chunk, input_split_sizes=s_chunk, group=self.group)
        total = sum(recv_rows)
        outs = [torch.empty(total, dtype=c.dtype, device=dev) for c in columns]
        off, row0 = 0, 0
        for n in recv_rows:                             # unpack
            for o, w in zip(outs, widths):
                o[row0: row0 + n] = recv[off: off + w * n].view(o.dtype)
                off += _pad8(w * n)
            row0 += n
        self.stats = {"alltoall_bytes": int(sum(s_chunk) - s_chunk[self.rank])}
        return outs


class B2CommExchange(NativeHandle):
    """C-ABI transport (b2_comm_*): NCCL through libarrow_b200.so, every column's sends/receives in one
    NCCL group.  The 128-byte unique id is distributed with torch.distributed (any backend)."""

    def __init__(self, ctx, group=None):
        self.check = check
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        ident = (C.c_uint8 * cabi.COMM_ID_BYTES)()
        if self.rank == 0:
            check(ctx.lib.b2_comm_unique_id(ident))
        box = [bytes(ident)]
        if self.world > 1:
            dist.broadcast_object_list(box, src=0, group=group)
        ident = (C.c_uint8 * cabi.COMM_ID_BYTES).from_buffer_copy(box[0])
        super().__init__(ctx, "b2_comm_destroy", lambda h: ctx.lib.b2_comm_init(ctx.handle, self.rank, self.world, ident, h))
        self.stats = {}

    def all_gather_i64(self, row: torch.Tensor) -> torch.Tensor:
        row = row.contiguous()
        out = torch.empty(self.world * row.numel(), dtype=torch.int64, device=row.device)
        self.check(self.ctx.lib.b2_comm_all_gather(self.handle, row.data_ptr(), out.data_ptr(), row.numel() * 8, self.ctx.stream))
        return out.view(self.world, row.numel())

    def all_gather_bytes(self, buf: torch.Tensor) -> torch.Tensor:
        buf = buf.contiguous()
        out = torch.empty(self.world * buf.numel(), dtype=torch.uint8, device=buf.device)
        self.check(self.ctx.lib.b2_comm_all_gather(self.handle, buf.data_ptr(), out.data_ptr(), buf.numel(), self.ctx.stream))
        return out.view(self.world, buf.numel())

    def all_to_all_columns(self, columns, send_rows, recv_rows):
        P = self.world
        I64 = C.c_int64 * P
        total = sum(recv_rows)
        outs = [torch.empty(total, dtype=c.dtype, device=c.device) for c in columns]
        s_off = np.concatenate([[0], np.cumsum(send_rows)[:-1]]).astype(np.int64)
        r_off = np.concatenate([[0], np.cumsum(recv_rows)[:-1]]).astype(np.int64)
        lib = self.ctx.lib
        self.check(lib.b2_comm_group_start(self.handle))
        sent = 0
        for c, o in zip(columns, outs):
            w = c.element_size()
            c = c.contiguous()
            self.check(lib.b2_comm_all_to_all_v(
                self.handle, c.data_ptr(), I64(*[int(x) * w for x in s_off]), I64(*[int(n) * w for n in send_rows]),
                o.data_ptr(), I64(*[int(x) * w for x in r_off]), I64(*[int(n) * w for n in recv_rows]), self.ctx.stream))
            sent += w * (sum(send_rows) - send_rows[self.rank])
        self.check(lib.b2_comm_group_end(self.handle))
        self.stats = {"alltoall_bytes": int(sent)}
        return outs


# ------------------------------------------------------------------------------------------------
# the two distributed operators (backend agnostic)
# ------------------------------------------------------------------------------------------------
def partial_sum_bits(sums: pa.Array) -> int:
    """the single partial sum in `sums` (host int64 / uint64 / float64) as the int64 with the same 64 bits: how the
    null-key group's sum travels in the int64 metadata row (a uint64 sum >= 2^63 does not fit an int64 by value).
    A null sum (count 0) travels as 0."""
    v = sums[0].as_py() if sums[0].is_valid else 0
    return int(np.array([v], dtype=sums.type.to_pandas_dtype()).view(np.int64)[0])


def group_by_sum_count(keys, values, ops, xchg=None, expected_groups: int = 0):
    """Distributed `group_by(key).aggregate(sum, count)` over row-range shards.
    Returns this rank's owned groups: (keys, sums, counts) -- disjoint across ranks, union = all.
    With world == 1 this is exactly the local fused group-by."""
    xchg = xchg or TorchExchange()
    P, rank = xchg.world, xchg.rank
    with ops.stream_guard():
        k, s, c = ops.local_group_by(keys, values, expected_groups)   # partial groups of this shard
        if P == 1:
            return k, s, c
        k, s, c, null_info = ops.split_null_group(k, s, c)             # null key: [has, sum, count]
        dest = ops.hash_partition(k, P)                                # owner of every partial group
        order, send_rows = ops.partition_plan(dest, P)
        k, s, c = ops.take(k, order), ops.take(s, order), ops.take(c, order)
        meta = xchg.all_gather_i64(ops.meta_tensor(list(send_rows) + list(null_info)))
        meta_h = meta.cpu().numpy()
        recv_rows = [int(meta_h[src, rank]) for src in range(P)]
        t0 = ops.mark()
        rk, rs, rc = xchg.all_to_all_columns([ops.raw_tensor(k), ops.raw_tensor(s), ops.raw_tensor(c)], send_rows, recv_rows)
        ops.note_exchange(t0, xchg)
        nulls = np.ascontiguousarray(meta_h[:, P:])
        null_group = None
        if rank == 0 and nulls[:, 0].any():
            bits = np.ascontiguousarray(nulls[:, 1])
            if pa.types.is_floating(ops.type_of(s)):     # partial sums travel as raw bits
                total = np.array([bits.view(np.float64).sum()], dtype=np.float64).view(np.int64)[0]
            else:
                total = bits.view(np.uint64).sum(dtype=np.uint64).astype(np.int64)
            null_group = (int(total), int(nulls[:, 2].sum()))
        return ops.merge_partials(rk, rs, rc, ops.type_of(k), ops.type_of(s), null_group)


def sort_indices(values, ops, xchg=None, samples_per_rank: int = 4096, return_keys: bool = False):
    """Distributed stable `sort_indices(values, ascending, nulls at end)` over row-range shards.
    Returns (sorted_global_indices_segment, null_global_indices_segment) for this rank (torch tensors);
    the rank-ordered concatenation of the value segments followed by that of the null segments is the
    single-process answer."""
    xchg = xchg or TorchExchange()
    P, rank = xchg.world, xchg.rank
    with ops.stream_guard():
        n_local = ops.length(values)
        if P == 1:
            order = ops.stable_sort_indices(values)
            n_valid = n_local - ops.null_count(values)
            t = ops.raw_tensor(order)
            if return_keys:   # the keys in sorted order (verification aid for bench.py / tests)
                return t[:n_valid], t[n_valid:], ops.raw_tensor(ops.take(values, ops.slice(order, 0, n_valid)))
            return t[:n_valid], t[n_valid:]
        # one all-gather carries the shard lengths and a sample of the valid rows
        sample = ops.sample_valid(values, samples_per_rank)            # typed tensor, <= samples_per_rank
        width = sample.element_size()
        buf = torch.zeros(16 + samples_per_rank * width, dtype=torch.uint8, device=sample.device)
        head = torch.tensor([n_local, sample.numel()], dtype=torch.int64).view(torch.uint8)
        buf[:16] = head.to(buf.device)
        buf[16: 16 + sample.numel() * width] = sample.contiguous().view(torch.uint8)
        gathered = xchg.all_gather_bytes(buf)
        heads = gathered[:, :16].cpu().contiguous().view(torch.int64).view(P, 2).numpy()
        row0 = int(heads[:rank, 0].sum())
        parts = [gathered[r, 16: 16 + int(heads[r, 1]) * width].contiguous().view(sample.dtype) for r in range(P)]
        splitters = ops.pick_splitters(torch.cat(parts), P, ops.type_of(values))
        # P - 1 splitters, or none when no rank holds a valid row: then there is one value bin and the null bin
        # follows it, so the bins are counted from the splitters, never from P
        bins = ops.length(splitters) + 1
        n_total = int(heads[:, 0].sum())
        narrow = n_total < (1 << 32)        # global row numbers fit 32 bits: they travel as uint32 and ride along the
        if narrow:                          # owner's radix passes as the sort payload (no gather afterwards)
            # one stable split of (value, global row) by range id: count -> scan -> scatter (b2_range_split)
            valid_all, rows_all, counts = ops.range_split(values, splitters, row0)
            n_valid = sum(counts[:bins])
            valid_part, gsend = ops.slice(valid_all, 0, n_valid), ops.slice(rows_all, 0, n_valid)
            null_idx = ops.raw_tensor(ops.slice(rows_all, n_valid, n_local - n_valid))
            null_idx = null_idx.to(torch.int64) & 0xFFFFFFFF
        else:
            dest = ops.range_partition(values, splitters)              # nulls get id bins (= #splitters + 1)
            order, counts = ops.partition_plan(dest, bins + 1)
            n_valid = sum(counts[:bins])
            gidx = ops.add_offset(order, row0)                         # global row numbers, partition order
            valid_part = ops.take(values, ops.slice(order, 0, n_valid))
            gsend = ops.slice(gidx, 0, n_valid)
            null_idx = ops.raw_tensor(ops.slice(gidx, n_valid, n_local - n_valid))
        send_rows = list(counts[:bins]) + [0] * (P - bins)
        meta = xchg.all_gather_i64(ops.meta_tensor(send_rows)).cpu().numpy()
        recv_rows = [int(meta[src, rank]) for src in range(P)]
        t0 = ops.mark()
        rk, ri = xchg.all_to_all_columns([ops.raw_tensor(valid_part), ops.raw_tensor(gsend)], send_rows, recv_rows)
        ops.note_exchange(t0, xchg)
        # received rows are grouped by source rank (ascending) and ascending global row inside each
        # group, so a STABLE local sort keeps ties in global row order
        rk_arr = ops.from_raw_tensor(rk, ops.type_of(values))
        if narrow and not return_keys:
            return ops.raw_tensor(ops.sort_payload(rk_arr, ops.from_raw_tensor(ri, pa.uint32()))), null_idx
        local = ops.stable_sort_indices(rk_arr)
        seg = ops.raw_tensor(ops.take(ops.from_raw_tensor(ri, pa.uint32() if narrow else pa.uint64()), local))
        if narrow:
            seg = seg.to(torch.int64) & 0xFFFFFFFF if seg.dtype != torch.int64 else seg
        if return_keys:
            return seg, null_idx, ops.raw_tensor(ops.take(rk_arr, local))
        return seg, null_idx


# ------------------------------------------------------------------------------------------------
# device backend
# ------------------------------------------------------------------------------------------------
class _CudaView:
    """__cuda_array_interface__ adapter: lets torch view a pool buffer without a copy."""

    def __init__(self, ptr: int, n: int, typestr: str, owner):
        self.owner = owner
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


_TYPESTR = {pa.int8(): "|i1", pa.uint8(): "|u1", pa.int16(): "<i2", pa.uint16(): "<u2", pa.int32(): "<i4", pa.uint32(): "<u4",
            pa.int64(): "<i8", pa.uint64(): "<u8", pa.float32(): "<f4", pa.float64(): "<f8"}
_TORCH = {pa.int8(): torch.int8, pa.uint8(): torch.uint8, pa.int16(): torch.int16, pa.int32(): torch.int32, pa.int64(): torch.int64,
          pa.float32(): torch.float32, pa.float64(): torch.float64, pa.uint16(): torch.int16, pa.uint32(): torch.int32,
          pa.uint64(): torch.int64}


class DeviceOps:
    """ops interface over DeviceArray + the C-ABI kernels (everything stays in HBM).

    Stream discipline: C-ABI calls run on ctx.stream and torch ops / collectives on torch's current
    stream, so the two must be the same stream.  If the context has no explicit stream yet, DeviceOps
    creates a torch side stream, installs it as ctx.stream and runs every operator under it
    (stream_guard); a caller that already set ctx.stream (bench.py) must have made it torch's current
    stream."""

    def __init__(self, ctx=None):
        from . import compute as bc
        from .device import Context, DeviceArray
        self.bc, self.DeviceArray = bc, DeviceArray
        self.ctx = ctx or Context.get(torch.cuda.current_device())
        self._own_stream = None
        if not self.ctx.stream:
            self._own_stream = torch.cuda.Stream()
            assert self._own_stream.cuda_stream != 0
            self.ctx.stream = self._own_stream.cuda_stream
        self.exchange_ms: List[float] = []
        self.exchange_bytes: List[int] = []

    @contextlib.contextmanager
    def stream_guard(self):
        if self._own_stream is None:
            yield
            return
        outer = torch.cuda.current_stream()
        self._own_stream.wait_stream(outer)       # inputs produced on the caller's stream
        with torch.cuda.stream(self._own_stream):
            yield
        outer.wait_stream(self._own_stream)       # results consumed on the caller's stream

    # -- array <-> tensor (zero copy) --
    def _tensor(self, arr, t=None):
        t = t or arr.type
        n = arr.length
        if n == 0:
            return torch.empty(0, dtype=_TORCH[t], device="cuda")
        width = t.bit_width // 8
        view = _CudaView(arr.buffers[1].ptr + arr.offset * width, n, _TYPESTR[t], arr)
        out = torch.as_tensor(view, device="cuda")
        return out.view(_TORCH[t]) if out.dtype != _TORCH[t] else out

    def _array(self, tensor, t, validity=None, null_count=0):
        tensor = tensor.contiguous()
        return self.DeviceArray.from_pointers(self.ctx, t, tensor.numel(), tensor.data_ptr() if tensor.numel() else 0,
                                              validity_ptr=validity.data_ptr() if validity is not None else 0,
                                              null_count=null_count, keepalive=(tensor, validity))

    def type_of(self, arr):
        return arr.type

    def length(self, arr):
        return arr.length

    def null_count(self, arr):
        if arr.null_count < 0:
            return arr.length - self.bc.count(arr).as_py()
        return arr.null_count

    def raw_tensor(self, arr):
        return self._tensor(arr)

    def from_raw_tensor(self, t, typ):
        return self._array(t, typ)

    def meta_tensor(self, ints):
        return torch.tensor([int(x) for x in ints], dtype=torch.int64).to("cuda", non_blocking=False)

    def mark(self):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e

    def note_exchange(self, t0, xchg):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self._pending = (t0, e, xchg.stats.get("alltoall_bytes", 0))

    def exchange_stats(self):
        """(ms, bytes sent to peers) of the last data exchange; synchronises."""
        p = getattr(self, "_pending", None)
        if p is None:
            return 0.0, 0
        p[1].synchronize()
        return p[0].elapsed_time(p[1]), p[2]

    # -- kernels --
    def local_group_by(self, keys, values, expected_groups=0):
        g = self.bc.GroupBySumCount(keys.type, values.type, expected_groups=expected_groups, ctx=self.ctx)
        g.consume(keys, values)
        return g.finalize()

    def split_null_group(self, k, s, c):
        if k.null_count == 0 or k.buffers[0] is None:
            return k, s, c, (0, 0, 0)
        bc = self.bc
        pos = bc.take_indices_from_filter(bc.is_null(k))           # the (single) null-key group
        ns, nc = bc.take(s, pos).to_arrow(), bc.take(c, pos).to_arrow()
        keep = bc.is_valid(k)
        return bc.filter(k, keep), bc.filter(s, keep), bc.filter(c, keep), (1, partial_sum_bits(ns), nc[0].as_py())

    def hash_partition(self, keys, n_parts):
        return self.bc._call(self.ctx, "b2_hash_partition", pa.uint32(), C.byref(keys._c()), int(n_parts))

    def range_partition(self, values, splitters):
        return self.bc._call(self.ctx, "b2_range_partition", pa.uint32(), C.byref(values._c()), C.byref(splitters._c()), 0)

    def partition_plan(self, dest, n_bins):
        """stable grouping of the rows by destination id: (gather order, rows per destination)"""
        counts = (C.c_int64 * n_bins)()
        cd = dest._c()
        check(self.ctx.lib.b2_bincount(self.ctx.handle, C.byref(cd), n_bins, counts, self.ctx.stream))
        return self.bc.array_sort_indices(dest), [int(x) for x in counts]

    def stable_sort_indices(self, arr):
        return self.bc.array_sort_indices(arr)

    def take(self, arr, idx):
        return self.bc.take(arr, idx)

    def slice(self, arr, off, length):
        return arr.slice(off, length)

    def add_offset(self, idx_arr, off):
        return self.bc.add(idx_arr, pa.scalar(int(off), pa.uint64()))

    def range_split(self, values, splitters, row0):
        """(values regrouped by destination, uint32 global rows regrouped the same way, rows per destination [+ nulls last])"""
        n_bins = splitters.length + 2
        counts = (C.c_int64 * n_bins)()
        cv, cs, ov, orows = values._c(), splitters._c(), cabi.B2Array(), cabi.B2Array()
        check(self.ctx.lib.b2_range_split(self.ctx.handle, C.byref(cv), C.byref(cs), 0, int(row0), C.byref(ov), C.byref(orows), counts,
                                          self.ctx.stream))
        return (self.DeviceArray._from_c(self.ctx, ov, values.type), self.DeviceArray._from_c(self.ctx, orows, pa.uint32()),
                [int(x) for x in counts])

    def to_uint32(self, arr):
        return self.bc.cast(arr, pa.uint32(), safe=False)

    def sort_payload(self, arr, payload):
        return self.bc.sort_payload(arr, payload)

    def sample_valid(self, values, k):
        """<= k rows evenly spaced among the valid rows, as a typed tensor: a shard with a valid row always
        contributes to the splitters, wherever its valid rows lie"""
        if self.null_count(values):
            values = self.bc.filter(values, self.bc.is_valid(values))
        n = values.length
        if n == 0:
            return torch.empty(0, dtype=_TORCH[values.type], device="cuda")
        step = max(1, -(-n // k))
        pos = torch.arange(0, n, step, dtype=torch.int64, device="cuda")
        return self._tensor(self.bc.take(values, self._array(pos, pa.int64()))).clone()

    def pick_splitters(self, gathered, world, typ):
        if gathered.numel() == 0 or world == 1:
            return self._array(gathered[:0], typ)
        g = self._array(gathered, typ)
        g = self.bc.take(g, self.bc.array_sort_indices(g))
        pos = (torch.arange(1, world, dtype=torch.int64, device="cuda") * gathered.numel()) // world
        return self.bc.take(g, self._array(pos.clamp(max=gathered.numel() - 1), pa.int64()))

    def merge_partials(self, rk, rs, rc, keys_type, sum_type, null_group):
        """owner-side merge = GroupByNode::Merge: re-consume the uniques, add the partial states"""
        bc = self.bc
        n = rk.numel()
        validity, nulls = None, 0
        if null_group is not None:   # rank 0 owns the null key: append it as one more partial with a cleared validity bit
            rk = torch.cat([rk, torch.zeros(1, dtype=rk.dtype, device=rk.device)])
            rs = torch.cat([rs, torch.tensor([null_group[0]], dtype=torch.int64, device=rs.device).view(rs.dtype)])
            rc = torch.cat([rc, torch.tensor([null_group[1]], dtype=rc.dtype, device=rc.device)])
            validity = torch.full(((n + 1 + 7) // 8 + 8,), 0xFF, dtype=torch.uint8, device="cuda")
            validity[n >> 3] = 0xFF & ~(1 << (n & 7))
            nulls = 1
        keys = self._array(rk, keys_type, validity, nulls)
        # one kernel: every partial finds / claims its key's slot and adds its sum and count (b2_groupby_sumcount_merge)
        value_type = {pa.int64(): pa.int64(), pa.uint64(): pa.uint64(), pa.float64(): pa.float64()}[sum_type]
        g = bc.GroupBySumCount(keys_type, value_type, expected_groups=max(1, n), ctx=self.ctx)
        g.merge(keys, self._array(rs, sum_type), self._array(rc, pa.int64()))
        return g.finalize()
