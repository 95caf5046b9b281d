"""Device-side data model: Context (pool + stream), DeviceBuffer, DeviceArray.

DeviceArray is the device twin of arrow::ArrayData (cpp/src/arrow/array/data.h:80-420):
type, length, null_count, offset and the buffer list [validity, data, (data2)] -- the same
layout the reference uses (a list<T> is [validity, int32 offsets] plus its child in
`children`), but every buffer lives in HBM, allocated from the context pool
(the CudaMemoryManager stand-in, cpp/src/arrow/gpu/cuda_context.h:253).
pyarrow is used here only as the host container / type vocabulary (what libarrow is to
the C++ host); no pyarrow.compute kernel is ever called on the product path.
"""
from __future__ import annotations

import ctypes as C
import threading
from typing import Optional, Sequence

import numpy as np
import pyarrow as pa

from . import _cabi as cabi

_STATUS_EXC = {
    cabi.OUT_OF_MEMORY: pa.ArrowMemoryError,
    cabi.KEY_ERROR: pa.ArrowKeyError,
    cabi.TYPE_ERROR: pa.ArrowTypeError,
    cabi.INVALID: pa.ArrowInvalid,
    cabi.IO_ERROR: pa.ArrowIOError,
    cabi.CAPACITY_ERROR: pa.ArrowCapacityError,
    cabi.INDEX_ERROR: pa.ArrowIndexError,
    cabi.NOT_IMPLEMENTED: pa.ArrowNotImplementedError,
}


class CudaError(RuntimeError):
    pass


def check(status: int) -> None:
    if status == cabi.OK:
        return
    msg = cabi.last_error()
    exc = _STATUS_EXC.get(status)
    if exc is None:
        raise CudaError(msg)
    raise exc(msg)


# ---- arrow type -> physical B2 type id -------------------------------------------------
_NUMERIC = {
    pa.int8(): cabi.INT8, pa.uint8(): cabi.UINT8, pa.int16(): cabi.INT16, pa.uint16(): cabi.UINT16,
    pa.int32(): cabi.INT32, pa.uint32(): cabi.UINT32, pa.int64(): cabi.INT64, pa.uint64(): cabi.UINT64,
    pa.float32(): cabi.FLOAT, pa.float64(): cabi.DOUBLE,
}
_FROM_ID = {v: k for k, v in _NUMERIC.items()}
_FROM_ID[cabi.BOOL] = pa.bool_()
_WIDTH = {cabi.INT8: 1, cabi.UINT8: 1, cabi.INT16: 2, cabi.UINT16: 2, cabi.INT32: 4, cabi.UINT32: 4,
          cabi.INT64: 8, cabi.UINT64: 8, cabi.FLOAT: 4, cabi.DOUBLE: 8, cabi.HALF_FLOAT: 2}


def type_id(t: pa.DataType) -> int:
    """Physical type id handed to the C-ABI (logical temporal types use their storage)."""
    if t in _NUMERIC:
        return _NUMERIC[t]
    if pa.types.is_boolean(t):
        return cabi.BOOL
    if pa.types.is_date32(t) or pa.types.is_time32(t):
        return cabi.INT32
    if pa.types.is_date64(t) or pa.types.is_time64(t) or pa.types.is_timestamp(t) or pa.types.is_duration(t):
        return cabi.INT64
    if pa.types.is_float16(t):
        return cabi.HALF_FLOAT
    if pa.types.is_large_string(t):
        return cabi.LARGE_STRING
    if pa.types.is_large_binary(t):
        return cabi.LARGE_BINARY
    if pa.types.is_string(t):
        return cabi.STRING
    if pa.types.is_binary(t):
        return cabi.BINARY
    if pa.types.is_fixed_size_binary(t):
        return cabi.FIXED_SIZE_BINARY
    if pa.types.is_dictionary(t):
        return type_id(t.index_type)
    if pa.types.is_list(t):
        type_id(t.value_type)
        return cabi.LIST
    raise pa.ArrowNotImplementedError(f"arrow_b200: type {t} is not supported on device")


def arrow_type(tid: int) -> pa.DataType:
    return _FROM_ID[tid]


class Context:
    """One per device: owns the pool and the default stream (B2Context)."""

    _instances: dict = {}
    _lock = threading.Lock()

    def __init__(self, device: int = 0):
        self.lib = cabi.lib()
        h = C.c_void_p()
        check(self.lib.b2_context_create(device, C.byref(h)))
        self.handle = h
        self.device = device
        self.stream: Optional[int] = None  # None => the context's own stream

    @classmethod
    def get(cls, device: int = 0) -> "Context":
        with cls._lock:
            ctx = cls._instances.get(device)
            if ctx is None:
                ctx = cls._instances[device] = Context(device)
            return ctx

    # -- memory --
    def alloc(self, nbytes: int) -> "DeviceBuffer":
        p = C.c_void_p()
        check(self.lib.b2_alloc(self.handle, int(nbytes), C.byref(p)))
        return DeviceBuffer(self, p.value, int(nbytes), owned=True)

    def adopt(self, ptr: Optional[int], nbytes: int) -> Optional["DeviceBuffer"]:
        """Take ownership of a pool pointer returned by a kernel entry point."""
        if not ptr:
            return None
        return DeviceBuffer(self, ptr, nbytes, owned=True)

    def sync(self) -> None:
        check(self.lib.b2_sync(self.handle, self.stream))

    def pool_stats(self):
        a, b, c = C.c_int64(), C.c_int64(), C.c_int64()
        check(self.lib.b2_pool_stats(self.handle, C.byref(a), C.byref(b), C.byref(c)))
        return {"bytes_in_use": a.value, "bytes_reserved": b.value, "max_in_use": c.value}

    def trim(self) -> None:
        check(self.lib.b2_pool_trim(self.handle))

    def h2d(self, dst_ptr: int, src_ptr: int, n: int, stream: Optional[int] = None) -> None:
        """async host->device copy on `stream` (default: the context's current stream)"""
        check(self.lib.b2_memcpy_h2d(self.handle, dst_ptr, src_ptr, n, self.stream if stream is None else stream))

    def d2h(self, dst_ptr: int, src_ptr: int, n: int, stream: Optional[int] = None) -> None:
        check(self.lib.b2_memcpy_d2h(self.handle, dst_ptr, src_ptr, n, self.stream if stream is None else stream))


class NativeHandle:
    """Owner of one native object: `create(&handle)` makes it, and the entry point named `destroy` releases it at
    close(), at the end of a `with` block, or when the owner is garbage-collected."""

    def __init__(self, ctx: Context, destroy: str, create):
        self.ctx, self._destroy = ctx, destroy
        h = C.c_void_p()
        check(create(C.byref(h)))
        self.handle = h

    def close(self) -> None:
        if getattr(self, "handle", None):
            getattr(self.ctx.lib, self._destroy)(self.handle)
            self.handle = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc) -> None:
        self.close()


class DeviceBuffer:
    """A device allocation (arrow::cuda::CudaBuffer twin, cuda_memory.h:39)."""

    __slots__ = ("ctx", "ptr", "size", "owned", "keepalive", "__weakref__")

    def __init__(self, ctx: Context, ptr: int, size: int, owned: bool, keepalive=None):
        self.ctx, self.ptr, self.size, self.owned, self.keepalive = ctx, ptr, size, owned, keepalive

    def __del__(self):
        if getattr(self, "owned", False) and self.ptr:
            try:
                self.ctx.lib.b2_free(self.ctx.handle, self.ptr)
            except Exception:
                pass
            self.ptr = 0

    @classmethod
    def from_host(cls, ctx: Context, host: np.ndarray | pa.Buffer | bytes) -> "DeviceBuffer":
        if isinstance(host, pa.Buffer):
            addr, n = host.address, host.size
        else:
            host = np.ascontiguousarray(np.frombuffer(host, dtype=np.uint8) if isinstance(host, (bytes, bytearray)) else host)
            addr, n = host.ctypes.data, host.nbytes
        buf = ctx.alloc(max(n, 1))
        if n:
            ctx.h2d(buf.ptr, addr, n)
            ctx.sync()
        buf.size = n
        return buf

    def to_numpy(self, nbytes: Optional[int] = None) -> np.ndarray:
        n = self.size if nbytes is None else nbytes
        out = np.empty(n, dtype=np.uint8)
        if n:
            self.ctx.d2h(out.ctypes.data, self.ptr, n)
            self.ctx.sync()
        return out


class DeviceArray:
    """Device twin of arrow::ArrayData."""

    def __init__(self, ctx: Context, type: pa.DataType, length: int, null_count: int, offset: int,
                 buffers: Sequence[Optional[DeviceBuffer]], dictionary: Optional["DeviceArray"] = None,
                 children: Sequence["DeviceArray"] = ()):
        self.ctx, self.type, self.length = ctx, type, int(length)
        self.null_count, self.offset = int(null_count), int(offset)
        self.buffers = list(buffers)
        self.dictionary = dictionary
        self.children = list(children)

    def __len__(self):
        return self.length

    # -- construction ------------------------------------------------------------------
    @classmethod
    def from_arrow(cls, arr: pa.Array, ctx: Optional[Context] = None) -> "DeviceArray":
        ctx = ctx or Context.get()
        if isinstance(arr, pa.ChunkedArray):
            arr = arr.combine_chunks()
        dictionary = None
        if pa.types.is_list(arr.type):
            # buffers() lists the child's buffers too: keep [validity, offsets]; the child (whole, as the offsets index it)
            bufs = arr.buffers()[:2]
            dev = [None if b is None else DeviceBuffer.from_host(ctx, b) for b in bufs]
            return cls(ctx, arr.type, len(arr), arr.null_count, arr.offset, dev, children=[cls.from_arrow(arr.values, ctx)])
        if pa.types.is_dictionary(arr.type):
            dictionary = cls.from_arrow(arr.dictionary, ctx)
            bufs = arr.indices.buffers()
        else:
            type_id(arr.type)  # raises for unsupported types
            bufs = arr.buffers()
        dev = [None if b is None else DeviceBuffer.from_host(ctx, b) for b in bufs]
        return cls(ctx, arr.type, len(arr), arr.null_count, arr.offset, dev, dictionary)

    @classmethod
    def from_pointers(cls, ctx: Context, type: pa.DataType, length: int, data_ptr: int, *,
                      validity_ptr: int = 0, null_count: int = 0, offset: int = 0, data2_ptr: int = 0,
                      keepalive=None) -> "DeviceArray":
        """Zero-copy view of device memory owned by someone else (e.g. a torch tensor)."""
        bufs = [DeviceBuffer(ctx, validity_ptr, 0, False, keepalive) if validity_ptr else None,
                DeviceBuffer(ctx, data_ptr, 0, False, keepalive)]
        if data2_ptr:
            bufs.append(DeviceBuffer(ctx, data2_ptr, 0, False, keepalive))
        return cls(ctx, type, length, null_count if validity_ptr else 0, offset, bufs)

    @classmethod
    def _from_c(cls, ctx: Context, c: cabi.B2Array, type: pa.DataType,
                dictionary: Optional["DeviceArray"] = None) -> "DeviceArray":
        """Adopt the buffers a C-ABI entry point allocated for its output."""
        tid = c.type
        n = c.length
        if tid == cabi.BOOL:
            data_bytes = (n + 7) // 8
        elif tid in (cabi.STRING, cabi.BINARY):
            data_bytes = 4 * (n + 1)
        elif tid in (cabi.LARGE_STRING, cabi.LARGE_BINARY):
            data_bytes = 8 * (n + 1)
        elif tid == cabi.FIXED_SIZE_BINARY:
            data_bytes = n * c.byte_width
        else:
            data_bytes = n * _WIDTH[tid]
        bufs = [ctx.adopt(c.validity, (n + 7) // 8), ctx.adopt(c.data, data_bytes)]
        if tid in (cabi.STRING, cabi.BINARY, cabi.LARGE_STRING, cabi.LARGE_BINARY):
            b2 = ctx.adopt(c.data2, 0)
            bufs.append(b2)
        return cls(ctx, type, n, c.null_count, c.offset, bufs, dictionary)

    # -- views ---------------------------------------------------------------------------
    def slice(self, offset: int = 0, length: Optional[int] = None) -> "DeviceArray":
        """Zero-copy slice (ArrayData::Slice, array/data.cc:228-250): null_count becomes
        unknown unless it was 0 (or the slice is the whole array)."""
        offset = min(max(offset, 0), self.length)
        length = self.length - offset if length is None else min(length, self.length - offset)
        if self.null_count == 0:
            nc = 0
        elif offset == 0 and length == self.length:
            nc = self.null_count
        else:
            nc = -1
        return DeviceArray(self.ctx, self.type, length, nc, self.offset + offset, self.buffers, self.dictionary, self.children)

    def _c(self) -> cabi.B2Array:
        tid = type_id(self.type)
        c = cabi.B2Array()
        c.validity = self.buffers[0].ptr if self.buffers[0] is not None else None
        c.data = self.buffers[1].ptr if len(self.buffers) > 1 and self.buffers[1] is not None else None
        c.data2 = self.buffers[2].ptr if len(self.buffers) > 2 and self.buffers[2] is not None else None
        c.length, c.offset, c.null_count, c.type = self.length, self.offset, self.null_count, tid
        c.byte_width = self.type.byte_width if pa.types.is_fixed_size_binary(self.type) else 0
        if c.validity is None:
            c.null_count = 0
        return c

    # -- back to host ----------------------------------------------------------------------
    def to_arrow(self) -> pa.Array:
        tid = type_id(self.type)
        n, off = self.length, self.offset
        validity = None
        if self.buffers[0] is not None and self.null_count != 0:
            validity = pa.py_buffer(self.buffers[0].to_numpy((off + n + 7) // 8))
        if tid == cabi.LIST:
            offs = self.buffers[1].to_numpy(4 * (off + n + 1))
            return pa.Array.from_buffers(self.type, n, [validity, pa.py_buffer(offs)], null_count=self.null_count if validity else 0,
                                         offset=off, children=[self.children[0].to_arrow()])
        if tid == cabi.BOOL:
            data = pa.py_buffer(self.buffers[1].to_numpy((off + n + 7) // 8)) if n + off else pa.py_buffer(b"")
            bufs = [validity, data]
        elif tid in (cabi.STRING, cabi.BINARY, cabi.LARGE_STRING, cabi.LARGE_BINARY):
            ow = 8 if tid in (cabi.LARGE_STRING, cabi.LARGE_BINARY) else 4
            offs = self.buffers[1].to_numpy(ow * (off + n + 1)) if self.buffers[1] is not None else np.zeros(ow, np.uint8)
            o = offs.view(np.int64 if ow == 8 else np.int32)
            nbytes = int(o[off + n]) if len(o) else 0
            chars = self.buffers[2].to_numpy(nbytes) if (len(self.buffers) > 2 and self.buffers[2] is not None and nbytes) else np.zeros(0, np.uint8)
            bufs = [validity, pa.py_buffer(offs), pa.py_buffer(chars)]
        else:
            w = self.type.byte_width if tid == cabi.FIXED_SIZE_BINARY else _WIDTH[tid]
            data = self.buffers[1].to_numpy(w * (off + n)) if (self.buffers[1] is not None and n + off) else np.zeros(0, np.uint8)
            bufs = [validity, pa.py_buffer(data)]
        nc = self.null_count if validity is not None else 0
        if pa.types.is_dictionary(self.type):
            idx = pa.Array.from_buffers(self.type.index_type, n, bufs, null_count=nc, offset=off)
            return pa.DictionaryArray.from_arrays(idx, self.dictionary.to_arrow())
        return pa.Array.from_buffers(self.type, n, bufs, null_count=nc, offset=off)

    def __repr__(self):
        return f"<arrow_b200.DeviceArray {self.type} length={self.length} null_count={self.null_count} offset={self.offset}>"


class PinnedBuffer:
    """Page-locked host staging (arrow::cuda::CudaHostBuffer twin, cuda_memory.h:113)."""

    def __init__(self, nbytes: int):
        self.lib = cabi.lib()
        p = C.c_void_p()
        check(self.lib.b2_host_alloc(int(nbytes), C.byref(p)))
        self.ptr, self.size = p.value, int(nbytes)

    def numpy(self, dtype=np.uint8) -> np.ndarray:
        arr = (C.c_uint8 * self.size).from_address(self.ptr)
        return np.frombuffer(arr, dtype=dtype)

    def __del__(self):
        if getattr(self, "ptr", None):
            try:
                self.lib.b2_host_free(self.ptr)
            except Exception:
                pass
            self.ptr = None
