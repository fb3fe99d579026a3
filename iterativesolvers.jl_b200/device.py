"""Context (device + stream [+ NCCL communicator]) and raw device arrays."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import check, lib

_DT = {np.dtype(np.float64): _lib.F64, np.dtype(np.float32): _lib.F32,
       np.dtype(np.complex128): _lib.CF64, np.dtype(np.complex64): _lib.CF32}
_DT_OF_CODE = {code: dt for dt, code in _DT.items()}


def dtype_code(dt) -> int:
    dt = np.dtype(dt)
    if dt not in _DT:
        raise TypeError(f"unsupported element type {dt}: the device path handles Float64, Float32, ComplexF64 and "
                        "ComplexF32")
    return _DT[dt]


def dtype_of_code(code: int) -> np.dtype:
    """the numpy dtype of a B200_* element type code"""
    return _DT_OF_CODE[int(code)]


class Context:
    """One per (process, GPU).  `Context.distributed()` builds the NCCL communicator from an
    initialised torch.distributed process group (one process per GPU)."""

    def __init__(self, device: int = 0, _handle=None):
        self._h = C.c_void_p()
        if _handle is not None:
            self._h = _handle
        else:
            check(lib().b200_ctx_create(device, C.byref(self._h)))
        dev, rank, world, sms = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        check(lib().b200_ctx_info(self._h, C.byref(dev), C.byref(rank), C.byref(world), C.byref(sms)))
        self.device, self.rank, self.world, self.sm_count = dev.value, rank.value, world.value, sms.value

    @classmethod
    def distributed(cls, device: int | None = None):
        import torch
        import torch.distributed as dist
        rank, world = dist.get_rank(), dist.get_world_size()
        if device is None:
            device = rank % max(torch.cuda.device_count(), 1)
        uid = torch.zeros(128, dtype=torch.uint8)
        if rank == 0:
            buf = (C.c_ubyte * 128)()
            check(lib().b200_nccl_unique_id(buf))
            uid = torch.tensor(list(buf), dtype=torch.uint8)
        if dist.get_backend() == "nccl":
            uid = uid.cuda(device)
        dist.broadcast(uid, src=0)
        raw = bytes(uid.cpu().tolist())
        h = C.c_void_p()
        check(lib().b200_ctx_create_dist(device, rank, world, raw, C.byref(h)))
        return cls(_handle=h)

    def set_option(self, name: str, value: int):
        """b200_ctx_set_option (include/b200krylov.h lists the options), e.g. set_option("rowptr64", 1)."""
        check(lib().b200_ctx_set_option(self._h, name.encode(), int(value)))

    def get_option(self, name: str) -> int:
        v = C.c_int64()
        check(lib().b200_ctx_get_option(self._h, name.encode(), C.byref(v)))
        return int(v.value)

    def use_stream(self, cuda_stream: int):
        check(lib().b200_ctx_set_stream(self._h, C.c_void_p(cuda_stream)))

    def sync(self):
        check(lib().b200_ctx_sync(self._h))

    def barrier(self):
        check(lib().b200_ctx_barrier(self._h))

    def launch_count(self) -> int:
        return int(lib().b200_ctx_launch_count(self._h))

    def timer_start(self):
        check(lib().b200_ctx_timer_start(self._h))

    def timer_stop(self) -> float:
        ms = C.c_float()
        check(lib().b200_ctx_timer_stop(self._h, C.byref(ms)))
        return float(ms.value)

    def allreduce(self, values, op="sum"):
        arr = (C.c_double * len(values))(*values)
        check(lib().b200_ctx_allreduce_f64(self._h, arr, len(values), 1 if op == "max" else 0))
        return list(arr)

    def close(self):
        if self._h:
            lib().b200_ctx_destroy(self._h)
            self._h = C.c_void_p()


_default = None


def default_context() -> Context:
    global _default
    if _default is None:
        _default = Context(0)
    return _default


class DeviceArray:
    """A dense device vector / column-major matrix owned by the library allocator
    (`similar`, `copyto!`).  shape = (n,) or (n, k) with leading dimension n."""

    def __init__(self, ctx: Context, shape, dtype=np.float64):
        self.ctx = ctx
        self.shape = (shape,) if np.isscalar(shape) else tuple(int(s) for s in shape)
        self.dtype = np.dtype(dtype)
        self.code = dtype_code(dtype)
        self.nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        self._p = C.c_void_p()
        check(lib().b200_malloc(ctx._h, self.nbytes, C.byref(self._p)))
        self._owner = True

    @property
    def ptr(self) -> int:
        return self._p.value or 0

    def data_ptr(self) -> int:
        return self.ptr

    @property
    def size(self):
        return int(np.prod(self.shape))

    @classmethod
    def from_numpy(cls, ctx: Context, a: np.ndarray):
        a = np.asarray(a)
        out = cls(ctx, a.shape, a.dtype)
        out.upload(a)
        return out

    @classmethod
    def zeros(cls, ctx: Context, shape, dtype=np.float64):
        out = cls(ctx, shape, dtype)
        check(lib().b200_fill(ctx._h, out.size, 0.0, out._p, out.code))
        return out

    def upload(self, a: np.ndarray):
        a = np.asarray(a, dtype=self.dtype)
        a = np.asfortranarray(a) if a.ndim == 2 else np.ascontiguousarray(a)
        assert a.shape == self.shape, (a.shape, self.shape)
        check(lib().b200_upload(self.ctx._h, self._p, a.ctypes.data_as(C.c_void_p), self.nbytes))

    def numpy(self) -> np.ndarray:
        out = np.empty(self.shape, dtype=self.dtype, order="F")
        check(lib().b200_download(self.ctx._h, out.ctypes.data_as(C.c_void_p), self._p, self.nbytes))
        return out

    @classmethod
    def view(cls, ctx: Context, ptr: int, n: int, dtype) -> "DeviceArray":
        """non-owning vector view of `n` elements at the raw device address `ptr` (operator callbacks)."""
        v = object.__new__(cls)
        v.ctx, v.shape, v.dtype, v.code = ctx, (int(n),), np.dtype(dtype), dtype_code(dtype)
        v.nbytes = int(n) * v.dtype.itemsize
        v._p = C.c_void_p(ptr)
        v._owner = False
        return v

    def column(self, j: int) -> "DeviceArray":
        """view(V, :, j) -- non-owning."""
        v = object.__new__(DeviceArray)
        v.ctx, v.shape, v.dtype, v.code = self.ctx, (self.shape[0],), self.dtype, self.code
        v.nbytes = self.shape[0] * self.dtype.itemsize
        v._p = C.c_void_p(self.ptr + j * v.nbytes)
        v._owner = False
        return v

    def free(self):
        if getattr(self, "_owner", False) and self._p:
            lib().b200_free(self.ctx._h, self._p)
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def pinned_empty(shape, dtype=np.float64) -> np.ndarray:
    """numpy array backed by page-locked host memory (cudaMallocHost through the C ABI): host<->device
    copies of such arrays run at full PCIe/C2C bandwidth.  The memory lives until process exit."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape))
    p = C.c_void_p()
    check(lib().b200_host_alloc_pinned(max(n * dtype.itemsize, 16), C.byref(p)))
    buf = (C.c_char * (n * dtype.itemsize)).from_address(p.value)
    return np.frombuffer(buf, dtype=dtype, count=n).reshape(shape)


def as_device_ptr(v):
    """raw device address of a DeviceArray or of a torch CUDA tensor (zero-copy)."""
    if isinstance(v, DeviceArray):
        return C.c_void_p(v.ptr)
    if hasattr(v, "data_ptr") and hasattr(v, "is_cuda"):
        if not v.is_cuda or not v.is_contiguous():
            raise TypeError("torch tensors passed to the device path must be contiguous CUDA tensors")
        return C.c_void_p(v.data_ptr())
    raise TypeError(f"not a device array: {type(v)}")


def is_device(v) -> bool:
    return isinstance(v, DeviceArray) or (hasattr(v, "data_ptr") and getattr(v, "is_cuda", False))
