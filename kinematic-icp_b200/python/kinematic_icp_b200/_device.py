"""Arrays already in GPU memory: any object exposing __cuda_array_interface__ (torch CUDA tensors, CuPy, Numba).  Nothing here
imports torch unless the caller passed a torch tensor, and nothing is ever copied between host and device."""
from typing import NamedTuple

from ._capi import KICP_DTYPE_F32, KICP_DTYPE_F64

CUDA_STREAM_LEGACY = 1  # cudaStreamLegacy


def interface(obj):
    """The object's __cuda_array_interface__ dict, or None for host data."""
    return getattr(obj, "__cuda_array_interface__", None)


def is_device(obj):
    return interface(obj) is not None


class DevicePoints(NamedTuple):
    """A device array as kicp_frame_input / kicp_scan_attach_device take it."""
    ptr: int
    n: int
    dtype: int
    point_step: int
    offsets: tuple


def _itemsize(typestr):
    return int(typestr[2:])


def _strides(cai):
    """Byte strides of the array (C-contiguous when the interface gives none)."""
    shape, w = tuple(cai["shape"]), _itemsize(cai["typestr"])
    if cai.get("strides") is not None:
        return tuple(cai["strides"])
    out, acc = [], w
    for d in reversed(shape):
        out.append(acc)
        acc *= d
    return tuple(reversed(out))


def _contiguous(cai):
    shape = tuple(cai["shape"])
    if cai.get("strides") is None:
        return True
    acc = _itemsize(cai["typestr"])
    for d, s in zip(reversed(shape), reversed(cai["strides"])):
        if d > 1 and s != acc:
            return False
        acc *= d
    return True


def device_points(obj, point_step=0, offsets=(0, 0, 0)):
    """Map a device array to a DevicePoints.

    - (N, 3) or (N, k >= 3) float32 / float64 with unit column stride: point_step = the row stride in bytes, offsets 0 / w / 2w;
    - with point_step > 0: C-contiguous records (uint8 or any type, read as bytes, as the host path takes them), float32 x, y, z at
      `offsets`, n = bytes // point_step.
    Anything else raises ValueError."""
    cai = interface(obj)
    if cai is None:
        raise ValueError("expected an object exposing __cuda_array_interface__")
    shape, typestr = tuple(cai["shape"]), cai["typestr"]
    ptr = int(cai["data"][0] or 0)
    if point_step:
        if not _contiguous(cai):
            raise ValueError("records with point_step must be C-contiguous")
        nbytes = _itemsize(typestr)
        for d in shape:
            nbytes *= d
        return DevicePoints(ptr, nbytes // int(point_step), KICP_DTYPE_F32, int(point_step), tuple(int(o) for o in offsets))
    if typestr not in ("<f4", "<f8") or len(shape) != 2 or shape[1] < 3:
        raise ValueError("expected an (N, 3) or (N, k) float32 / float64 device array, got shape %s typestr %s" % (shape, typestr))
    w = _itemsize(typestr)
    row, col = _strides(cai)
    if col != w or (shape[0] > 1 and row < shape[1] * w):
        raise ValueError("device points need unit column stride and rows that do not overlap (strides %s)" % ((row, col),))
    if shape[0] <= 1:
        row = shape[1] * w
    return DevicePoints(ptr, shape[0], KICP_DTYPE_F32 if w == 4 else KICP_DTYPE_F64, row, (0, w, 2 * w))


def device_vector(obj, typestr, what):
    """(pointer, length) of a 1-D device array of `typestr` elements with unit stride."""
    cai = interface(obj)
    shape = tuple(cai["shape"])
    if cai["typestr"] != typestr or len(shape) != 1 or (shape[0] > 1 and _strides(cai)[0] != _itemsize(typestr)):
        raise ValueError("%s: expected a 1-D contiguous %s device array" % (what, typestr))
    return int(cai["data"][0] or 0), shape[0]


def device_output(obj, what):
    """(pointer, capacity, dtype code) of a contiguous (cap, 3) float32 / float64 device array."""
    cai = interface(obj)
    if cai is None:
        raise ValueError("%s: expected a device array" % what)
    shape, typestr = tuple(cai["shape"]), cai["typestr"]
    if typestr not in ("<f4", "<f8") or len(shape) != 2 or shape[1] != 3 or not _contiguous(cai):
        raise ValueError("%s: expected a contiguous (cap, 3) float32 / float64 device array" % what)
    return int(cai["data"][0] or 0), shape[0], KICP_DTYPE_F32 if typestr == "<f4" else KICP_DTYPE_F64


def output_f64(obj, shape, what):
    """Pointer of `obj`, a C-contiguous float64 device array of exactly `shape` ((n, 3) or (n,))."""
    cai = interface(obj)
    if cai is None or cai["typestr"] != "<f8" or tuple(cai["shape"]) != tuple(shape) or not _contiguous(cai):
        raise ValueError("%s: expected a contiguous float64 device array of shape %s" % (what, tuple(shape)))
    return int(cai["data"][0] or 0)


def output_u8(obj, n, what):
    """Pointer of `obj`, a contiguous uint8 device array of shape (n,)."""
    cai = interface(obj)
    if cai is None or cai["typestr"] != "|u1" or tuple(cai["shape"]) != (n,) or not _contiguous(cai):
        raise ValueError("%s: expected a contiguous uint8 device array of shape (%d,)" % (what, n))
    return int(cai["data"][0] or 0)


def empty_u8(like, n, what):
    """A new uint8 torch tensor of shape (n,) on the device of `like`, a torch tensor; any other device input needs out=."""
    if not _is_torch_tensor(like):
        raise ValueError("%s: pass out= for a device input that is not a torch tensor" % what)
    import torch
    return torch.empty((n,), dtype=torch.uint8, device=like.device)


def empty_f64(like, shape, what):
    """A new float64 torch tensor of `shape` on the device of `like`, a torch tensor; any other device input needs out=."""
    if not _is_torch_tensor(like):
        raise ValueError("%s: pass out= for a device input that is not a torch tensor" % what)
    import torch
    return torch.empty(shape, dtype=torch.float64, device=like.device)


def _is_torch_tensor(obj):
    return type(obj).__module__.split(".")[0] == "torch" and hasattr(obj, "device")


def resolve_stream(stream, array=None):
    """The cudaStream_t (an int) a call on `array` is ordered with: `stream` itself (an int, or an object with .cuda_stream (torch) or
    .ptr (CuPy)); when it is None, the interface's version-3 "stream" entry, else for a torch tensor torch.cuda.current_stream of its
    device, else the legacy default stream."""
    if stream is not None:
        if isinstance(stream, int):
            return stream
        for attr in ("cuda_stream", "ptr"):
            if hasattr(stream, attr):
                return int(getattr(stream, attr))
        raise TypeError("stream: expected an int cudaStream_t or an object with .cuda_stream or .ptr")
    cai = interface(array) if array is not None else None
    if cai is not None and cai.get("stream") is not None:
        return int(cai["stream"])
    if array is not None and _is_torch_tensor(array):
        import torch
        return int(torch.cuda.current_stream(array.device).cuda_stream)
    return CUDA_STREAM_LEGACY


class DeviceCloud:
    """A zero-copy view of context-owned device memory: an (n, 3) array exposing __cuda_array_interface__ (torch.as_tensor /
    cupy.asarray consume it).  It keeps its owner alive; the memory itself is valid until the owner's next front-end call.  The
    interface does not flag it read-only (torch refuses such arrays), but writing into it changes nothing the library reads later."""

    def __init__(self, ptr, n, dtype, owner):
        self.ptr, self.n, self.dtype, self._owner = int(ptr or 0), int(n), dtype, owner
        self.shape = (self.n, 3)

    def __len__(self):
        return self.n

    @property
    def __cuda_array_interface__(self):
        return {"shape": self.shape, "typestr": "<f4" if self.dtype == KICP_DTYPE_F32 else "<f8",
                "data": (self.ptr if self.n else 0, False), "version": 3, "strides": None, "stream": None}


class DeviceArray:
    """A zero-copy view of context-owned device memory of any shape and element type (`typestr`, e.g. "<f8", "|u1"), exposing
    __cuda_array_interface__ like DeviceCloud, with DeviceCloud's lifetime rules."""

    def __init__(self, ptr, shape, typestr, owner):
        self.ptr, self.shape, self.typestr, self._owner = int(ptr or 0), tuple(int(s) for s in shape), typestr, owner

    def __len__(self):
        return self.shape[0]

    @property
    def __cuda_array_interface__(self):
        return {"shape": self.shape, "typestr": self.typestr, "data": (self.ptr if self.shape[0] else 0, False), "version": 3,
                "strides": None, "stream": None}
