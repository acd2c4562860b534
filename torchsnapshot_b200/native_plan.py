"""Turns stagers / consumers into C-ABI copy descriptors: the only code that knows how a tensor maps to its wire image.

Both the engine's file jobs (``scheduler``) and the asyncio ``stage_buffer`` / ``consume_buffer`` seam use it.  It works
on this package's classes and, by duck typing on the attribute names they share, on the reference's own
``TensorBufferStager`` / ``BatchedBufferStager`` / ``GPUBatchedBufferStager`` / ``TensorBufferConsumer`` /
``ShardedTensorBufferConsumer`` / ``BatchedBufferConsumer`` objects (T:io_preparers/tensor.py:223-350,
T:batcher.py:51-162,358-384, T:io_preparers/sharded_tensor.py:285-323) — which is what lets
``torchsnapshot_b200.install()`` put the engine underneath an unmodified torchsnapshot."""
from __future__ import annotations

import os
import struct
from typing import Any, List, Optional, Tuple

import torch

from . import _native
from .prepare import _CASTABLE, _FLOATS, PER_CHANNEL_FP8, PER_CHANNEL_QTENSOR, PER_TENSOR_QTENSOR, PerChannel, fused_cast_of
from .serialization import RAW_DTYPES, Serializer, dtype_to_element_size, string_to_dtype

RAW = Serializer.BUFFER_PROTOCOL.value
_DTYPES = {str(dt): dt for dt in RAW_DTYPES}

Described = Tuple[List["_native.CopyDesc"], List[torch.Tensor], int]  # descriptors, keep-alive, wire bytes


PER_CHANNEL = (PER_CHANNEL_QTENSOR, PER_CHANNEL_FP8)  # serializers of the per-channel formats
_PARAM_BYTES = {PER_CHANNEL_QTENSOR: 16, PER_CHANNEL_FP8: 4}  # bytes of parameters per channel


def entry_nbytes(entry: Any, axis: Optional[int] = None) -> int:
    """Payload size of a tensor entry.  A per-tensor quantised one carries ``[q_scale: double][q_zero_point: int64]``
    behind the int_repr bytes (T:serialization.py:278-310); a per-channel one ``[axis: int64]`` before them and, given
    the axis (only the file records it), its parameters behind them: ``[scales: f64 x C][zero_points: i64 x C]`` for
    int8, ``[scales: f32 x C]`` for float8."""
    n = dtype_to_element_size(string_to_dtype(entry.dtype))
    for s in entry.shape:
        n *= s
    if entry.serializer == PER_TENSOR_QTENSOR:
        n += 16
    elif entry.serializer in PER_CHANNEL:
        n += 8 + (_PARAM_BYTES[entry.serializer] * entry.shape[axis] if axis is not None else 0)
    return n


def raw_castable(src: torch.dtype, dst: torch.dtype) -> bool:
    """dtype pairs the scatter kernel handles itself; others fall back to Tensor.copy_ semantics."""
    if src == dst:
        return src in RAW_DTYPES
    return src in _CASTABLE and dst in _CASTABLE


# ---- save side -----------------------------------------------------------------------------------
class HostCloneBudget:
    """Host bytes ``async_take`` may spend on private copies of CPU tensors (the engine reads host memory after
    ``async_take`` has returned, so the caller's tensor must not be the source).  The reference admits staging only while the
    per-rank memory budget allows and lets ``async_take`` wait for writes to free it (T:scheduler.py:259-281); here a CPU
    tensor that no longer fits is not copied at all: its request is marked blocking and written out before ``async_take``
    returns, straight from the caller's memory."""

    def __init__(self, nbytes: int) -> None:
        self.remaining = max(0, int(nbytes))
        self.cloned_bytes = 0
        self.blocking_bytes = 0
        self._blocking = False

    def admit(self, nbytes: int) -> bool:
        if self._blocking or nbytes > self.remaining:
            self._blocking = True  # the rest of this request is read in place as well
            self.blocking_bytes += nbytes
            return False
        self.remaining -= nbytes
        self.cloned_bytes += nbytes
        return True

    def take_blocking(self) -> bool:
        """Did the request described since the last call leave a CPU tensor uncopied?"""
        b, self._blocking = self._blocking, False
        return b


def _describe_tensor_stager(st: Any, offset: int, clones: Optional[HostCloneBudget]) -> Optional[Described]:
    entry = getattr(st, "entry", None)
    tensor = getattr(st, "tensor", None)
    serializer = getattr(entry, "serializer", None)
    if not isinstance(tensor, torch.Tensor):
        return None
    t = tensor.detach()
    # quantise-on-save (prepare.quantize_on_save): the stager computed the parameters once, when it was created
    q = getattr(st, "qparams", None) if serializer in (PER_TENSOR_QTENSOR,) + PER_CHANNEL else None
    wire_dtype = qparams = axis = None
    if isinstance(q, PerChannel):
        # the engine writes the axis header, the int or float8 body behind it and the channel parameters behind the body
        wire_dtype, axis, nbytes, offset = q.dtype, q.axis, entry_nbytes(entry, q.axis), offset + 8
    elif q is not None:
        # the pack kernel writes int_repr + the 16-byte trailer
        wire_dtype, qparams, nbytes = q[0], q[1:], entry_nbytes(entry)
    elif serializer == RAW and entry.dtype in _DTYPES:
        func = getattr(st, "_tensor_prepare_func", None)
        if func is not None:
            wire_dtype = fused_cast_of(func, t)
            if wire_dtype is None:
                t = func(t, False).detach()  # persist the processed tensor (DESIGN.md §6)
            # else: a pure float cast — the pack kernel converts while it gathers, no processed tensor is materialised
        if str(wire_dtype or t.dtype) != entry.dtype or list(t.shape) != list(entry.shape):
            return None
        nbytes = entry_nbytes(entry)
        if t.numel() == 0:
            return [], [], nbytes
    else:
        return None
    if _native.needs_contiguous_copy(t):
        t = t.contiguous()
    elif getattr(st, "is_async_snapshot", False) and t.device.type == "cpu":
        # host memory is read after async_take returned: a private copy while the budget lasts, else a blocking request
        if clones is None or clones.admit(t.numel() * t.element_size()):
            t = t.clone()
    return [_native.save_desc(t, offset, wire_dtype=wire_dtype, qparams=qparams, axis=axis)], [t], nbytes


def describe_stager(st: Any, clones: Optional[HostCloneBudget] = None) -> Optional[Described]:
    """(descriptors, keep-alive tensors, wire size) of one WriteReq's stager, or None when it has to go
    through its own ``stage_buffer`` (pickled objects, complex / quantized tensors, foreign stagers).
    Without ``clones`` every CPU source of an async snapshot is copied."""
    members = getattr(st, "byte_range_to_buffer_stager", None)
    if members is not None:
        descs: List[Any] = []
        keep: List[torch.Tensor] = []
        end = 0
        for (lo, hi), member in members.items():
            one = _describe_tensor_stager(member, lo, clones)
            if one is None or one[2] != hi - lo or lo != end:
                return None
            descs += one[0]
            keep += one[1]
            end = hi
        return descs, keep, end
    return _describe_tensor_stager(st, 0, clones)


# ---- restore side ----------------------------------------------------------------------------------
def per_channel_axis(head: bytes, size: int, entry: Any, where: str) -> int:
    """Axis of a per-channel image of ``size`` bytes that starts with the 8 bytes ``head``, checked against the entry's
    shape: the manifest records neither the axis nor the size.  ``where`` names the image in the error."""
    shape = list(entry.shape)
    axis = struct.unpack("<q", head)[0] if len(head) == 8 else -1
    if not 0 <= axis < len(shape):
        raise RuntimeError(f"{where}: per-channel header names axis {axis}, but the saved tensor has shape {shape}")
    want = entry_nbytes(entry, axis)
    if size != want:
        raise RuntimeError(f"{where}: {size} bytes, but a per-channel image of shape {shape} along axis {axis} has {want}")
    return axis


def _describe_tensor_consumer(c: Any, offset: int, root: Optional[str] = None, buf: Any = None) -> Optional[Described]:
    entry = getattr(c, "entry", None)
    serializer = getattr(entry, "serializer", None)
    raw = serializer == RAW and entry.dtype in _DTYPES
    if not raw and serializer not in PER_CHANNEL:
        return None
    shape = list(entry.shape)
    regions = getattr(c, "overlapping_regions", None)
    if regions is not None:
        # reshard-on-load: each overlap is one strided copy out of the saved piece's C-order image
        targets = [(r.dst_tensor, r.overlap_region) for r in regions]
    else:
        tensor = getattr(c, "tensor", None)
        if not isinstance(tensor, torch.Tensor) or list(tensor.shape) != shape:
            return None
        targets = [(tensor, ())]
    skip = int(getattr(c, "wire_skip", 0) or 0)
    axis = None
    if raw:
        wire_dtype = _DTYPES[entry.dtype]
        if not all(raw_castable(wire_dtype, t.dtype) for t, _ in targets):
            return None
        nbytes = entry_nbytes(entry) if getattr(c, "wire_len", None) is None else int(c.wire_len)
        esz, body = dtype_to_element_size(wire_dtype), offset - skip
    else:
        # dequantising scatter into float targets; quantised targets keep torch's own copy semantics
        if skip or getattr(entry, "byte_range", None) is not None or (root is None and buf is None):
            return None
        if not all(t.dtype in _FLOATS for t, _ in targets):
            return None
        if buf is None:
            where = os.path.join(root, entry.location)
            nbytes = os.stat(where).st_size
            with open(where, "rb") as f:
                head = f.read(8)
        else:
            where, nbytes, head = entry.location, len(buf), bytes(buf[:8])
        axis = per_channel_axis(head, nbytes, entry, where)
        wire_dtype, esz, body = string_to_dtype(entry.dtype), 1, offset + 8
    strides = _native._c_strides(shape)
    descs, keep = [], []
    for tensor, narrows in targets:
        dst, first = tensor.detach(), 0
        for dim, so, do, n in narrows:
            dst = dst.narrow(dim, do, n)
            first += so * strides[dim]
        if dst.numel():
            d = _native.load_desc(dst, body + first * esz, wire_dtype=wire_dtype, wire_strides=strides)
            descs.append(d if axis is None else _native.per_channel(d, shape, axis, body))
            keep.append(tensor)
    return descs, keep, nbytes


def describe_consumer(c: Any, root: Optional[str] = None, buf: Any = None) -> Optional[Described]:
    """(descriptors, keep-alive tensors, wire size) of one ReadReq's consumer, or None when it has to go through its own
    ``consume_buffer``.  A per-channel entry's layout is read from ``buf`` (the bytes the consumer was handed) or else
    from its file under ``root``, the directory the entries' locations are relative to."""
    members = getattr(c, "byte_range_to_buffer_consumer", None)
    if members is not None:
        descs: List[Any] = []
        keep: List[torch.Tensor] = []
        for (lo, hi), member in members.items():
            one = _describe_tensor_consumer(member, lo)
            if one is None:
                return None
            descs += one[0]
            keep += one[1]
        return descs, keep, int(getattr(c, "buf_sz_bytes", 0))
    return _describe_tensor_consumer(c, 0, root, buf)


def native_root(storage: Any, op: str = "write") -> Optional[str]:
    """Root directory when `storage` is a plain local-filesystem plugin the engine may do the I/O for.

    A subclass that overrides ``write`` / ``read`` (fault injection, throttling, auditing …) keeps control of that
    operation: the engine only takes over when the method is the stock one."""
    cls = type(storage)
    root = getattr(storage, "native_root", None)
    if root is not None:
        from .storage_plugins.fs import FSStoragePlugin

        stock = getattr(FSStoragePlugin, op, None)
        if isinstance(storage, FSStoragePlugin) and getattr(cls, op, None) is not stock:
            return None
        return root
    if cls.__name__ == "FSStoragePlugin" and cls.__module__.endswith("storage_plugins.fs") and isinstance(getattr(storage, "root", None), str):
        return storage.root
    return None
