"""Turns stagers / consumers into C-ABI copy descriptors.

Works on this package's classes and, by duck typing on the attribute names they share, on the
reference's own ``TensorBufferStager`` / ``BatchedBufferStager`` / ``GPUBatchedBufferStager`` /
``TensorBufferConsumer`` / ``ShardedTensorBufferConsumer`` / ``BatchedBufferConsumer`` objects
(T:io_preparers/tensor.py:223-350, T:batcher.py:51-162,358-384, T:io_preparers/sharded_tensor.py:285-323) —
which is what lets ``torchsnapshot_b200.install()`` put the engine underneath an unmodified torchsnapshot."""
from __future__ import annotations

import os
import struct
from typing import Any, List, Optional, Tuple

import torch

from . import _native
from .prepare import PER_CHANNEL_QTENSOR
from .serialization import BUFFER_PROTOCOL_SUPPORTED_DTYPES

RAW = "buffer_protocol"
_FLOATS = (torch.float16, torch.bfloat16, torch.float32, torch.float64)
_DTYPES = {str(dt): dt for dt in BUFFER_PROTOCOL_SUPPORTED_DTYPES}

Described = Tuple[List["_native.CopyDesc"], List[torch.Tensor], int]  # descriptors, keep-alive, wire bytes


def _entry_nbytes(entry: Any) -> int:
    n = torch.empty(0, dtype=_DTYPES[entry.dtype]).element_size()
    for s in entry.shape:
        n *= s
    return n


def _castable(src: torch.dtype, dst: torch.dtype) -> bool:
    return src == dst or (src in _FLOATS and dst in _FLOATS)


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


def _describe_tensor_stager(st: Any, offset: int, clones: Optional[HostCloneBudget] = None) -> Optional[Described]:
    entry = getattr(st, "entry", None)
    tensor = getattr(st, "tensor", None)
    if entry is not None and isinstance(tensor, torch.Tensor) and getattr(st, "qparams", None) is not None:
        # quantise-on-save: the pack kernel produces int_repr + trailer, or the engine the whole per-channel image
        # (prepare.quantize_on_save)
        descs, keep = st.native_descs(offset)
        return descs, keep, st.wire_nbytes()
    if entry is None or not isinstance(tensor, torch.Tensor) or getattr(entry, "serializer", None) != RAW:
        return None
    if entry.dtype not in _DTYPES:
        return None
    t = tensor.detach()
    func = getattr(st, "_tensor_prepare_func", None)
    wire_dtype = None
    if func is not None:
        from .prepare import fused_cast_of

        wire_dtype = fused_cast_of(func, t)
        if wire_dtype is None:
            t = func(t, False).detach()  # persist the processed tensor (DESIGN.md §6)
        # else: a pure float cast — the pack kernel converts while it gathers, no processed tensor is materialised
    if str(wire_dtype or t.dtype) != entry.dtype or list(t.shape) != list(entry.shape):
        return None
    nbytes = _entry_nbytes(entry)
    if t.numel() == 0:
        return [], [], nbytes
    if _native.needs_contiguous_copy(t):
        t = t.contiguous()
    elif getattr(st, "is_async_snapshot", False) and t.device.type == "cpu":
        # host memory is read after async_take returned: a private copy while the budget lasts, else a blocking request
        if clones is None or clones.admit(t.numel() * t.element_size()):
            t = t.clone()
    return [_native.save_desc(t, offset, wire_dtype=wire_dtype)], [t], nbytes


def describe_stager(st: Any, clones: Optional[HostCloneBudget] = None) -> Optional[Described]:
    """(descriptors, keep-alive tensors, wire size) of one WriteReq's stager, or None when it has to go
    through its own ``stage_buffer`` (pickled objects, complex / quantized tensors, foreign stagers)."""
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
def per_channel_layout(path: str, entry: Any) -> Tuple[int, int]:
    """(file size, axis) of a per-channel file, from the file itself: the manifest records neither."""
    from .io_preparers.tensor import per_channel_wire_nbytes

    shape = list(entry.shape)
    size = os.stat(path).st_size
    with open(path, "rb") as f:
        head = f.read(8)
    axis = struct.unpack("<q", head)[0] if len(head) == 8 else -1
    if not 0 <= axis < len(shape):
        raise RuntimeError(f"{path}: per-channel header names axis {axis}, but the saved tensor has shape {shape}")
    if size != per_channel_wire_nbytes(shape, axis):
        raise RuntimeError(f"{path}: {size} bytes, but a per-channel image of shape {shape} along axis {axis} has "
                           f"{per_channel_wire_nbytes(shape, axis)}")
    return size, axis


def _describe_per_channel_consumer(c: Any, offset: int, root: Optional[str]) -> Optional[Described]:
    """Dequantising scatter of a per-channel entry into float targets (the whole tensor or reshard overlaps)."""
    entry = c.entry
    regions = getattr(c, "overlapping_regions", None)
    targets = [r.dst_tensor for r in regions] if regions is not None else [getattr(c, "tensor", None)]
    if root is None or getattr(entry, "byte_range", None) is not None or int(getattr(c, "wire_skip", 0) or 0):
        return None
    if not all(isinstance(t, torch.Tensor) and t.dtype in _FLOATS for t in targets):
        return None  # quantised targets keep torch's own copy semantics
    nbytes, axis = per_channel_layout(os.path.join(root, entry.location), entry)
    qdtype = {"torch.qint8": torch.qint8, "torch.quint8": torch.quint8}[entry.dtype]
    shape = list(entry.shape)
    strides = _native._c_strides(shape)
    body = offset + 8

    def desc(dst: torch.Tensor, first: int):
        return _native.per_channel(_native.load_desc(dst, body + first, wire_dtype=qdtype, wire_strides=strides), shape, axis, body)

    if regions is None:
        dst = c.tensor.detach()
        if list(dst.shape) != shape:
            return None
        return ([desc(dst, 0)] if dst.numel() else []), [dst], nbytes
    descs, keep = [], []
    for region in regions:
        dst = region.dst_tensor.detach()
        first = 0
        for dim, so, do, n in region.overlap_region:
            dst = dst.narrow(dim, do, n)
            first += so * strides[dim]
        if dst.numel():
            descs.append(desc(dst, first))
            keep.append(region.dst_tensor)
    return descs, keep, nbytes


def _describe_tensor_consumer(c: Any, offset: int, root: Optional[str] = None) -> Optional[Described]:
    entry = getattr(c, "entry", None)
    if entry is not None and getattr(entry, "serializer", None) == PER_CHANNEL_QTENSOR:
        return _describe_per_channel_consumer(c, offset, root)
    if entry is None or getattr(entry, "serializer", None) != RAW or entry.dtype not in _DTYPES:
        return None
    src_dtype = _DTYPES[entry.dtype]
    nbytes = _entry_nbytes(entry)
    regions = getattr(c, "overlapping_regions", None)
    if regions is not None:
        # reshard-on-load: each overlap is one strided copy out of the saved piece's C-order image
        shape = list(entry.shape)
        esz = torch.empty(0, dtype=src_dtype).element_size()
        strides = [1] * len(shape)
        for i in range(len(shape) - 2, -1, -1):
            strides[i] = strides[i + 1] * shape[i + 1]
        descs, keep = [], []
        skip = int(getattr(c, "wire_skip", 0) or 0)
        if getattr(c, "wire_len", None) is not None:
            nbytes = int(c.wire_len)
        for region in regions:
            dst = region.dst_tensor.detach()
            if not _castable(src_dtype, dst.dtype) or dst.is_quantized:
                return None
            first = 0
            for dim, so, do, n in region.overlap_region:
                dst = dst.narrow(dim, do, n)
                first += so * strides[dim]
            if dst.numel() == 0:
                continue
            descs.append(_native.load_desc(dst, offset + first * esz - skip, wire_dtype=src_dtype, wire_strides=strides))
            keep.append(region.dst_tensor)
        return descs, keep, nbytes
    tensor = getattr(c, "tensor", None)
    if not isinstance(tensor, torch.Tensor) or tensor.is_quantized or not _castable(src_dtype, tensor.dtype):
        return None
    dst = tensor.detach()
    if list(dst.shape) != list(entry.shape):
        return None
    if dst.numel() == 0:
        return [], [], nbytes
    return [_native.load_desc(dst, offset, wire_dtype=src_dtype)], [dst], nbytes


def describe_consumer(c: Any, root: Optional[str] = None) -> Optional[Described]:
    """(descriptors, keep-alive tensors, wire size) of one ReadReq's consumer, or None when it has to go through its own
    ``consume_buffer``.  ``root``: directory the entries' locations are relative to; per-channel entries need it to read
    their layout from the file."""
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
    return _describe_tensor_consumer(c, 0, root)


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
