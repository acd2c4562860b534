"""Wire-format vocabulary: dtype names, serializer tags and the raw ("buffer_protocol") codec.

The raw payload of a tensor is ``numel * element_size`` bytes: the C-contiguous, native-endian image
of the *logical* view, no header (T:serialization.py:177-204, 254-265).  On the device path these
bytes are produced by the pack kernel; the helpers below are the host-side equivalents used for CPU
objects that do not go through the engine and by the tests."""
from __future__ import annotations

import io
import warnings
from enum import Enum
from typing import Dict, List

import torch

# name <-> dtype: exactly the strings the reference persists (T:serialization.py:72-88)
_NAMES: Dict[torch.dtype, str] = {
    dt: str(dt)
    for dt in (
        torch.float64,
        torch.float32,
        torch.float16,
        torch.bfloat16,
        torch.complex128,
        torch.complex64,
        torch.int64,
        torch.int32,
        torch.int16,
        torch.int8,
        torch.uint8,
        torch.bool,
        torch.qint32,
        torch.qint8,
        torch.quint8,
        torch.float8_e4m3fn,
        torch.float8_e5m2,
    )
}
_BY_NAME: Dict[str, torch.dtype] = {v: k for k, v in _NAMES.items()}
_ELEMENT_SIZE: Dict[torch.dtype, int] = {
    torch.float64: 8, torch.float32: 4, torch.float16: 2, torch.bfloat16: 2,
    torch.complex128: 16, torch.complex64: 8,
    torch.int64: 8, torch.int32: 4, torch.int16: 2, torch.int8: 1, torch.uint8: 1, torch.bool: 1,
    torch.qint32: 4, torch.qint8: 1, torch.quint8: 1,
    torch.float8_e4m3fn: 1, torch.float8_e5m2: 1,
}  # fmt: skip

# The public lists are exactly the reference's: code written against it (and its own test files) iterates over them
# and builds test tensors with torch.rand, which has no float8 kernel.  The float8 formats are known to the name and size
# tables above and travel raw (RAW_DTYPES), but are not listed here.
FLOAT8_DTYPES: List[torch.dtype] = [torch.float8_e4m3fn, torch.float8_e5m2]
ALL_SUPPORTED_DTYPES: List[torch.dtype] = [dt for dt in _NAMES if dt not in FLOAT8_DTYPES]
SUPPORTED_QUANTIZED_DTYPES: List[torch.dtype] = [torch.qint32, torch.qint8, torch.quint8]
# dtypes whose payload is the raw image (T:serialization.py:162-173); everything else uses torch.save
BUFFER_PROTOCOL_SUPPORTED_DTYPES: List[torch.dtype] = [
    torch.float64, torch.float32, torch.float16, torch.bfloat16,
    torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8, torch.bool,
]  # fmt: skip
# every dtype whose payload is the raw image: the reference's ten, and the two float8 formats (1-byte images, as int8)
RAW_DTYPES: List[torch.dtype] = BUFFER_PROTOCOL_SUPPORTED_DTYPES + FLOAT8_DTYPES


class Serializer(Enum):
    TORCH_SAVE = "torch_save"
    BUFFER_PROTOCOL = "buffer_protocol"
    PER_TENSOR_QTENSOR = "per_tensor_qtensor"
    PER_CHANNEL_QTENSOR = "per_channel_qtensor"
    PER_CHANNEL_FP8 = "per_channel_fp8"  # this package's scaled float8 format (per_channel_fp8_as_bytes)


def _unsupported(what) -> ValueError:
    return ValueError(f"Unsupported dtype {what}. (Supported dtypes are: {ALL_SUPPORTED_DTYPES})")


def dtype_to_string(dtype: torch.dtype) -> str:
    try:
        return _NAMES[dtype]
    except KeyError:
        raise _unsupported(dtype) from None


def string_to_dtype(s: str) -> torch.dtype:
    try:
        return _BY_NAME[s]
    except KeyError:
        raise _unsupported(s) from None


def dtype_to_element_size(dtype: torch.dtype) -> int:
    try:
        return _ELEMENT_SIZE[dtype]
    except KeyError:
        raise _unsupported(dtype) from None


def tensor_as_memoryview(tensor: torch.Tensor) -> memoryview:
    """Zero-copy raw image of a CPU tensor (a copy is made only if the view is not dense)."""
    if tensor.dtype not in RAW_DTYPES:
        raise ValueError(f"tensor_as_memoryview() doesn't support the dtype {tensor.dtype}.")
    if tensor.device.type != "cpu":
        raise ValueError("tensor_as_memoryview() only accepts CPU tensors.")
    flat = tensor.detach().contiguous().reshape(-1)
    if flat.numel() == 0:
        return memoryview(b"")
    # reinterpret as bytes: works for every raw dtype incl. bfloat16, which numpy cannot name
    return memoryview(flat.view(torch.uint8).numpy()).cast("b")


def tensor_from_memoryview(mv, dtype: torch.dtype, shape: List[int]) -> torch.Tensor:
    numel = 1
    for s in shape:
        numel *= s
    if numel == 0:
        return torch.empty(shape, dtype=dtype)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # read-only buffers are fine: the result is a temporary
        return torch.frombuffer(mv, dtype=dtype).reshape(shape)


def torch_save_as_bytes(obj) -> bytes:
    buf = io.BytesIO()
    torch.save(obj, buf)
    return buf.getvalue()


def torch_load_from_bytes(buf):
    return torch.load(io.BytesIO(buf), weights_only=False)


# ---- quantized tensors: the reference's self-describing formats (T:serialization.py:278-477) ---------------
# Specified and unit-tested by the reference but not wired into any of its preparers (quantized tensors travel
# as torch.save pickles); kept here with the same names so that either side can adopt them later.
#
#   per-tensor : [ int_repr bytes, C order ][ q_scale: C double ][ q_zero_point: C long long ]
#   per-channel: [ axis: C long long ][ int_repr bytes, C order ][ scales: float64 x shape[axis] ][ zero_points: int64 x shape[axis] ]
import struct as _struct

_INT_REPR = {torch.qint8: torch.int8, torch.quint8: torch.uint8, torch.qint32: torch.int32}


def _int_repr_bytes(tensor: torch.Tensor) -> bytes:
    return bytes(tensor_as_memoryview(tensor.contiguous().int_repr()))


def _int_repr_from(buf: memoryview, dtype: torch.dtype, shape: List[int]) -> torch.Tensor:
    return tensor_from_memoryview(buf, dtype=_INT_REPR[dtype], shape=shape)


def per_tensor_qtensor_as_bytes(tensor: torch.Tensor) -> bytes:
    if not tensor.is_quantized or tensor.qscheme() != torch.per_tensor_affine:
        raise RuntimeError("per_tensor_qtensor_as_bytes() only supports per_tensor_affine quantized tensor.")
    return _int_repr_bytes(tensor) + _struct.pack("d", tensor.q_scale()) + _struct.pack("q", tensor.q_zero_point())


def per_tensor_qtensor_from_bytes(buf: bytes, dtype: torch.dtype, shape: List[int]) -> torch.Tensor:
    view = memoryview(buf)
    body = len(view) - 16
    expected = dtype_to_element_size(dtype)
    for s in shape:
        expected *= s
    if body != expected:
        raise RuntimeError(f"The size of the buffer ({len(view)}) does not match the dtype/shape ({expected} + 16).")
    (scale,) = _struct.unpack("d", view[body : body + 8])
    (zero_point,) = _struct.unpack("q", view[body + 8 : body + 16])
    return torch._make_per_tensor_quantized_tensor(_int_repr_from(view[:body], dtype, shape), scale, zero_point)


def per_channel_qtensor_as_bytes(tensor: torch.Tensor) -> bytes:
    if not tensor.is_quantized or tensor.qscheme() not in (torch.per_channel_affine, torch.per_channel_affine_float_qparams):
        raise RuntimeError("per_channel_qtensor_as_bytes() only supports per_channel_affine quantized tensor.")
    scales = tensor.q_per_channel_scales().to(torch.float64)
    zero_points = tensor.q_per_channel_zero_points().to(torch.int64)
    return (
        _struct.pack("q", tensor.q_per_channel_axis())
        + _int_repr_bytes(tensor)
        + bytes(tensor_as_memoryview(scales))
        + bytes(tensor_as_memoryview(zero_points))
    )


def per_channel_qtensor_from_bytes(buf: bytes, dtype: torch.dtype, shape: List[int]) -> torch.Tensor:
    view = memoryview(buf)
    (axis,) = _struct.unpack("q", view[:8])
    body = dtype_to_element_size(dtype)
    for s in shape:
        body *= s
    channels = shape[axis]
    if len(view) != 8 + body + 16 * channels:
        raise RuntimeError(f"The size of the buffer ({len(view)}) does not match the dtype/shape/axis.")
    ints = _int_repr_from(view[8 : 8 + body], dtype, shape)
    scales = tensor_from_memoryview(view[8 + body : 8 + body + 8 * channels], dtype=torch.float64, shape=[channels])
    zero_points = tensor_from_memoryview(view[8 + body + 8 * channels :], dtype=torch.int64, shape=[channels])
    return torch._make_per_channel_quantized_tensor(ints, scales, zero_points, axis)


# ---- per-channel scaled float8 (this package's format; the reference has no reader for it) ------------------------
#   [ axis: int64 ][ float8 bytes, C order ][ scales: float32 x shape[axis] ], little-endian
def per_channel_fp8_as_bytes(q: torch.Tensor, scales: torch.Tensor, axis: int) -> bytes:
    """The payload of a float8 tensor ``q`` with fp32 ``scales`` along ``axis`` (``prepare.per_channel_fp8`` gives both)."""
    if q.dtype not in FLOAT8_DTYPES or scales.numel() != q.shape[axis]:
        raise RuntimeError("per_channel_fp8_as_bytes() takes a float8 tensor and one scale per channel along axis.")
    return _struct.pack("<q", axis) + bytes(tensor_as_memoryview(q.cpu())) + bytes(tensor_as_memoryview(scales.cpu().float()))


def per_channel_fp8_from_bytes(buf: bytes, dtype: torch.dtype, shape: List[int]) -> torch.Tensor:
    """The dequantised fp32 tensor of a per_channel_fp8 payload: ``q.float() * scale`` of its channel."""
    from .prepare import dequantize_fp8

    view = memoryview(buf)
    axis = _struct.unpack("<q", view[:8])[0] if len(view) >= 8 else -1
    if not 0 <= axis < len(shape):
        raise RuntimeError(f"per_channel_fp8 header names axis {axis}, but the saved tensor has shape {list(shape)}")
    body = 1
    for s in shape:
        body *= s
    channels = shape[axis]
    if dtype not in FLOAT8_DTYPES or len(view) != 8 + body + 4 * channels:
        raise RuntimeError(f"The size of the buffer ({len(view)}) does not match the dtype/shape/axis.")
    q = tensor_from_memoryview(view[8 : 8 + body], dtype=dtype, shape=shape)
    scales = tensor_from_memoryview(view[8 + body :], dtype=torch.float32, shape=[channels])
    return dequantize_fp8(q, scales, axis)
