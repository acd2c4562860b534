"""``_custom_tensor_prepare_func`` helpers (T:snapshot.py:120-122, 591-595; T:io_preparers/tensor.py:59-81).

The reference traces the hook at plan time to fill ``TensorEntry.dtype`` but then stages the *unprocessed* tensor
(T:io_preparers/tensor.py:240-258), so a casting hook yields an unreadable snapshot there.  Here the processed tensor
is what gets persisted — and when the hook is one of the recognisable casts below, no processed tensor is ever
materialised: the conversion is fused into the pack kernel (``tsnap_copy_desc.dst_dtype != src_dtype``), which reads
the live tensor once and writes the narrower wire image straight into the staging arena."""
from __future__ import annotations

import fnmatch
import functools
from typing import Callable, Optional

import torch

_FLOATS = (torch.float16, torch.bfloat16, torch.float32, torch.float64)  # what the quantisers (and cast sources) take
# cast_on_save targets and the float dtypes a restore converts between: the four wide floats and the two plain float8
# formats (raw 1-byte images, converted with torch's rounding; no scales)
_CASTABLE = _FLOATS + (torch.float8_e4m3fn, torch.float8_e5m2)


class _Traced:
    """What a tracing call returns when materialising the processed tensor would be wasteful or impossible
    (quantised meta tensors do not exist): dtype and shape, the two things T:io_preparers/tensor.py:59-81 reads."""

    def __init__(self, shape, dtype) -> None:
        self.shape, self.dtype = torch.Size(shape), dtype


def cast_on_save(dtype: torch.dtype, only: Optional[str] = None) -> Callable[[str, torch.Tensor, bool], torch.Tensor]:
    """A ``_custom_tensor_prepare_func`` that stores floating-point tensors as ``dtype`` (e.g. fp32 master weights as
    bf16).  ``only``: glob on the logical path; other tensors are stored unchanged.

    ``dtype`` may be ``torch.float8_e4m3fn`` or ``torch.float8_e5m2``: fp64 / fp32 / fp16 / bf16 tensors are then
    rounded to float8 as ``Tensor.to`` does it (values past e4m3fn's range become NaN, e5m2 overflows to inf).  Tensors
    that already are float8 are stored unchanged.

        Snapshot.take(path, app_state, _custom_tensor_prepare_func=cast_on_save(torch.bfloat16, only="model/*"))
    """
    if dtype not in _CASTABLE:
        raise ValueError(f"cast_on_save supports {_CASTABLE}, not {dtype}")

    def applies(logical_path: Optional[str], tensor: torch.Tensor) -> Optional[torch.dtype]:
        if tensor.dtype not in _FLOATS or tensor.dtype == dtype or tensor.is_quantized:
            return None
        if only is not None and (logical_path is None or not fnmatch.fnmatch(logical_path, only)):
            return None
        return dtype

    def prepare(logical_path: str, tensor: torch.Tensor, tracing: bool) -> torch.Tensor:
        target = applies(logical_path, tensor)
        if target is None:
            return tensor
        if tracing:  # the planner only looks at dtype and shape
            return torch.empty(tensor.shape, dtype=target, device="meta")
        return tensor.to(target)

    prepare.tsnap_cast = applies  # type: ignore[attr-defined]  # recognised by native_plan: fused into the pack kernel
    return prepare


def fused_cast_of(func, tensor: torch.Tensor) -> Optional[torch.dtype]:
    """Wire dtype when ``func`` (possibly wrapped in functools.partial(func, logical_path), as Snapshot does,
    T:snapshot.py:591-595) is a recognised pure cast for ``tensor``; None otherwise."""
    args = []
    inner = func
    while isinstance(inner, functools.partial):
        args = list(inner.args) + args
        inner = inner.func
    spec = getattr(inner, "tsnap_cast", None)
    if spec is None:
        return None
    return spec(args[0] if args else None, tensor)


PER_TENSOR_QTENSOR = "per_tensor_qtensor"  # TensorEntry.serializer of the reference's per-tensor format (T:serialization.py:278-310)
PER_CHANNEL_QTENSOR = "per_channel_qtensor"  # ... and of its per-channel format (T:serialization.py:366-477)
# this package's per-channel scaled float8 format: [axis: int64][fp8 body, C order][scales: float32 x C]
PER_CHANNEL_FP8 = "per_channel_fp8"
FP8_MAX = {torch.float8_e4m3fn: 448.0, torch.float8_e5m2: 57344.0}  # largest finite value of each format


class PerChannel:
    """What a per-channel quantise-on-save hook reports for a tensor: wire dtype (qint8, quint8 or a float8 format)
    and the (non-negative) axis."""

    def __init__(self, dtype: torch.dtype, axis: int) -> None:
        self.dtype, self.axis = dtype, axis


def per_channel_qparams(t: torch.Tensor, dtype: torch.dtype, axis: int) -> "tuple[torch.Tensor, torch.Tensor]":
    """The default rule of ``quantize_on_save`` per channel, computed by torch: (scales: float64, zero_points: int64)
    of ``t`` along ``axis``.  The engine computes the same on the device or host while it packs; this is what the
    ``tracing=False`` path of the hook (and the tests) use."""
    x = t.detach().float().movedim(axis, 0).reshape(t.shape[axis], -1)
    if not bool(torch.isfinite(x).all()):
        raise ValueError("per-channel quantisation: a channel holds a NaN or Inf")
    lo = x.amin(1).clamp(max=0).double()
    hi = x.amax(1).clamp(min=0).double()
    # divisors as tensors: a Python-scalar divisor is applied as a multiplication by its reciprocal on CUDA, which is
    # not the rule's (correctly rounded) division
    if dtype == torch.qint8:
        scale = torch.maximum(hi, -lo) / torch.full_like(hi, 127.0)
        zp = torch.zeros_like(scale, dtype=torch.int64)
    else:
        scale = (hi - lo) / torch.full_like(hi, 255.0)
    scale = torch.where(scale == 0, torch.ones_like(scale), scale)
    if dtype == torch.quint8:
        zp = torch.round(-lo / scale).to(torch.int64)  # round half to even, like Python's round()
    return scale, zp


def _channel_view(s: torch.Tensor, ndim: int, axis: int) -> torch.Tensor:
    shape = [1] * ndim
    shape[axis] = -1
    return s.view(shape)


def per_channel_fp8(t: torch.Tensor, dtype: torch.dtype, axis: int) -> "tuple[torch.Tensor, torch.Tensor]":
    """The scaled float8 rule of ``quantize_on_save(float8 dtype, axis=k)``, computed by torch: (q: ``dtype`` tensor of
    ``t``'s shape, scales: float32 of ``shape[axis]``).  The engine computes the same bytes on the device or host while
    it packs.  Divisions are tensor / tensor, IEEE on the CPU and on CUDA (a Python-scalar divisor would become a
    reciprocal multiplication on CUDA)."""
    fmax = FP8_MAX[dtype]
    x = t.detach().float()  # fp64 rounds to fp32 first
    flat = x.movedim(axis, 0).reshape(x.shape[axis], -1)
    if not bool(torch.isfinite(flat).all()):
        raise ValueError("per-channel quantisation: a channel holds a NaN or Inf")
    amax = flat.abs().amax(1)
    s = amax / torch.full_like(amax, fmax)
    s = torch.where(s == 0, torch.ones_like(s), s)  # all-zero channels, and amax so small that s underflows
    q = (x / _channel_view(s, x.dim(), axis)).clamp(-fmax, fmax).to(dtype)
    return q, s


def dequantize_fp8(q: torch.Tensor, scales: torch.Tensor, axis: int) -> torch.Tensor:
    """The restore half of the rule: ``q.float() * s`` in fp32; a restore converts this once to the target dtype."""
    return q.float() * _channel_view(scales.float().to(q.device), q.dim(), axis)


def quantize_on_save(dtype: torch.dtype = torch.qint8, qparams: Optional[Callable[[str, torch.Tensor], "tuple[float, int]"]] = None,
                     only: Optional[str] = None, axis: Optional[int] = None) -> Callable[[str, torch.Tensor, bool], torch.Tensor]:
    """A ``_custom_tensor_prepare_func`` that stores floating-point tensors per-tensor affine quantised
    (``torch.qint8`` / ``torch.quint8``) in the reference's self-describing per-tensor format — int_repr bytes followed
    by ``[q_scale: double][q_zero_point: int64]`` (T:serialization.py:278-310, specified and unit-tested there but
    never wired into a preparer).  The quantisation runs inside the pack kernel (``TSNAP_QINT8``/``TSNAP_QUINT8``
    wire dtype); restoring into a floating-point tensor dequantises (``tensor_copy`` semantics,
    T:io_preparers/tensor.py:385-409).

    ``qparams(logical_path, tensor) -> (scale, zero_point)``; default: symmetric abs-max scaling for qint8
    (zero_point 0), min/max affine for quint8.

    ``axis=k`` (negative counts from the end) quantises per channel along ``k`` instead, in the reference's per-channel
    format ``[axis: int64][int_repr bytes][scales: float64 x C][zero_points: int64 x C]`` (T:serialization.py:366-477),
    with the default rule applied to each channel.  It applies to floating-point tensors with ``ndim >= 2`` and
    ``ndim > k`` and at least one element; 1-d tensors (biases, norms) are stored unchanged, since 16 bytes of
    parameters per channel would outweigh them.  The engine computes the parameters while it packs; a channel
    holding a NaN or Inf fails the take.

    ``dtype`` ``torch.float8_e4m3fn`` or ``torch.float8_e5m2`` (``axis`` required) stores the same tensors as float8
    with one fp32 scale per channel (``per_channel_fp8`` states the rule), in this package's format
    ``[axis: int64][fp8 bytes][scales: float32 x C]``: a state such as Adam's ``exp_avg_sq``, whose magnitudes span
    many orders, keeps every channel in float8's range.  Float8 sources are stored unchanged, and restoring into a
    floating-point tensor dequantises on the engine; ``read_object`` gives the dequantised fp32 tensor."""
    if dtype in FP8_MAX:
        if axis is None:
            raise ValueError("quantize_on_save: float8 needs axis=k (per-channel scales); cast_on_save(dtype) stores an "
                             "unscaled float8 cast")
        if qparams is not None:
            raise ValueError("quantize_on_save: float8 per-channel scales are computed by the engine, not by qparams")
        return _quantize_per_channel_on_save(dtype, int(axis), only)
    if dtype not in (torch.qint8, torch.quint8):
        raise ValueError("quantize_on_save supports torch.qint8, torch.quint8, torch.float8_e4m3fn and torch.float8_e5m2")
    if axis is not None:
        if qparams is not None:
            raise ValueError("quantize_on_save: axis (per-channel) does not take caller-supplied qparams")
        return _quantize_per_channel_on_save(dtype, int(axis), only)
    cache: dict = {}

    def default_qparams(_path: str, t: torch.Tensor):
        tf = t.detach().float()
        if dtype == torch.qint8:
            amax = float(tf.abs().max().item()) if tf.numel() else 0.0
            return (amax / 127.0) or 1.0, 0
        lo, hi = (float(tf.min().item()), float(tf.max().item())) if tf.numel() else (0.0, 0.0)
        lo, hi = min(lo, 0.0), max(hi, 0.0)
        scale = ((hi - lo) / 255.0) or 1.0
        return scale, int(round(-lo / scale))

    def applies(logical_path: Optional[str], tensor: torch.Tensor):
        if tensor.dtype not in _FLOATS or tensor.is_quantized or tensor.numel() == 0:
            return None
        if only is not None and (logical_path is None or not fnmatch.fnmatch(logical_path, only)):
            return None
        key = (logical_path, tensor.data_ptr(), tuple(tensor.shape), tensor._version)
        if key not in cache:
            cache.clear()  # planning and staging ask about the same tensor back to back: one entry is enough
            scale, zp = (qparams or default_qparams)(logical_path or "", tensor)
            cache[key] = (dtype, float(scale), int(zp))
        return cache[key]

    def prepare(logical_path: str, tensor: torch.Tensor, tracing: bool) -> torch.Tensor:
        spec = applies(logical_path, tensor)
        if spec is None:
            return tensor
        _, scale, zp = spec
        if tracing:  # the planners (this package's and the reference's) only look at .dtype and .shape
            return _Traced(tensor.shape, dtype)
        return torch.quantize_per_tensor(tensor.detach().float(), scale, zp, dtype)

    prepare.tsnap_quant = applies  # type: ignore[attr-defined]
    return prepare


def _quantize_per_channel_on_save(dtype: torch.dtype, axis: int, only: Optional[str]):
    def applies(logical_path: Optional[str], tensor: torch.Tensor) -> Optional[PerChannel]:
        if tensor.dtype not in _FLOATS or tensor.is_quantized or tensor.numel() == 0 or tensor.dim() < 2:
            return None
        if not -tensor.dim() <= axis < tensor.dim():
            return None
        if only is not None and (logical_path is None or not fnmatch.fnmatch(logical_path, only)):
            return None
        return PerChannel(dtype, axis % tensor.dim())

    def prepare(logical_path: str, tensor: torch.Tensor, tracing: bool) -> torch.Tensor:
        spec = applies(logical_path, tensor)
        if spec is None:
            return tensor
        if tracing:
            return _Traced(tensor.shape, dtype)
        if dtype in FP8_MAX:  # what read_object gives back
            return dequantize_fp8(*per_channel_fp8(tensor, dtype, spec.axis), spec.axis)
        scales, zps = per_channel_qparams(tensor, dtype, spec.axis)
        x = tensor.detach().float()
        return torch.quantize_per_channel(x, scales.to(x.device), zps.to(x.device), spec.axis, dtype)

    prepare.tsnap_quant = applies  # type: ignore[attr-defined]
    return prepare


def fused_quant_of(func, tensor: torch.Tensor):
    """(qdtype, scale, zero_point) when ``func`` is a recognised per-tensor quantise-on-save hook for ``tensor``, a
    ``PerChannel`` when it is a per-channel one, else None."""
    args = []
    inner = func
    while isinstance(inner, functools.partial):
        args = list(inner.args) + args
        inner = inner.func
    spec = getattr(inner, "tsnap_quant", None)
    if spec is None:
        return None
    return spec(args[0] if args else None, tensor)
