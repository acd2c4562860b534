"""Adversarial inputs for the converting and quantising copy paths, and the layouts they are placed in.

Plain torch only: the host and device conversion tests share these cases and compute every expectation with torch,
on the device the engine ran on.  Values are chosen where conversions go wrong: rounding ties at both parities and one
source ulp either side of them, double-rounding cases of fp64 sources, overflow thresholds, subnormals, signed zeros,
infinities and NaNs; the quantisers get values at and a few fp32 ulps around (k + 1/2) * scale.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, List, Optional, Tuple

import torch

from tests.util import det_tensor

FLOATS = [torch.float64, torch.float32, torch.float16, torch.bfloat16]
PAIRS = [(s, d) for s in FLOATS for d in FLOATS if s != d]

_FMT = {torch.float16: (5, 10), torch.bfloat16: (8, 7), torch.float32: (8, 23), torch.float64: (11, 52)}  # exponent, mantissa bits
_BITS = {torch.float16: torch.int16, torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}


def _from_bits(dt: torch.dtype, bits: List[int]) -> torch.Tensor:
    """fp64 values of non-negative bit patterns of `dt`."""
    return torch.tensor(bits, dtype=_BITS[dt]).view(dt).to(torch.float64)


def _max_finite_bits(dt: torch.dtype) -> int:
    e, m = _FMT[dt]
    return (((1 << e) - 2) << m) | ((1 << m) - 1)


def _grid(dt: torch.dtype) -> List[int]:
    """Bit patterns of positive finite values of `dt`: both mantissa parities at the bottom and top of the subnormal and
    normal ranges and mid-range, up to the largest finite value."""
    e, m = _FMT[dt]
    emax = (1 << e) - 2
    exps = sorted({0, 1, 2, emax // 2, emax // 2 + 1, emax - 1, emax})
    return [(x << m) | f for x in exps for f in (0, 1, 2, 3, (1 << m) - 2, (1 << m) - 1)]


def _ulp32(x: float) -> float:
    """Spacing of fp32 around |x| (x finite, not 0)."""
    _, ex = math.frexp(abs(x))
    return max(2.0 ** (ex - 24), 2.0 ** -149)


def _src_neighbours(x: torch.Tensor, src: torch.dtype) -> torch.Tensor:
    """x rounded to `src`, and the `src` values one ulp below and above it (fp64)."""
    s = x.to(src)
    b = s.view(_BITS[src])
    return torch.cat([s.to(torch.float64), (b + 1).view(src).to(torch.float64), (b - 1).view(src).to(torch.float64)])


# fp64 values whose fp32 rounding lands exactly on a 16-bit tie, so rounding once and rounding through fp32 differ: just
# above a rounding tie, just above the underflow tie, just below the overflow threshold
DOUBLE_ROUNDING = {
    torch.float16: [1 + 2**-11 + 2**-40, 2.0**-25 + 2**-60, 65519.99999, -65519.99999],
    torch.bfloat16: [1 + 2**-8 + 2**-40, 2.0**-134 + 2**-160, (2 - 2**-8) * 2.0**127 - 2.0**90, -((2 - 2**-8) * 2.0**127 - 2.0**90)],
}


def edge_values(src: torch.dtype, dst: torch.dtype) -> torch.Tensor:
    """Deterministic 1-D fp64 tensor of values representable in `src` where converting to `dst` is hard."""
    vals: List[torch.Tensor] = [torch.tensor(DOUBLE_ROUNDING.get(dst, []), dtype=torch.float64)]
    nan = torch.tensor([0x7FF8000000000000, -0x0008000000000000], dtype=torch.int64).view(torch.float64)  # +NaN, -NaN
    vals.append(torch.cat([torch.tensor([0.0, -0.0, math.inf, -math.inf], dtype=torch.float64), nan]))
    for dt in (src, dst):  # smallest / largest subnormal and normal, largest finite
        m = _FMT[dt][1]
        vals.append(_from_bits(dt, [1, (1 << m) - 1, 1 << m, ((1 << m) + 1), _max_finite_bits(dt)]))
    if dst != torch.float64:
        g = _grid(dst)
        lo = _from_bits(dst, g)
        top = _max_finite_bits(dst)
        # the next value up; past the largest finite value that is the overflow threshold's other side
        hi = torch.where(torch.tensor(g) == top, 2 * lo - _from_bits(dst, [p - 1 if p == top else p for p in g]), _from_bits(dst, [min(p + 1, top) for p in g]))
        mid = (lo + hi) / 2  # exact halfway points (fp64 holds them), including the underflow ties (0, min subnormal)
        vals += [lo, _src_neighbours(mid, src)]
        ulp = torch.tensor([_ulp32(float(x)) for x in mid], dtype=torch.float64)
        vals.append(torch.cat([mid + ulp / 4, mid - ulp / 4]))  # fp32 rounds these to the tie: the double-rounding cases
    out = torch.cat(vals)
    out = torch.cat([out, -out])
    return out.to(src).to(torch.float64)


def case_values(src: torch.dtype, dst: torch.dtype, numel: int, seed: int = 1) -> torch.Tensor:
    """`numel` elements of `src` (1-D): det_tensor bit patterns, which span every exponent, with edge_values at both ends
    (so that they also land in ragged tails).  A single element is the first edge value."""
    out = det_tensor((numel,), src, seed)
    e = edge_values(src, dst).to(src)
    k = min(len(e), numel)
    out[numel - k :] = e.flip(0)[:k]
    out[:k] = e[:k]
    return out


def tie_values(scale: float, zp: int, qdtype: torch.dtype) -> torch.Tensor:
    """fp32 inputs of an affine quantiser with (scale, zp): (k + 1/2) * scale rounded to fp32 for every k whose tie lies
    in or next to the integer range, +-1..8 fp32 ulps around each, values past the clamp range, and -0.0."""
    qmin, qmax = (-128, 127) if qdtype == torch.qint8 else (0, 255)
    k = torch.arange(qmin - zp - 1, qmax - zp + 1, dtype=torch.float64)
    ties = ((k + 0.5) * scale).float()
    bits = ties.view(torch.int32)
    near = [(bits + d).view(torch.float32) for d in range(-8, 9) if d]
    past = torch.tensor([qmin - zp - 3, qmax - zp + 3, qmin - zp - 1000, qmax - zp + 1000], dtype=torch.float64) * scale
    return torch.cat([ties, *near, past.float(), torch.tensor([-0.0])])


# (lo, hi) channel ranges whose quint8 zero point -lo / ((hi - lo) / 255) is exactly j + 1/2 in double, j even and odd
HALF_ZERO_POINT_RANGES = [(-1.0, 1.0), (-1.0, 5.0), (-1.0, 9.0), (-1.0, 29.0), (-1.0, 33.0), (-1.0, 101.0), (-3.0, 7.0), (-3.0, 31.0), (-5.0, 1.0)]


def tie_channels(channels: int, length: int, qdtype: torch.dtype) -> torch.Tensor:
    """fp32 [channels, length]: every element at, or a few fp32 ulps from, (k + 1/2) * scale for the scale the default
    rule gives the channel.  Element 0 (and 1 for quint8) sets the channel's range; odd qint8 channels have a negative
    extreme; every third quint8 channel has a range whose zero point is an exact .5."""
    c = torch.arange(channels, dtype=torch.float64)[:, None]
    j = torch.arange(length, dtype=torch.float64)[None, :]
    a = ((0.3 + 0.0137 * (c % 101)) * torch.pow(2.0, (c % 7) - 3)).float().double()  # channel extremes, fp32 values
    if qdtype == torch.qint8:
        scale = a / 127.0
        k = (j * 37 + c * 11) % 253 - 126  # ties inside [-a, a]
        x = ((k + 0.5) * scale).float()
    else:
        idx = (c.long() % len(HALF_ZERO_POINT_RANGES)).squeeze(1)
        r = torch.tensor(HALF_ZERO_POINT_RANGES, dtype=torch.float64)[idx] * torch.pow(2.0, (c % 5) - 2)
        lo = torch.where(c % 3 == 0, r[:, :1], -a * (0.2 + 0.05 * (c % 9)))
        hi = torch.where(c % 3 == 0, r[:, 1:], a)
        lo, hi = lo.float().double(), hi.float().double()
        scale = (hi - lo) / 255.0
        zp = torch.round(-lo / scale)
        k = (j * 37 + c * 11) % 255
        x = torch.minimum(torch.maximum((k - zp + 0.5) * scale, lo), hi).float()
    d = ((j * 5 + c * 3) % 17 - 8).to(torch.int32)  # -8..8 fp32 ulps
    x = (x.view(torch.int32) + d).view(torch.float32)
    if qdtype == torch.qint8:
        x[:, 0] = torch.where(c[:, 0] % 2 == 1, -a[:, 0], a[:, 0]).float()
        x[:, 1:] = x[:, 1:].clamp(-a.float(), a.float())
    else:
        x[:, 0], x[:, 1] = lo[:, 0].float(), hi[:, 0].float()
        x[:, 2:] = torch.minimum(torch.maximum(x[:, 2:], lo.float()), hi.float())
    return x


# ---- layouts -------------------------------------------------------------------------------------------------------
_DENSE = 3 * 65536 + 4096  # >= 3 LSU tiles (128 KiB of destination bytes) for every destination dtype; a multiple of 8


@dataclass(frozen=True)
class Layout:
    """Where a converting member sits: `cut` turns a 1-D tensor of `storage` elements into the view the engine reads
    (save) or writes (restore), `offset` is the member's wire offset.  `piece` = (shape, box) makes a restore a reshard
    sub-box: the wire holds a piece of `shape` and the view receives `piece[box]`."""

    name: str
    storage: int
    cut: Callable[[torch.Tensor], torch.Tensor]
    offset: int = 0
    piece: Optional[Tuple[Tuple[int, ...], Tuple[slice, ...]]] = None


LAYOUTS = [Layout(f"dense_mod8_{r}", _DENSE + r, lambda s: s) for r in range(8)] + [
    Layout("transposed", 67 * 61, lambda s: s.view(67, 61).t()),
    Layout("narrowed", 53 * 97, lambda s: s.view(53, 97)[2:51, 3:90]),
    Layout("zero_dim", 1, lambda s: s[0]),
    Layout("odd_offset", 70001, lambda s: s, offset=3),
    Layout("odd_offset_strided", 53 * 97, lambda s: s.view(53, 97)[:, 5:70].t(), offset=5),
    Layout("subbox", 30 * 60, lambda s: s.view(30, 60)[3:27, 10:55], piece=((40, 67), (slice(7, 31), slice(5, 50)))),
    Layout("subbox_odd_offset", 30 * 60, lambda s: s.view(30, 60)[3:27, 10:55], offset=7, piece=((40, 67), (slice(7, 31), slice(5, 50)))),
]
SAVE_LAYOUTS = [l for l in LAYOUTS if l.piece is None]  # a save always writes a whole piece


def _c_strides(shape) -> List[int]:
    acc, out = 1, []
    for n in reversed(shape):
        out.append(acc)
        acc *= n
    return out[::-1]


@dataclass
class SaveCase:
    view: torch.Tensor      # source view (src dtype)
    offset: int             # wire offset of the member
    expected: torch.Tensor  # its wire elements (dst dtype, 1-D), converted by torch on the view's device


def save_case(layout: Layout, src: torch.dtype, dst: torch.dtype, device) -> SaveCase:
    view = layout.cut(case_values(src, dst, layout.storage).to(device))
    return SaveCase(view, layout.offset, view.to(dst).reshape(-1))


@dataclass
class RestoreCase:
    storage: torch.Tensor      # the target's whole storage (dst dtype, 1-D, pre-filled with other bits)
    view: torch.Tensor         # the target view cut from it
    wire: torch.Tensor         # the wire image (uint8): `layout.offset` filler bytes, then the saved piece (src dtype)
    desc_offset: int           # wire offset of the view's first element
    wire_strides: Optional[List[int]]
    expected: torch.Tensor     # `storage` after view.copy_(saved values), by torch on the same device


def restore_case(layout: Layout, src: torch.dtype, dst: torch.dtype, device) -> RestoreCase:
    storage = det_tensor((layout.storage,), dst, 99).to(device)
    view = layout.cut(storage)
    if layout.piece is None:
        piece = case_values(src, dst, max(1, view.numel())).to(device).reshape(view.shape)
        vals, first, strides = piece, 0, None
    else:
        shape, box = layout.piece
        numel = math.prod(shape)
        piece = case_values(src, dst, numel).to(device).reshape(shape)
        vals = piece[box]
        first, strides = vals.storage_offset(), _c_strides(shape)
    expected = storage.clone()
    layout.cut(expected).copy_(vals)
    filler = torch.full((layout.offset,), 0xA5, dtype=torch.uint8, device=device)
    wire = torch.cat([filler, piece.contiguous().reshape(-1).view(torch.uint8)])
    es = torch.empty(0, dtype=src).element_size()
    return RestoreCase(storage, view, wire, layout.offset + first * es, strides, expected)


def same_values(got: torch.Tensor, want: torch.Tensor, nan_bits: bool) -> Optional[str]:
    """None when equal bit for bit; with nan_bits=False NaNs only have to sit at the same positions.  Else a message
    naming the first differing elements."""
    g, w = got.reshape(-1), want.reshape(-1)
    assert g.dtype == w.dtype and g.numel() == w.numel()
    it = _BITS[g.dtype]
    gb, wb = g.view(it), w.view(it)
    if nan_bits:
        bad = gb != wb
    else:
        gn, wn = g.isnan(), w.isnan()
        bad = (gn != wn) | (~gn & ~wn & (gb != wb))
    if not bool(bad.any()):
        return None
    idx = bad.nonzero().reshape(-1)[:5].tolist()
    mask = (1 << (8 * g.element_size())) - 1
    return f"{int(bad.sum())} of {g.numel()} elements differ, e.g. " + ", ".join(
        f"[{i}] got {int(gb[i]) & mask:#x} want {int(wb[i]) & mask:#x}" for i in idx)
