"""Adversarial inputs for conversions with a float8 side (torch.float8_e4m3fn / torch.float8_e5m2), in the layouts of
tests/conversion_cases.py.

The float8 formats are not IEEE-shaped throughout (e4m3fn's top exponent holds finite values and it has no infinity),
so their edge values come from their own generator: every float8 pattern, every rounding tie of a float8 destination
with the source values one ulp either side and the fp64 values a quarter fp32 ulp either side (the double-rounding
cases), the overflow and underflow thresholds, signed zeros, infinities and NaNs.  Plain torch only: every expectation
is computed by torch on the device the engine ran on.
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch

from tests.conversion_cases import FLOATS, Layout, RestoreCase, SaveCase, _c_strides, _ulp32
from tests.util import det_tensor

FP8 = [torch.float8_e4m3fn, torch.float8_e5m2]
# every ordered pair of the six floats with a float8 side
FP8_PAIRS = [(s, d) for s in FLOATS + FP8 for d in FLOATS + FP8 if s != d and (s in FP8 or d in FP8)]

_BITS = {torch.float16: torch.int16, torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64,
         torch.float8_e4m3fn: torch.int8, torch.float8_e5m2: torch.int8}
# largest finite value, the overflow tie above it, the exponent of the smallest subnormal
_FMT = {torch.float8_e4m3fn: (448.0, 464.0, -9), torch.float8_e5m2: (57344.0, 61440.0, -16)}

# fp64 values that fp32 rounds onto a float8 tie, so rounding once and rounding through fp32 differ: 1 + 2^-4 is the
# tie between 1 and 1 + 2^-3 (e4m3fn), 1 + 2^-3 the one between 1 and 1 + 2^-2 (e5m2); just below the overflow ties;
# just above the underflow ties
DOUBLE_ROUNDING = {
    torch.float8_e4m3fn: [1 + 2**-4 + 2**-30, 464 - 2**-30, 2.0**-10 + 2**-40, 1.5 * 2.0**-10 + 2**-40],
    torch.float8_e5m2: [1 + 2**-3 + 2**-30, 61440 - 2**-30, 2.0**-17 + 2**-40, 1.5 * 2.0**-17 + 2**-40],
}


def every_pattern(dt: torch.dtype) -> torch.Tensor:
    """The 256 values of a float8 dtype, in bit-pattern order."""
    return torch.arange(256, dtype=torch.int32).to(torch.uint8).view(dt)


def _src_neighbours(x: torch.Tensor, src: torch.dtype) -> torch.Tensor:
    """x rounded to `src`, and the `src` values one ulp below and above it (fp64)."""
    s = x.to(src)
    b = s.view(_BITS[src])
    return torch.cat([s.to(torch.float64), (b + 1).view(src).to(torch.float64), (b - 1).view(src).to(torch.float64)])


def edge_values(src: torch.dtype, dst: torch.dtype) -> torch.Tensor:
    """Deterministic 1-D fp64 tensor of values representable in `src` where converting to `dst` is hard."""
    nan = torch.tensor([0x7FF8000000000000, -0x0008000000000000], dtype=torch.int64).view(torch.float64)
    vals: List[torch.Tensor] = [torch.cat([torch.tensor([0.0, -0.0, math.inf, -math.inf], dtype=torch.float64), nan])]
    for dt in (d for d in FP8 if d in (src, dst)):
        vals.append(every_pattern(dt).to(torch.float64))
    if dst in FP8:
        top, tie, sub = _FMT[dst]
        grid = every_pattern(dst)[:128].to(torch.float64)
        grid = torch.cat([grid[grid.isfinite() & (grid <= top)], torch.tensor([2 * tie - top], dtype=torch.float64)])
        mid = (grid[1:] + grid[:-1]) / 2  # exact in fp64: the ties, from half the smallest subnormal up to `tie`
        ulp = torch.tensor([_ulp32(float(x)) for x in mid], dtype=torch.float64)
        vals += [_src_neighbours(mid, src), mid + ulp / 4, mid - ulp / 4]
        vals.append(torch.tensor([top, tie, 2 * tie - top, 1e30, 2.0 ** (sub - 1), 1.5 * 2.0 ** (sub - 1), 2.0 ** (sub - 2)], dtype=torch.float64))
        vals.append(torch.tensor(DOUBLE_ROUNDING[dst], dtype=torch.float64))
    out = torch.cat(vals)
    out = torch.cat([out, -out])
    return out.to(src).to(torch.float64)


def case_values(src: torch.dtype, dst: torch.dtype, numel: int, seed: int = 1) -> torch.Tensor:
    """`numel` elements of `src` (1-D): det_tensor bit patterns with edge_values at both ends (so that they also land in
    ragged tails).  A single element is the first edge value."""
    out = det_tensor((numel,), src, seed)
    e = edge_values(src, dst).to(src)
    k = min(len(e), numel)
    out[numel - k :] = e.view(_BITS[src]).flip(0).view(src)[:k]  # flipped as bits: torch has no float8 flip
    out[:k] = e[:k]
    return out


def save_case(layout: Layout, src: torch.dtype, dst: torch.dtype, device) -> SaveCase:
    view = layout.cut(case_values(src, dst, layout.storage).to(device))
    return SaveCase(view, layout.offset, view.to(dst).reshape(-1))


def restore_case(layout: Layout, src: torch.dtype, dst: torch.dtype, device) -> RestoreCase:
    storage = det_tensor((layout.storage,), dst, 99).to(device)
    view = layout.cut(storage)
    if layout.piece is None:
        piece = case_values(src, dst, max(1, view.numel())).to(device).reshape(view.shape)
        vals, first, strides = piece, 0, None
    else:
        shape, box = layout.piece
        piece = case_values(src, dst, math.prod(shape)).to(device).reshape(shape)
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
        # torch has no isnan for float8 on every device: compare as fp32, which keeps NaN-ness
        gn, wn = g.float().isnan(), w.float().isnan()
        bad = (gn != wn) | (~gn & ~wn & (gb != wb))
    if not bool(bad.any()):
        return None
    idx = bad.nonzero().reshape(-1)[:5].tolist()
    mask = (1 << (8 * g.element_size())) - 1
    return f"{int(bad.sum())} of {g.numel()} elements differ, e.g. " + ", ".join(
        f"[{i}] got {int(gb[i]) & mask:#x} want {int(wb[i]) & mask:#x}" for i in idx)
