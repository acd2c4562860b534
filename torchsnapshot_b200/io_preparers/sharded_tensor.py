"""ShardedTensor leg: shard subdivision on save, reshard-on-load on restore.

Reference (T:io_preparers/sharded_tensor.py): ``subdivide_shard`` (48-78) splits a local shard along
the sharding dim into pieces of at most the shard-size knob; ``prepare_read`` (197-271) intersects
every saved piece with every local shard and reads each overlapping piece once; the consumer
(310-323) narrows both sides and copies.  Here the intersection is plain box arithmetic and each
overlap becomes ONE strided copy descriptor for the scatter kernel — the saved piece is never
materialised as a tensor."""
from __future__ import annotations

import asyncio
import math
from concurrent.futures import Executor
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple, Union

import torch
from torch.distributed._shard.sharded_tensor import Shard as ShardedTensorShard, ShardedTensor, ShardMetadata
from torch.distributed._shard.sharding_spec import ChunkShardingSpec

from .. import _native
from ..io_types import BufferConsumer, Future, ReadReq, WriteReq
from ..knobs import get_max_shard_size_bytes
from ..manifest import Shard, ShardedTensorEntry, TensorEntry
from ..native_plan import RAW, describe_consumer, entry_nbytes, raw_castable
from ..serialization import dtype_to_element_size, string_to_dtype
from .tensor import PICKLED, PrepareFunc, TensorBufferConsumer, TensorIOPreparer, engine_for, tensor_copy

Box = Tuple[List[int], List[int]]  # (offsets, sizes) in global coordinates


def boxes_overlap(a_off: Sequence[int], a_sz: Sequence[int], b_off: Sequence[int], b_sz: Sequence[int]) -> bool:
    """Non-empty intersection of two axis-aligned boxes (what torch's
    _check_shard_metadata_pair_overlap decides for T:io_preparers/sharded_tensor.py:239)."""
    if len(a_off) != len(b_off):
        return False
    for ao, asz, bo, bsz in zip(a_off, a_sz, b_off, b_sz):
        if ao >= bo + bsz or bo >= ao + asz:
            return False
    return True


def overlap_narrows(saved: Box, current: Box) -> List[Tuple[int, int, int, int]]:
    """Per dim ``(dim, offset in saved piece, offset in current shard, length)`` of the intersection
    (T:io_preparers/sharded_tensor.py:80-127)."""
    out = []
    for d, (so, ss, co, cs) in enumerate(zip(saved[0], saved[1], current[0], current[1])):
        lo = max(so, co)
        hi = min(so + ss, co + cs)
        out.append((d, lo - so, lo - co, hi - lo))
    return out


@dataclass
class _OverlappingRegion:
    dst_tensor: torch.Tensor
    overlap_region: List[Tuple[int, int, int, int]]  # (dim, src_offset, dst_offset, length)

    def get_views(self, src_tensor: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        s, d = src_tensor, self.dst_tensor
        for dim, so, do, n in self.overlap_region:
            s = s.narrow(dim, so, n)
            d = d.narrow(dim, do, n)
        return s, d


class ShardedTensorBufferConsumer(BufferConsumer):
    def __init__(self, overlapping_regions: List[_OverlappingRegion], entry: TensorEntry, wire_skip: int = 0, wire_len: Optional[int] = None) -> None:
        self.overlapping_regions = overlapping_regions
        self.entry = entry
        # the buffer handed to this consumer starts `wire_skip` bytes into the saved piece and is `wire_len` bytes
        # long (the hull of the bytes the regions need); 0 / None = the whole piece, as in the reference
        self.wire_skip = wire_skip
        self.wire_len = wire_len

    def is_raw(self) -> bool:
        if self.entry.serializer != RAW:
            return False
        src = string_to_dtype(self.entry.dtype)
        return all(raw_castable(src, r.dst_tensor.dtype) for r in self.overlapping_regions)

    async def consume_buffer(self, buf: bytes, executor: Optional[Executor] = None) -> None:
        def work() -> None:
            described = describe_consumer(self, buf=buf)
            if described is not None:
                if described[0]:
                    engine_for(self.overlapping_regions[0].dst_tensor).consume(buf, described[0])
                return
            if self.wire_skip or self.wire_len is not None:
                raise AssertionError("partial reads are only planned for raw entries")
            saved = TensorBufferConsumer.deserialize_tensor(buf, self.entry)
            for region in self.overlapping_regions:
                s, d = region.get_views(saved)
                tensor_copy(d, s)

        if executor is not None:
            await asyncio.get_running_loop().run_in_executor(executor, work)
        else:
            work()

    def get_consuming_cost_bytes(self) -> int:
        n = entry_nbytes(self.entry) if self.wire_len is None else self.wire_len
        return 2 * n if self.entry.serializer == PICKLED else n


def needed_hull(entry: TensorEntry, regions: List[_OverlappingRegion]) -> Optional[Tuple[int, int]]:
    """Byte hull [lo, hi) inside the saved piece that the overlap regions touch, or None when the whole piece is
    needed (or the piece is not a raw image).  The reference always reads whole pieces (T:io_preparers/
    sharded_tensor.py:252-270: "read each persisted shard once"), which amplifies reads whenever a local shard only
    needs a few rows of a 512 MiB piece; reading the hull is the cheap half of SURVEY.md's N3."""
    if entry.serializer != RAW:
        return None
    shape = list(entry.shape)
    esz = dtype_to_element_size(string_to_dtype(entry.dtype))
    strides = _native._c_strides(shape)
    lo, hi = None, None
    for r in regions:
        first = sum(so * strides[d] for d, so, _, _ in r.overlap_region)
        last = first + sum((n - 1) * strides[d] for d, _, _, n in r.overlap_region)
        lo = first if lo is None else min(lo, first)
        hi = last + 1 if hi is None else max(hi, last + 1)
    if lo is None:
        return None
    total = 1
    for s_ in shape:
        total *= s_
    if lo == 0 and hi == total:
        return None
    return lo * esz, hi * esz


def overlap_read_reqs(shards: List[Shard], local: List[Tuple[torch.Tensor, List[int], List[int]]]) -> List[ReadReq]:
    """One ReadReq per saved piece that intersects any local shard; piece order is preserved."""
    reqs: List[ReadReq] = []
    for piece in shards:
        regions = [
            _OverlappingRegion(t, overlap_narrows((piece.offsets, piece.sizes), (off, sz)))
            for t, off, sz in local
            if boxes_overlap(piece.offsets, piece.sizes, off, sz)
        ]
        if not regions:
            continue
        consumer = ShardedTensorBufferConsumer(regions, piece.tensor)
        byte_range = piece.tensor.byte_range_tuple
        hull = needed_hull(piece.tensor, regions) if consumer.is_raw() else None
        if hull is not None:
            base = byte_range[0] if byte_range is not None else 0
            consumer.wire_skip, consumer.wire_len = hull[0], hull[1] - hull[0]
            byte_range = (base + hull[0], base + hull[1])
        reqs.append(ReadReq(path=piece.tensor.location, buffer_consumer=consumer, byte_range=byte_range))
    return reqs


class ShardedTensorIOPreparer:
    @staticmethod
    def subdivide_shard(
        shard: torch.Tensor, offsets: List[int], sizes: List[int], dim: int, max_shard_sz_bytes: int
    ) -> List[Tuple[torch.Tensor, List[int], List[int]]]:
        if max_shard_sz_bytes <= 0:
            raise ValueError(f"max_shard_sz_bytes must be a positive integer (got {max_shard_sz_bytes}).")
        numel = 1
        for s in sizes:
            numel *= s
        slice_bytes = numel // sizes[dim] * shard.element_size()
        rows_per_piece = max(math.floor(max_shard_sz_bytes / slice_bytes), 1)
        pieces = []
        for lo in range(0, sizes[dim], rows_per_piece):
            n = min(rows_per_piece, sizes[dim] - lo)
            p_off, p_sz = list(offsets), list(sizes)
            p_off[dim] += lo
            p_sz[dim] = n
            pieces.append((shard.narrow(dim, lo, n), p_off, p_sz))
        return pieces

    @staticmethod
    def _shards_get_overlap_region_wrt_saved_tensor(saved_shard: ShardMetadata, current_shard: ShardMetadata):
        return overlap_narrows(
            (list(saved_shard.shard_offsets), list(saved_shard.shard_sizes)),
            (list(current_shard.shard_offsets), list(current_shard.shard_sizes)),
        )

    @classmethod
    def prepare_write(
        cls,
        storage_path: str,
        obj: ShardedTensor,
        is_async_snapshot: bool = False,
        _tensor_prepare_func: Optional[PrepareFunc] = None,
    ) -> Tuple[ShardedTensorEntry, List[WriteReq]]:
        spec = obj.sharding_spec()
        dim = spec.dim if isinstance(spec, ChunkShardingSpec) else 0
        shards: List[Shard] = []
        reqs: List[WriteReq] = []
        for local in obj.local_shards():
            for view, off, sz in cls.subdivide_shard(
                local.tensor, list(local.metadata.shard_offsets), list(local.metadata.shard_sizes), dim, get_max_shard_size_bytes()
            ):
                tag = "_".join(str(i) for i in off)
                e, wr = TensorIOPreparer.prepare_write(f"{storage_path}_{tag}", view, is_async_snapshot, _tensor_prepare_func)
                reqs.extend(wr)
                shards.append(Shard(offsets=off, sizes=sz, tensor=e))
        return ShardedTensorEntry(shards=shards), reqs

    @staticmethod
    def _get_global_shape(entry: ShardedTensorEntry) -> List[int]:
        shape = [0] * len(entry.shards[0].sizes)
        for sh in entry.shards:
            for d, (o, s) in enumerate(zip(sh.offsets, sh.sizes)):
                shape[d] = max(shape[d], o + s)
        return shape

    @classmethod
    def prepare_read(
        cls, entry: ShardedTensorEntry, obj_out: Optional[Union[ShardedTensor, torch.Tensor]] = None
    ) -> Tuple[List[ReadReq], Future[Union[ShardedTensor, torch.Tensor]]]:
        if obj_out is None:
            # no runtime object: materialise the full tensor on the host (T:io_preparers/sharded_tensor.py:273-282)
            obj_out = torch.empty(entry.get_tensor_shape(), dtype=string_to_dtype(entry.shards[0].tensor.dtype))
        if type(obj_out) is ShardedTensor:
            local = [(s.tensor, list(s.metadata.shard_offsets), list(s.metadata.shard_sizes)) for s in obj_out.local_shards()]
        elif type(obj_out) is torch.Tensor or isinstance(obj_out, torch.nn.Parameter):
            local = [(obj_out, [0] * obj_out.dim(), list(obj_out.shape))]
        else:
            raise RuntimeError(f"obj_out must either be a Tensor or ShardedTensor (got {type(obj_out)})")
        return overlap_read_reqs(entry.shards, local), Future(obj=obj_out)

    @staticmethod
    def empty_tensor_from_sharded_tensor_entry(entry: ShardedTensorEntry) -> torch.Tensor:
        return torch.empty(entry.get_tensor_shape(), dtype=string_to_dtype(entry.shards[0].tensor.dtype))
