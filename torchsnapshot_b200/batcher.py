"""Slab batching of small raw tensors.

Slab *assignment* must reproduce the reference bit for bit, because it decides ``location`` and
``byte_range`` of every TensorEntry in the manifest (T:batcher.py:204-355): requests are visited in
order; only raw (buffer_protocol, no prepare func) tensors strictly smaller than the threshold are
batchable; CPU and GPU tensors fill separate slab lists; a new slab is opened when
``current + size >= threshold``; members sit back to back, no padding.

Slab *staging* is where the implementations part ways.  The reference allocates a byte tensor per slab
and issues one D2D copy per member plus a blocking pageable ``.cpu()`` (T:batcher.py:144-159).  Here a
slab is just a list of copy descriptors handed to the engine: all slabs of a snapshot are packed by
one kernel launch into the HBM arena and drained through the pinned ring."""
from __future__ import annotations

import asyncio
import os
import uuid
from collections import defaultdict
from concurrent.futures import Executor
from typing import Dict, List, Optional, Tuple

from .io_preparers.tensor import TensorBufferStager, current_stream_of, engine_for
from .io_types import BufferConsumer, BufferStager, BufferType, ReadReq, WriteReq
from .knobs import get_slab_size_threshold_bytes
from .manifest import ChunkedTensorEntry, DTensorEntry, Entry, ShardedTensorEntry, TensorEntry
from .native_plan import describe_stager
from .serialization import Serializer

ByteRange = Tuple[int, int]


def is_batchable(buffer_stager: BufferStager) -> bool:
    return (
        isinstance(buffer_stager, TensorBufferStager)
        and buffer_stager.entry.serializer == Serializer.BUFFER_PROTOCOL.value
        and buffer_stager._tensor_prepare_func is None
    )


class BatchedBufferStager(BufferStager):
    """A slab: raw tensor members at consecutive byte ranges of one storage object."""

    def __init__(self, byte_range_to_buffer_stager: Dict[ByteRange, BufferStager]) -> None:
        end = 0
        for lo, hi in byte_range_to_buffer_stager:
            if lo != end:
                raise AssertionError("The byte ranges are not consecutive.")
            end = hi
        self.byte_range_to_buffer_stager = byte_range_to_buffer_stager
        self.slab_sz_bytes: int = end

    def is_raw(self) -> bool:
        return all(isinstance(s, TensorBufferStager) and s.is_raw() for s in self.byte_range_to_buffer_stager.values())

    async def stage_buffer(self, executor: Optional[Executor] = None) -> BufferType:
        described = describe_stager(self)
        if described is None:
            raise AssertionError("a slab member is not a raw tensor that fills its byte range")
        descs, keep, _ = described
        if not descs:
            return memoryview(bytes(self.slab_sz_bytes))
        if len({(t.device.type, t.device.index) for t in keep if t.is_cuda}) > 1:
            # members on several GPUs of this process (the slab assignment keys on is_cuda only, T:batcher.py:300-303):
            # every member is staged by the engine of its own device, the slab is assembled on the host
            slab = bytearray(self.slab_sz_bytes)
            for (lo, hi), stager in self.byte_range_to_buffer_stager.items():
                if hi > lo:
                    slab[lo:hi] = await stager.stage_buffer(executor)
            return memoryview(slab)
        staged = engine_for(keep[0]).stage(descs, self.slab_sz_bytes, stream=current_stream_of(keep[0]), keepalive=keep)
        if executor is not None:
            return await asyncio.get_running_loop().run_in_executor(executor, staged.wait)
        return staged.wait()

    def get_staging_cost_bytes(self) -> int:
        return self.slab_sz_bytes


class GPUBatchedBufferStager(BatchedBufferStager):
    """Slab whose members all live on the GPU (same admission checks as T:batcher.py:119-142)."""

    def __init__(self, byte_range_to_buffer_stager: Dict[ByteRange, BufferStager]) -> None:
        super().__init__(byte_range_to_buffer_stager)
        for stager in byte_range_to_buffer_stager.values():
            if not isinstance(stager, TensorBufferStager):
                raise AssertionError(f"GPUBatchedBufferStager only supports TensorBufferStagers (got {type(stager)}).")
            if not is_batchable(stager):
                raise AssertionError(f"GPUBatchedBufferStager only supports batchable entries (got {stager.entry}).")
            if not stager.tensor.is_cuda:
                raise AssertionError("GPUBatchedBufferStager only supports GPU tensors.")


class _Slab:
    def __init__(self, on_gpu: bool) -> None:
        self.on_gpu = on_gpu
        self.members: Dict[ByteRange, BufferStager] = {}
        self.location = os.path.join("batched", str(uuid.uuid4()))
        self.sz_bytes = 0

    def add(self, nbytes: int, stager: BufferStager) -> ByteRange:
        br = (self.sz_bytes, self.sz_bytes + nbytes)
        self.members[br] = stager
        self.sz_bytes += nbytes
        return br

    def build(self) -> BufferStager:
        return (GPUBatchedBufferStager if self.on_gpu else BatchedBufferStager)(self.members)


def _leaf_tensor_entries(entries: List[Entry]) -> Dict[str, TensorEntry]:
    out: Dict[str, TensorEntry] = {}
    for e in entries:
        if isinstance(e, TensorEntry):
            out[e.location] = e
        elif isinstance(e, ChunkedTensorEntry):
            out.update((c.tensor.location, c.tensor) for c in e.chunks)
        elif isinstance(e, (ShardedTensorEntry, DTensorEntry)):
            out.update((s.tensor.location, s.tensor) for s in e.shards)
    return out


def batch_write_requests(
    entries: List[Entry], write_reqs: List[WriteReq], slab_size_threshold_bytes: Optional[int] = None
) -> Tuple[List[Entry], List[WriteReq]]:
    """Returns (entries, batched write requests); relocates the affected TensorEntrys in place."""
    threshold = slab_size_threshold_bytes or get_slab_size_threshold_bytes()
    passthrough: List[WriteReq] = []
    slabs: Dict[bool, List[_Slab]] = {False: [_Slab(False)], True: [_Slab(True)]}
    moved: Dict[str, Tuple[str, int, int]] = {}
    for wr in write_reqs:
        stager = wr.buffer_stager
        if not is_batchable(stager):
            passthrough.append(wr)
            continue
        t = stager.tensor
        nbytes = t.nelement() * t.element_size()
        if nbytes >= threshold:
            passthrough.append(wr)
            continue
        chain = slabs[bool(t.is_cuda)]
        if chain[-1].sz_bytes + nbytes >= threshold:
            chain.append(_Slab(bool(t.is_cuda)))
        lo, hi = chain[-1].add(nbytes, stager)
        moved[wr.path] = (chain[-1].location, lo, hi)
    out = list(passthrough)
    for slab in slabs[False] + slabs[True]:
        if slab.members:
            out.append(WriteReq(path=slab.location, buffer_stager=slab.build()))
    leaves = _leaf_tensor_entries(entries)
    for old, (new, lo, hi) in moved.items():
        if old not in leaves:
            raise RuntimeError(f"The tensor entry with the location {old} is not passed to batch_write.")
        leaves[old].location = new
        leaves[old].byte_range = [lo, hi]
    return entries, out


class BatchedBufferConsumer(BufferConsumer):
    """Several ranged reads of one file merged into a single read (T:batcher.py:358-384)."""

    def __init__(self, byte_range_to_buffer_consumer: Dict[ByteRange, BufferConsumer], buf_sz_bytes: int) -> None:
        self.byte_range_to_buffer_consumer = byte_range_to_buffer_consumer
        self.buf_sz_bytes = buf_sz_bytes

    def is_raw(self) -> bool:
        return all(getattr(c, "is_raw", lambda: False)() for c in self.byte_range_to_buffer_consumer.values())

    async def consume_buffer(self, buf: bytes, executor: Optional[Executor] = None) -> None:
        view = memoryview(buf)
        tasks = [
            asyncio.ensure_future(consumer.consume_buffer(view[lo:hi], executor))
            for (lo, hi), consumer in self.byte_range_to_buffer_consumer.items()
        ]
        if tasks:
            await asyncio.gather(*tasks)

    def get_consuming_cost_bytes(self) -> int:
        return self.buf_sz_bytes + sum(c.get_consuming_cost_bytes() for c in self.byte_range_to_buffer_consumer.values())


def batch_read_requests(read_reqs: List[ReadReq]) -> List[ReadReq]:
    """Merges the ranged reads that target one file into a single read of their hull
    (T:batcher.py:387-478).  Whole-file reads pass through."""
    out: List[ReadReq] = []
    ranged: Dict[str, List[ReadReq]] = defaultdict(list)
    for rr in read_reqs:
        if rr.byte_range is None:
            out.append(rr)
        else:
            ranged[rr.path].append(rr)
    for path, rrs in ranged.items():
        lo = min(rr.byte_range[0] for rr in rrs)
        hi = max(rr.byte_range[1] for rr in rrs)
        members = {(rr.byte_range[0] - lo, rr.byte_range[1] - lo): rr.buffer_consumer for rr in rrs}
        out.append(ReadReq(path=path, buffer_consumer=BatchedBufferConsumer(members, hi - lo), byte_range=(lo, hi)))
    return out
