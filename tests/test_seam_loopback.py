"""Preparer <-> preparer loopback through the asyncio seam (no storage, no scheduler): every WriteReq is staged
to ``{path: bytes}`` and the ReadReqs are fed from it — the fixture idea of the reference's own tests
(tests/test_tensor_io_preparer.py:34-58, test_batcher.py:402-413, test_sharded_tensor_resharding.py:103-106).
This drives ``stage_buffer`` / ``consume_buffer`` (C-ABI stager/consumer seam on the host engine) rather than
the engine's file jobs, i.e. the path third-party storage plugins take."""
import asyncio
import itertools
import random
import tempfile

import pytest
import torch
import torch.distributed as dist

from tests.util import ALL_RAW_DTYPES, det_tensor, wire_bytes
from torchsnapshot_b200 import knobs
from torchsnapshot_b200.batcher import BatchedBufferStager, batch_read_requests, batch_write_requests
from torchsnapshot_b200.io_preparer import prepare_read, prepare_write
from torchsnapshot_b200.io_preparers.chunked_tensor import ChunkedTensorIOPreparer
from torchsnapshot_b200.io_preparers.sharded_tensor import ShardedTensorIOPreparer
from torchsnapshot_b200.io_preparers.tensor import TensorIOPreparer
from torchsnapshot_b200.manifest import ChunkedTensorEntry, ShardedTensorEntry, TensorEntry


def fulfil(read_reqs, write_reqs):
    async def go():
        store = {}
        for wr in write_reqs:
            buf = await wr.buffer_stager.stage_buffer(None)
            if getattr(wr.buffer_stager, "is_raw", lambda: True)():
                assert len(buf) <= wr.buffer_stager.get_staging_cost_bytes()
            store[wr.path] = bytes(buf)
        for rr in read_reqs:
            data = store[rr.path]
            if rr.byte_range is not None:
                data = data[rr.byte_range[0] : rr.byte_range[1]]
            await rr.buffer_consumer.consume_buffer(data, None)
        return store

    return asyncio.new_event_loop().run_until_complete(go())


@pytest.mark.parametrize("dtype", ALL_RAW_DTYPES + [torch.complex64])
def test_tensor_round_trip_every_dtype(dtype):
    src = det_tensor((29, 13), dtype, 3) if dtype != torch.complex64 else torch.randn(29, 13, dtype=torch.complex64)
    for view in (src, src.t(), src[3:20, 2:9]):
        entry, wrs = TensorIOPreparer.prepare_write("0/x", view)
        assert entry.serializer == ("torch_save" if dtype == torch.complex64 else "buffer_protocol")
        dst = torch.zeros(view.shape, dtype=dtype)
        rrs, fut = TensorIOPreparer.prepare_read(entry, dst)
        store = fulfil(rrs, wrs)
        assert fut.obj is dst and torch.equal(dst, view) if dtype == torch.complex64 else wire_bytes(dst) == wire_bytes(view)
        if dtype != torch.complex64:
            assert store["0/x"] == wire_bytes(view)


def test_hook_whose_output_differs_from_its_trace_fails_to_stage():
    """The entry was planned from the traced dtype; writing the processed tensor's bytes would not match it."""

    def widens_late(t, tracing):
        return t if tracing else t.double()

    entry, wrs = TensorIOPreparer.prepare_write("0/x", torch.ones(4, 3), _tensor_prepare_func=widens_late)
    assert entry.serializer == "buffer_protocol" and entry.dtype == "torch.float32"
    with pytest.raises(RuntimeError, match="0/x"):
        fulfil([], wrs)


@pytest.mark.parametrize("limit", [1, 97, 1000, 10**6])
def test_tiled_read_strided_offset_prime_targets(limit):
    # reference tests/test_tensor_io_preparer.py:159-183
    src = det_tensor((131, 17), torch.float32, 5)
    entry, wrs = TensorIOPreparer.prepare_write("0/x", src)
    targets = [torch.zeros(131, 17), torch.zeros(17, 200).t()[20:151], torch.zeros(140, 40)[5:136, 11:28]]
    for dst in targets:
        rrs, fut = TensorIOPreparer.prepare_read(entry, dst, buffer_size_limit_bytes=limit)
        if limit < src.numel() * 4:
            assert len(rrs) > 1
            # torch.chunk semantics: ceil-sized tiles, so a tile may exceed the limit by less than one row / element
            assert all(rr.byte_range[1] - rr.byte_range[0] < limit + (17 * 4 if not dst.is_contiguous() else 4) for rr in rrs)
        fulfil(rrs, wrs)
        assert wire_bytes(dst) == wire_bytes(src)


def test_chunked_round_trip_and_entry():
    src = det_tensor((50, 12), torch.float64, 7).t()  # non-contiguous 12 x 50
    plan = ChunkedTensorIOPreparer.chunk_tensor(src, chunk_sz_bytes=1000)
    assert [(c.offsets, c.sizes) for c in plan] == [([0, 0], [3, 50]), ([3, 0], [3, 50]), ([6, 0], [3, 50]), ([9, 0], [3, 50])]
    entry, wrs = ChunkedTensorIOPreparer.prepare_write("0/big", src, plan)
    assert isinstance(entry, ChunkedTensorEntry) and [c.tensor.location for c in entry.chunks] == ["0/big_0_0", "0/big_3_0", "0/big_6_0", "0/big_9_0"]
    dst = torch.zeros(12, 50, dtype=torch.float64)
    rrs, _ = ChunkedTensorIOPreparer.prepare_read(entry, dst, buffer_size_limit_bytes=300)
    store = fulfil(rrs, wrs)
    assert wire_bytes(dst) == wire_bytes(src)
    for c in entry.chunks:
        assert store[c.tensor.location] == wire_bytes(src[c.offsets[0] : c.offsets[0] + c.sizes[0]])


@pytest.mark.parametrize("batch_reads", [False, True])
def test_batcher_fifty_tensors_shuffled(batch_reads):
    # reference tests/test_batcher.py:299-417
    rng = random.Random(0)
    tensors = {f"t{i}": det_tensor((rng.randint(1, 60), rng.randint(1, 40)), ALL_RAW_DTYPES[i % len(ALL_RAW_DTYPES)], i) for i in range(50)}
    tensors["big"] = det_tensor((300, 50), torch.float32, 99)  # above the threshold below: never batched
    entries, wrs = {}, []
    with knobs.override_max_chunk_size_bytes(8000):
        for k, t in tensors.items():
            e, w = prepare_write(t, f"x/{k}", rank=0, replicated=False)
            entries[k] = e
            wrs += w
    rng.shuffle(wrs)
    n_before = len(wrs)
    _, batched = batch_write_requests(list(entries.values()), wrs, slab_size_threshold_bytes=4096)
    assert len(batched) < n_before
    slabs = [w for w in batched if isinstance(w.buffer_stager, BatchedBufferStager)]
    assert slabs and all(w.buffer_stager.slab_sz_bytes < 4096 for w in slabs)
    with pytest.raises(RuntimeError, match="not passed to batch_write"):
        e2, w2 = prepare_write(torch.ones(3), "x/missing", rank=0, replicated=False)
        batch_write_requests([], w2, slab_size_threshold_bytes=4096)
    outs = {k: torch.zeros_like(t) for k, t in tensors.items()}
    rrs = []
    for k, e in entries.items():
        r, _ = prepare_read(e, outs[k])
        rrs += r
    if batch_reads:
        merged = batch_read_requests(rrs)
        assert len(merged) < len(rrs)
        rrs = merged
    fulfil(rrs, batched)
    for k in tensors:
        assert wire_bytes(outs[k]) == wire_bytes(tensors[k]), k


@pytest.fixture(scope="module")
def pg():
    if not dist.is_initialized():
        f = tempfile.NamedTemporaryFile(delete=False)
        dist.init_process_group("gloo", init_method=f"file://{f.name}", rank=0, world_size=1)
    yield
    if dist.is_initialized():
        dist.destroy_process_group()


def _sharded(full, spec):
    from torch.distributed._shard.sharded_tensor import Shard, ShardedTensor, ShardMetadata

    shards = []
    for off, sz in spec:
        t = full[off[0] : off[0] + sz[0], off[1] : off[1] + sz[1]].contiguous()
        shards.append(Shard(tensor=t, metadata=ShardMetadata(shard_offsets=list(off), shard_sizes=list(sz), placement="rank:0/cpu")))
    return ShardedTensor._init_from_local_shards(shards, tuple(full.shape))


def _specs(rows, cols):
    def chunks(n, k):
        step = -(-n // k)
        return [(lo, min(step, n - lo)) for lo in range(0, n, step)]

    return {
        "dim0x3": [((lo, 0), (n, cols)) for lo, n in chunks(rows, 3)],
        "dim0x5": [((lo, 0), (n, cols)) for lo, n in chunks(rows, 5)],
        "dim1x3": [((0, lo), (rows, n)) for lo, n in chunks(cols, 3)],
        "dim1x5": [((0, lo), (rows, n)) for lo, n in chunks(cols, 5)],
        "grid2x2": [((r, c), (rn, cn)) for r, rn in chunks(rows, 2) for c, cn in chunks(cols, 2)],
    }


@pytest.mark.parametrize("src_spec,dst_spec", list(itertools.product(["dim0x3", "dim0x5", "dim1x3", "dim1x5", "grid2x2"], repeat=2)))
def test_resharding_five_by_five(src_spec, dst_spec, pg):
    # reference tests/test_sharded_tensor_resharding.py:78-110
    rows, cols = 34, 26
    full = det_tensor((rows, cols), torch.float32, 11)
    specs = _specs(rows, cols)
    src = _sharded(full, specs[src_spec])
    dst = _sharded(torch.zeros(rows, cols), specs[dst_spec])
    with knobs.override_max_shard_size_bytes(400):
        entry, wrs = ShardedTensorIOPreparer.prepare_write("sharded/x", src)
    assert isinstance(entry, ShardedTensorEntry) and len(entry.shards) >= len(specs[src_spec])
    for sh, wr in zip(entry.shards, wrs):
        assert isinstance(sh.tensor, TensorEntry) and sh.tensor.shape == sh.sizes  # persisted size == view size
    entries = [entry]
    _, batched = batch_write_requests(entries, wrs, slab_size_threshold_bytes=2048)
    rrs, fut = ShardedTensorIOPreparer.prepare_read(entry, dst)
    fulfil(batch_read_requests(rrs), batched)
    for sh in dst.local_shards():
        o, s = sh.metadata.shard_offsets, sh.metadata.shard_sizes
        assert wire_bytes(sh.tensor) == wire_bytes(full[o[0] : o[0] + s[0], o[1] : o[1] + s[1]])
    # no runtime object -> whole tensor on the host
    rrs, fut = ShardedTensorIOPreparer.prepare_read(entry, None)
    fulfil(rrs, batched)
    assert wire_bytes(fut.obj) == wire_bytes(full)


def test_partial_overlap_reads_only_the_needed_hull(pg, tmp_path):
    """A local shard that needs a few rows of a saved piece reads just those rows (plus nothing else)."""
    import torchsnapshot_b200 as B
    from torchsnapshot_b200 import _native as N

    rows, cols = 4000, 64
    full = det_tensor((rows, cols), torch.float32, 21)
    src = _sharded(full, [((0, 0), (rows, cols))])  # one saved piece: the whole table (1 MB)
    with knobs.override_is_batching_disabled(True):
        snap = B.Snapshot.take(str(tmp_path / "s"), {"m": B.StateDict(t=src)})
    # target: rows 1000..1100 only
    dst_local = torch.zeros(100, cols)
    from torch.distributed._shard.sharded_tensor import Shard, ShardedTensor, ShardMetadata

    entry = snap.get_manifest()["0/m/t"]
    rrs, _ = ShardedTensorIOPreparer.prepare_read(entry, None)
    assert rrs[0].byte_range is None  # whole table wanted -> whole piece, like the reference
    from torchsnapshot_b200.io_preparers.sharded_tensor import overlap_read_reqs

    reqs = overlap_read_reqs(entry.shards, [(dst_local, [1000, 0], [100, cols])])
    assert len(reqs) == 1 and reqs[0].byte_range == (1000 * cols * 4, 1100 * cols * 4)
    eng = N.get_engine(-1)
    before = eng.stats()["bytes_read"]
    from torchsnapshot_b200.scheduler import sync_execute_read_reqs
    from torchsnapshot_b200.storage_plugin import url_to_storage_plugin_in_event_loop

    loop = asyncio.new_event_loop()
    storage = url_to_storage_plugin_in_event_loop(str(tmp_path / "s"), loop)
    sync_execute_read_reqs(reqs, storage, 1 << 30, 0, loop)
    assert eng.stats()["bytes_read"] - before == 100 * cols * 4
    assert wire_bytes(dst_local) == wire_bytes(full[1000:1100])
    # column slice of the same piece: the hull spans almost all rows, and the scatter still picks the right box
    dst_cols = torch.zeros(rows, 8)
    reqs = overlap_read_reqs(entry.shards, [(dst_cols, [0, 16], [rows, 8])])
    sync_execute_read_reqs(reqs, storage, 1 << 30, 0, loop)
    assert wire_bytes(dst_cols) == wire_bytes(full[:, 16:24])
    # and through the asyncio seam (non-native storage): the consumer is handed exactly the hull bytes
    dst2 = torch.zeros(100, cols)
    reqs = overlap_read_reqs(entry.shards, [(dst2, [1000, 0], [100, cols])])
    data = (tmp_path / "s" / entry.shards[0].tensor.location).read_bytes()
    lo, hi = reqs[0].byte_range
    loop.run_until_complete(reqs[0].buffer_consumer.consume_buffer(data[lo:hi], None))
    assert wire_bytes(dst2) == wire_bytes(full[1000:1100])
    loop.close()
