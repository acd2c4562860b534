"""Host-side planning logic against the oracle on random inputs (hypothesis): chunk plans, shard subdivision, slab
assignment / relocation, greedy partitioning, overlap boxes, knobs."""
import os

import pytest
import torch
from hypothesis import given, settings
from hypothesis import strategies as st

from oracle import ref_port as R
from torchsnapshot_b200 import knobs
from torchsnapshot_b200.batcher import batch_write_requests
from torchsnapshot_b200.io_preparers.chunked_tensor import ChunkedTensorIOPreparer
from torchsnapshot_b200.io_preparers.sharded_tensor import ShardedTensorIOPreparer, boxes_overlap, overlap_narrows
from torchsnapshot_b200.io_preparers.tensor import TensorIOPreparer
from torchsnapshot_b200.partitioner import _partition_write_loads, _WriteLoad

FAST = settings(max_examples=60, deadline=None)


@FAST
@given(st.lists(st.integers(1, 40), min_size=0, max_size=3), st.sampled_from([torch.uint8, torch.bfloat16, torch.float32, torch.float64]), st.integers(1, 5000))
def test_chunk_plan_matches_oracle(shape, dtype, limit):
    t = torch.zeros(shape, dtype=dtype)
    if t.numel() == 0:
        return
    plan = ChunkedTensorIOPreparer.chunk_tensor(t, chunk_sz_bytes=limit)
    assert [(c.offsets, c.sizes) for c in plan] == R.chunk_plan(shape, t.element_size(), limit)
    # chunks tile the tensor along dim 0
    rows = sum(c.sizes[0] for c in plan)
    assert rows == (shape[0] if shape else 1)


@FAST
@given(st.lists(st.integers(1, 30), min_size=1, max_size=3), st.integers(0, 2), st.integers(1, 3000), st.sampled_from([1, 2, 4, 8]))
def test_subdivide_matches_oracle(sizes, dim, limit, esz):
    dim = dim % len(sizes)
    dtype = {1: torch.uint8, 2: torch.int16, 4: torch.float32, 8: torch.float64}[esz]
    shard = torch.zeros(sizes, dtype=dtype)
    offsets = [3 * (i + 1) for i in range(len(sizes))]
    got = ShardedTensorIOPreparer.subdivide_shard(shard, offsets, sizes, dim, limit)
    want = R.subdivide_plan(offsets, sizes, dim, esz, limit)
    assert [(o, s) for _, o, s in got] == [(o, s) for _, o, s in want]
    assert sum(v.shape[dim] for v, _, _ in got) == sizes[dim]


@FAST
@given(st.lists(st.integers(1, 300), min_size=1, max_size=40), st.integers(16, 400))
def test_slab_assignment_and_relocation_match_oracle(sizes, threshold):
    entries, reqs = [], []
    for i, n in enumerate(sizes):
        e, w = TensorIOPreparer.prepare_write(f"0/t{i}", torch.zeros(n, dtype=torch.uint8))
        entries.append(e)
        reqs += w
    order = [(f"0/t{i}", n, False, True) for i, n in enumerate(sizes)]
    passthrough, slabs = R.slab_assign(order, threshold)
    _, batched = batch_write_requests(entries, reqs, slab_size_threshold_bytes=threshold)
    assert [w.path for w in batched if not w.path.startswith("batched/")] == passthrough
    got_slabs = [w for w in batched if w.path.startswith("batched/")]
    assert len(got_slabs) == len(slabs)
    for w, s in zip(got_slabs, slabs):
        assert list(w.buffer_stager.byte_range_to_buffer_stager.keys()) == [(lo, hi) for _, lo, hi in s["members"]]
    where = {loc: (k, lo, hi) for k, s in enumerate(slabs) for loc, lo, hi in s["members"]}
    for i, e in enumerate(entries):
        if f"0/t{i}" in where:
            k, lo, hi = where[f"0/t{i}"]
            assert e.location == got_slabs[k].path and e.byte_range == [lo, hi]
        else:
            assert e.location == f"0/t{i}" and e.byte_range is None


@FAST
@given(st.lists(st.integers(1, 1000), min_size=1, max_size=30), st.lists(st.integers(0, 500), min_size=1, max_size=6))
def test_greedy_partition_matches_oracle(sizes, initial_loads):
    world = len(initial_loads)
    from torchsnapshot_b200.manifest import TensorEntry

    entries = {f"p{i}": TensorEntry(f"replicated/p{i}", "buffer_protocol", "torch.uint8", [n], True) for i, n in enumerate(sizes)}
    loads = {f"p{i}": [_WriteLoad(f"p{i}", 0, n)] for i, n in enumerate(sizes)}
    got = _partition_write_loads([entries] * world, [loads] * world, list(initial_loads), world)
    want = R.partition_greedy([(f"p{i}", n) for i, n in enumerate(sizes)], initial_loads)
    assert [[wl.logical_path for wl in r] for r in got] == want
    # every path written exactly once
    assert sorted(wl.logical_path for r in got for wl in r) == sorted(loads)


@FAST
@given(st.integers(1, 3), st.data())
def test_overlap_boxes_match_oracle(nd, data):
    def box():
        off = [data.draw(st.integers(0, 20)) for _ in range(nd)]
        sz = [data.draw(st.integers(1, 20)) for _ in range(nd)]
        return off, sz

    a, b = box(), box()
    assert boxes_overlap(*a, *b) == R.boxes_overlap(*a, *b)
    if R.boxes_overlap(*a, *b):
        assert overlap_narrows(a, b) == R.overlap_region(a[0], a[1], b[0], b[1])
        assert all(n > 0 for _, _, _, n in overlap_narrows(a, b))


def test_knobs_follow_the_reference_environment_variables(monkeypatch):
    for env, getter, default in [
        ("TORCHSNAPSHOT_MAX_CHUNK_SIZE_BYTES_OVERRIDE", knobs.get_max_chunk_size_bytes, 512 << 20),
        ("TORCHSNAPSHOT_MAX_SHARD_SIZE_BYTES_OVERRIDE", knobs.get_max_shard_size_bytes, 512 << 20),
        ("TORCHSNAPSHOT_SLAB_SIZE_THRESHOLD_BYTES_OVERRIDE", knobs.get_slab_size_threshold_bytes, 128 << 20),
        ("TORCHSNAPSHOT_MAX_PER_RANK_IO_CONCURRENCY_OVERRIDE", knobs.get_max_per_rank_io_concurrency, 16),
    ]:
        monkeypatch.delenv(env, raising=False)
        assert getter() == default
        monkeypatch.setenv(env, "12345")
        assert getter() == 12345
    monkeypatch.delenv("TORCHSNAPSHOT_DISABLE_BATCHING", raising=False)
    assert knobs.is_batching_disabled() is False
    for v in ("1", "true", "True"):
        monkeypatch.setenv("TORCHSNAPSHOT_DISABLE_BATCHING", v)
        assert knobs.is_batching_disabled() is True
    with knobs.override_max_chunk_size_bytes(77):
        assert knobs.get_max_chunk_size_bytes() == 77
    monkeypatch.setenv("TORCHSNAPSHOT_PER_RANK_MEMORY_BUDGET_BYTES", "4096")
    from torchsnapshot_b200.pg_wrapper import PGWrapper
    from torchsnapshot_b200.scheduler import get_process_memory_budget_bytes

    assert get_process_memory_budget_bytes(PGWrapper(None)) == 4096


def test_views_with_more_than_eight_dims(tmp_path):
    """Descriptors hold 8 dims; views with more are folded (size-1 dims dropped, dense neighbours merged) and only a
    view that still needs more than 8 strided dims is made contiguous first, like the reference does for every
    non-contiguous source (T:batcher.py:156, T:serialization.py:196)."""
    import torch

    import torchsnapshot_b200 as B
    from tests.util import wire_bytes

    t = torch.randn(2, 3, 1, 2, 2, 3, 2, 2, 2, 2)  # 10-D contiguous
    u = torch.randn(2, 3, 2, 2, 2, 3, 2, 2, 2, 4)[..., ::2]  # 10-D, last dim stepped: merges to 2 dims
    v = torch.randn(3, 2, 2, 2, 2, 2, 2, 2, 2, 2).permute(9, 8, 7, 6, 5, 4, 3, 2, 1, 0)  # 10 non-mergeable dims
    snap = B.Snapshot.take(str(tmp_path / "s"), {"m": B.StateDict(t=t, u=u, v=v)})
    o = B.StateDict(t=torch.zeros_like(t), u=torch.zeros(2, 3, 2, 2, 2, 3, 2, 2, 2, 4)[..., ::2], v=torch.zeros(v.shape))
    snap.restore({"m": o})
    for k, a in (("t", t), ("u", u), ("v", v)):
        assert wire_bytes(a) == wire_bytes(o[k]), k


def test_cast_on_save_is_fused_and_matches_torch(tmp_path):
    """cast_on_save: the entry promises the target dtype and the payload is exactly tensor.to(dtype) — without the
    processed tensor ever being materialised (descriptor with dst_dtype != src_dtype; here executed by the host planner)."""
    import torch

    import torchsnapshot_b200 as B
    from tests.util import wire_bytes

    st = {"w": torch.randn(1000, 33), "wt": torch.randn(64, 48).t(), "i": torch.arange(10), "h": torch.randn(7).half(), "d": torch.randn(5, dtype=torch.float64)}
    snap = B.Snapshot.take(str(tmp_path / "s"), {"m": B.StateDict(**st)}, _custom_tensor_prepare_func=B.cast_on_save(torch.bfloat16, only="m/w*"))
    man = snap.get_manifest()
    assert man["0/m/w"].dtype == "torch.bfloat16" and man["0/m/wt"].dtype == "torch.bfloat16"
    assert man["0/m/h"].dtype == "torch.float16" and man["0/m/i"].dtype == "torch.int64" and man["0/m/d"].dtype == "torch.float64"
    for k in ("w", "wt"):
        data = open(tmp_path / "s" / man[f"0/m/{k}"].location, "rb").read()
        assert data == wire_bytes(st[k].to(torch.bfloat16)), k
    tgt = B.StateDict(w=torch.zeros(1000, 33, dtype=torch.bfloat16), wt=torch.zeros(48, 64, dtype=torch.bfloat16), i=torch.zeros(10, dtype=torch.long),
                      h=torch.zeros(7).half(), d=torch.zeros(5, dtype=torch.float64))
    snap.restore({"m": tgt})
    assert torch.equal(tgt["w"], st["w"].bfloat16()) and torch.equal(tgt["wt"], st["wt"].bfloat16()) and torch.equal(tgt["d"], st["d"])


def test_quantize_on_save_matches_torch_and_the_reference_format(tmp_path):
    """quantize_on_save: payload == int_repr bytes of torch.quantize_per_tensor + [scale: double][zero_point: int64]
    (the reference's per-tensor format, T:serialization.py:278-310; its own codec reads it back), restoring into the
    float tensors dequantises."""
    import struct
    import sys

    import torch

    import torchsnapshot_b200 as B
    from torchsnapshot_b200.serialization import per_tensor_qtensor_from_bytes

    torch.manual_seed(0)
    st = {"w": torch.randn(1000, 33), "wt": torch.randn(64, 48).t(), "h": torch.randn(77).bfloat16(), "u": torch.rand(501) * 3 - 1, "i": torch.arange(10)}
    for qdt in (torch.qint8, torch.quint8):
        path = str(tmp_path / f"s_{qdt}".replace(".", "_"))
        snap = B.Snapshot.take(path, {"m": B.StateDict(**st)}, _custom_tensor_prepare_func=B.quantize_on_save(qdt, only="m/[whu]*"))
        man = snap.get_manifest()
        assert man["0/m/i"].serializer == "buffer_protocol" and man["0/m/w"].serializer == "per_tensor_qtensor"
        hook = B.quantize_on_save(qdt)
        for k in ("w", "wt", "h", "u"):
            data = open(f"{path}/{man[f'0/m/{k}'].location}", "rb").read()
            _, scale, zp = hook.tsnap_quant(f"m/{k}", st[k])
            q = torch.quantize_per_tensor(st[k].float().contiguous(), scale, zp, qdt)
            want = q.int_repr().numpy().tobytes() + struct.pack("d", q.q_scale()) + struct.pack("q", q.q_zero_point())
            assert data == want, (qdt, k)
            back = per_tensor_qtensor_from_bytes(data, qdt, list(st[k].shape))
            assert torch.equal(back.int_repr(), q.int_repr()) and back.q_scale() == q.q_scale()
        tgt = B.StateDict(w=torch.zeros(1000, 33), wt=torch.zeros(48, 64), h=torch.zeros(77).bfloat16(), u=torch.zeros(501), i=torch.zeros(10, dtype=torch.long))
        snap.restore({"m": tgt})
        assert torch.equal(tgt["i"], st["i"])
        for k in ("w", "wt", "u"):
            _, scale, _ = hook.tsnap_quant(f"m/{k}", st[k])
            assert (tgt[k] - st[k]).abs().max().item() <= scale * 0.5 + 1e-6, k


@pytest.mark.parametrize("batching,quantize", [(True, False), (False, False), (True, True)], ids=["True", "False", "quantize_on_save"])
def test_async_take_counts_cpu_copies_against_the_memory_budget(tmp_path, monkeypatch, batching, quantize):
    """async_take may hand control back while the engine still reads host memory, so CPU tensors get a private copy —
    but only while the per-rank memory budget lasts (the reference gates staging on it, T:scheduler.py:259-281);
    what does not fit is written out before async_take returns, from the caller's memory.  Either way the snapshot
    holds the values at the time of the call.  Sources the pack kernel quantises are charged like any other."""
    import torchsnapshot_b200 as B
    from torchsnapshot_b200 import scheduler as S

    monkeypatch.setenv("TORCHSNAPSHOT_PER_RANK_MEMORY_BUDGET_BYTES", str(3 << 20))
    monkeypatch.setenv("TORCHSNAPSHOT_DISABLE_BATCHING", "0" if batching else "1")
    tensors = {f"t{i}": torch.full((1 << 18,), float(i)) for i in range(8)}  # 8 x 1 MiB
    hook = B.quantize_on_save(torch.qint8) if quantize else None
    expect = {k: hook(f"m/{k}", v, False).dequantize() if quantize else v.clone() for k, v in tensors.items()}
    pending = B.Snapshot.async_take(str(tmp_path / "s"), {"m": B.StateDict(**tensors)}, _custom_tensor_prepare_func=hook)
    cloned, in_place = S.LAST_STATS["host_clone_bytes"], S.LAST_STATS["host_blocking_bytes"]
    for v in tensors.values():
        v.add_(100.0)  # the caller owns its memory again
    snap = pending.wait()
    assert cloned <= 3 << 20 and in_place >= 5 << 20 and cloned + in_place == 8 << 20, (cloned, in_place)
    out = B.StateDict(**{k: torch.zeros_like(v) for k, v in tensors.items()})
    snap.restore({"m": out})
    for k, v in expect.items():
        assert torch.equal(out[k], v), k
    # with room for everything nothing blocks
    monkeypatch.setenv("TORCHSNAPSHOT_PER_RANK_MEMORY_BUDGET_BYTES", str(64 << 20))
    B.Snapshot.async_take(str(tmp_path / "s2"), {"m": B.StateDict(**tensors)}, _custom_tensor_prepare_func=hook).wait()
    assert S.LAST_STATS["host_blocking_bytes"] == 0 and S.LAST_STATS["host_clone_bytes"] == 8 << 20


def test_async_take_blocking_part_reports_storage_errors_at_wait(tmp_path, monkeypatch):
    """A storage error in the part async_take writes before returning (CPU tensors beyond the clone budget) surfaces where
    every other storage error of async_take does: PendingSnapshot.wait() (T:tests/test_async_take.py:58-66)."""
    import torchsnapshot_b200 as B

    monkeypatch.setenv("TORCHSNAPSHOT_PER_RANK_MEMORY_BUDGET_BYTES", "1024")
    monkeypatch.setenv("TORCHSNAPSHOT_DISABLE_BATCHING", "1")
    blocker = tmp_path / "not_a_dir"
    blocker.write_text("x")
    pending = B.Snapshot.async_take(str(blocker / "snap"), {"m": B.StateDict(t=torch.ones(1 << 16))})
    with pytest.raises(Exception):
        pending.wait()
    assert not (blocker / "snap").exists()
