"""quantize_on_save(float8 dtype, axis=...) on CPU tensors: the host engine writes the per_channel_fp8 format byte for
byte as the torch statement of the rule (prepare.per_channel_fp8) gives it, and restores it natively into float targets."""
import os
import struct
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import torchsnapshot_b200 as B
from torchsnapshot_b200 import _native
from torchsnapshot_b200 import storage_plugin as SP
from torchsnapshot_b200.io_preparers.tensor import TensorBufferConsumer
from torchsnapshot_b200.prepare import FP8_MAX, dequantize_fp8, per_channel_fp8
from torchsnapshot_b200.serialization import per_channel_fp8_as_bytes, per_channel_fp8_from_bytes
from torchsnapshot_b200.storage_plugins.fs import FSStoragePlugin

FLOATS = [torch.float64, torch.float32, torch.float16, torch.bfloat16]
FP8 = [torch.float8_e4m3fn, torch.float8_e5m2]
EUNSUP = -6  # TSNAP_EUNSUP


def expected_file(x: torch.Tensor, dtype: torch.dtype, axis: int) -> bytes:
    q, s = per_channel_fp8(x.cpu(), dtype, axis)
    return per_channel_fp8_as_bytes(q, s, axis)


def restored_like(x: torch.Tensor, dtype: torch.dtype, axis: int, target=None) -> torch.Tensor:
    """(q.float() * s).to(target dtype)"""
    q, s = per_channel_fp8(x.cpu(), dtype, axis)
    return dequantize_fp8(q, s, axis).to(target or x.dtype)


def sources(dtype):
    g = torch.Generator().manual_seed(11)
    rows = torch.logspace(-9, 2, 37, dtype=torch.float64)[:, None]  # channels of very different magnitudes
    return {
        "w": (torch.randn(37, 53, generator=g, dtype=torch.float64) * rows).to(dtype),
        "w_t": torch.randn(40, 24, generator=g).to(dtype).t(),
        "narrow": torch.randn(60, 70, generator=g).to(dtype)[5:50, 3:40],
        "cube": torch.randn(6, 5, 7, generator=g).to(dtype),
        "bias": torch.randn(9, generator=g).to(dtype),
    }


def take(root, state, hook, async_=False):
    app = {"m": B.StateDict(**state)}
    if async_:
        return B.Snapshot.async_take(root, app, _custom_tensor_prepare_func=hook)
    return B.Snapshot.take(root, app, _custom_tensor_prepare_func=hook)


def file_of(snap, root, key):
    e = snap.get_manifest()[f"0/m/{key}"]
    return e, open(os.path.join(root, e.location), "rb").read()


class Audited(FSStoragePlugin):
    """Overrides write / read, so the engine leaves the I/O to it: the stage / consume seam does the rest."""

    async def write(self, write_io):
        return await super().write(write_io)

    async def read(self, read_io):
        return await super().read(read_io)


def _no_codec(*a, **k):
    raise AssertionError("per-channel float8 restore fell back to the Python codec")


@pytest.mark.parametrize("fp8", FP8)
@pytest.mark.parametrize("dtype", FLOATS)
@pytest.mark.parametrize("axis", [0, 1, -1])
def test_file_bytes_and_native_restore(fp8, dtype, axis, tmp_path, monkeypatch):
    src = sources(dtype)
    root = str(tmp_path / "s")
    snap = take(root, src, B.quantize_on_save(fp8, axis=axis))
    for key in ("w", "w_t", "narrow", "cube"):  # axis 1 of the cube is its middle axis
        x = src[key]
        ax = axis % x.dim()
        e, raw = file_of(snap, root, key)
        assert e.serializer == "per_channel_fp8" and e.dtype == str(fp8) and list(e.shape) == list(x.shape)
        assert len(raw) == 8 + x.numel() + 4 * x.shape[ax]
        assert raw == expected_file(x, fp8, ax), key
    e, raw = file_of(snap, root, "bias")
    assert e.serializer == "buffer_protocol" and raw == src["bias"].contiguous().view(torch.uint8).numpy().tobytes()

    monkeypatch.setattr(TensorBufferConsumer, "deserialize_tensor", staticmethod(_no_codec))
    tgt = {k: torch.full_like(v, 123.0) for k, v in src.items()}
    B.Snapshot(root).restore({"m": B.StateDict(**tgt)})
    for key in ("w", "w_t", "narrow", "cube"):
        assert torch.equal(tgt[key], restored_like(src[key], fp8, axis % src[key].dim())), key
    assert torch.equal(tgt["bias"], src["bias"])


def _grid(fp8):
    """Every non-negative finite value of the format, ascending."""
    v = torch.arange(256, dtype=torch.uint8).view(fp8).float()
    v = v[torch.isfinite(v) & (v >= 0)]
    return torch.unique(v)


def _edge_rows(fp8):
    fmax = FP8_MAX[fp8]
    grid = _grid(fp8)
    ties = (grid[:-1] + grid[1:]) / 2  # exact midpoints: quotients on fp8 rounding ties when s == 1
    n = ties.numel() + 1
    rows = torch.zeros(8, n)
    rows[1, :3] = torch.tensor([1e-45, -1e-45, 0.0])  # amax subnormal, s = amax / FMAX underflows to 0 -> 1
    rows[2, :3] = torch.tensor([1e-38, -3e-39, 5e-40])  # s itself subnormal
    rows[3] = torch.linspace(-1, 1, n) * 3.7
    rows[3, 0], rows[3, 1] = 3.7, -3.7  # elements at +-amax land on +-FMAX
    rows[4, : ties.numel()] = ties
    rows[4, -1] = fmax  # s == 1
    rows[5, : ties.numel()] = -ties
    rows[5, -1] = fmax
    rows[6] = torch.logspace(-30, 30, n) * torch.where(torch.arange(n) % 2 == 0, 1.0, -1.0)  # 1e-30 .. 1e30
    rows[7, : ties.numel()] = ties * 0.75  # s = 0.75: quotients on the ties again, through the division
    rows[7, -1] = fmax * 0.75
    return rows


@pytest.mark.parametrize("fp8", FP8)
def test_edge_channels(fp8, tmp_path):
    rows = _edge_rows(fp8)
    one = torch.randn(5, 1) * torch.tensor([[0.0], [1e-40], [1.0], [-3e5], [7.0]])  # one-element channels
    root = str(tmp_path / "s")
    snap = take(root, {"rows": rows, "cols": rows.t().contiguous(), "one": one}, B.quantize_on_save(fp8, axis=0))
    for key, x in (("rows", rows), ("cols", rows.t().contiguous()), ("one", one)):
        assert file_of(snap, root, key)[1] == expected_file(x, fp8, 0), key
    q, s = per_channel_fp8(rows, fp8, 0)
    assert s[0] == 1 and s[1] == 1 and 0 < s[2] < torch.finfo(torch.float32).tiny and s[4] == 1
    assert q[3, 0].float() == FP8_MAX[fp8] and q[3, 1].float() == -FP8_MAX[fp8]
    assert (q[0].float() == 0).all()
    tgt = torch.zeros_like(rows)
    B.Snapshot(root).restore({"m": B.StateDict(rows=tgt)})
    assert torch.equal(tgt, restored_like(rows, fp8, 0))


@pytest.mark.parametrize("target", FLOATS)
@pytest.mark.parametrize("fp8", FP8)
def test_restore_into_float_dtypes_strided_and_narrowed(target, fp8, tmp_path):
    x = torch.randn(33, 48) * torch.logspace(-6, 1, 48)
    root = str(tmp_path / "s")
    take(root, {"w": x, "v": x.clone()}, B.quantize_on_save(fp8, axis=1))
    base = torch.zeros(48, 33, dtype=target)
    dst = base.t()  # a strided destination
    wide = torch.zeros(40, 60, dtype=target)
    narrowed = wide[3:36, 5:53]  # a narrowed one
    B.Snapshot(root).restore({"m": B.StateDict(w=dst, v=narrowed)})
    want = restored_like(x, fp8, 1, target)
    assert torch.equal(dst, want) and torch.equal(narrowed, want)
    assert (wide[:3] == 0).all() and (wide[:, :5] == 0).all() and (wide[36:] == 0).all() and (wide[:, 53:] == 0).all()


def test_read_object_returns_the_codec_fp32(tmp_path):
    x = torch.randn(20, 30, dtype=torch.bfloat16)
    root = str(tmp_path / "s")
    snap = take(root, {"w": x}, B.quantize_on_save(torch.float8_e5m2, axis=0))
    got = B.Snapshot(root).read_object("0/m/w")
    e, raw = file_of(snap, root, "w")
    assert got.dtype == torch.float32 and torch.equal(got, per_channel_fp8_from_bytes(raw, torch.float8_e5m2, [20, 30]))
    assert torch.equal(got, restored_like(x, torch.float8_e5m2, 0, torch.float32))
    # the hook's own non-tracing result is the same tensor
    hook = B.quantize_on_save(torch.float8_e5m2, axis=0)
    assert torch.equal(hook("w", x, False), got)


def test_non_float_target_goes_through_the_codec(tmp_path):
    x = torch.randn(12, 16)
    root = str(tmp_path / "s")
    take(root, {"w": x}, B.quantize_on_save(torch.float8_e4m3fn, axis=1))
    tgt = torch.zeros(12, 16, dtype=torch.float8_e4m3fn)
    B.Snapshot(root).restore({"m": B.StateDict(w=tgt)})
    assert torch.equal(tgt.view(torch.uint8), restored_like(x, torch.float8_e4m3fn, 1, torch.float32).to(torch.float8_e4m3fn).view(torch.uint8))


def test_chunked_tensor_pieces_have_their_own_scales(tmp_path, monkeypatch):
    monkeypatch.setenv("TORCHSNAPSHOT_MAX_CHUNK_SIZE_BYTES_OVERRIDE", "4096")
    x = torch.randn(64, 48) * torch.logspace(-8, 1, 64)[:, None]
    root = str(tmp_path / "s")
    snap = take(root, {"w": x}, B.quantize_on_save(torch.float8_e4m3fn, axis=-1))
    entry = snap.get_manifest()["0/m/w"]
    assert entry.type == "ChunkedTensor" and len(entry.chunks) > 1
    full = torch.zeros_like(x)
    for c in entry.chunks:
        assert c.tensor.serializer == "per_channel_fp8"
        piece = x[c.offsets[0] : c.offsets[0] + c.sizes[0]]
        raw = open(os.path.join(root, c.tensor.location), "rb").read()
        assert raw == expected_file(piece, torch.float8_e4m3fn, 1)
        full[c.offsets[0] : c.offsets[0] + c.sizes[0]] = restored_like(piece, torch.float8_e4m3fn, 1)
    tgt = torch.zeros_like(x)
    B.Snapshot(root).restore({"m": B.StateDict(w=tgt)})
    assert torch.equal(tgt, full)


def test_api_errors_and_skips(tmp_path):
    with pytest.raises(ValueError, match="cast_on_save"):
        B.quantize_on_save(torch.float8_e4m3fn)
    with pytest.raises(ValueError):
        B.quantize_on_save(torch.float8_e5m2, qparams=lambda p, t: (1.0, 0), axis=0)
    hook = B.quantize_on_save(torch.float8_e4m3fn, axis=1, only="m/w*")
    src = {
        "w": torch.randn(4, 5),
        "w_one_d": torch.randn(6),
        "w_ints": torch.arange(12).reshape(3, 4),
        "w_empty": torch.zeros(0, 3),
        "w_fp8": torch.randn(4, 5).to(torch.float8_e5m2),
        "other": torch.randn(4, 5),
    }
    root = str(tmp_path / "s")
    snap = take(root, src, hook)
    m = snap.get_manifest()
    assert m["0/m/w"].serializer == "per_channel_fp8"
    for key in ("w_one_d", "w_ints", "w_empty", "w_fp8", "other"):
        assert m[f"0/m/{key}"].serializer == "buffer_protocol", key
    # axis out of range for the tensor: stored unchanged
    snap = take(str(tmp_path / "t"), {"w": torch.randn(4, 5)}, B.quantize_on_save(torch.float8_e4m3fn, axis=2))
    assert snap.get_manifest()["0/m/w"].serializer == "buffer_protocol"
    # quantised sources are stored unchanged too
    qt = torch.quantize_per_tensor(torch.randn(4, 5), 0.1, 0, torch.qint8)
    assert hook("m/w", qt, True) is qt
    # tracing returns dtype and shape
    traced = hook("m/w", torch.randn(4, 5), True)
    assert traced.dtype == torch.float8_e4m3fn and traced.shape == torch.Size([4, 5])


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
def test_nonfinite_fails_the_take_without_a_manifest(bad, tmp_path):
    x = torch.randn(8, 8)
    x[3, 5] = bad
    root = str(tmp_path / "s")
    with pytest.raises(Exception, match="NaN or Inf"):
        take(root, {"w": x}, B.quantize_on_save(torch.float8_e4m3fn, axis=0))
    assert not os.path.exists(os.path.join(root, ".snapshot_metadata"))
    with pytest.raises(ValueError, match="NaN or Inf"):
        per_channel_fp8(x, torch.float8_e4m3fn, 0)


def test_async_take_copies_cpu_sources(tmp_path):
    x = torch.randn(64, 32)
    want = expected_file(x, torch.float8_e5m2, 0)
    root = str(tmp_path / "s")
    pending = take(root, {"w": x}, B.quantize_on_save(torch.float8_e5m2, axis=0), async_=True)
    x.mul_(-3.0).add_(1.0)  # after async_take returned
    snap = pending.wait()
    assert file_of(snap, root, "w")[1] == want


def test_plugin_that_overrides_io_gets_the_same_bytes(tmp_path, monkeypatch):
    monkeypatch.setattr(SP, "FSStoragePlugin", Audited)
    src = sources(torch.float32)
    root = str(tmp_path / "s")
    snap = take(root, src, B.quantize_on_save(torch.float8_e4m3fn, axis=0))
    for key in ("w", "w_t", "narrow", "cube"):
        assert file_of(snap, root, key)[1] == expected_file(src[key], torch.float8_e4m3fn, 0), key
    monkeypatch.setattr(TensorBufferConsumer, "deserialize_tensor", staticmethod(_no_codec))
    tgt = {k: torch.zeros_like(v) for k, v in src.items()}
    B.Snapshot(root).restore({"m": B.StateDict(**tgt)})
    for key in ("w", "w_t", "narrow", "cube"):
        assert torch.equal(tgt[key], restored_like(src[key], torch.float8_e4m3fn, 0)), key


def _corrupt_header_and_size(tmp_path):
    x = torch.randn(10, 12)
    root = str(tmp_path / "s")
    snap = take(root, {"w": x}, B.quantize_on_save(torch.float8_e4m3fn, axis=0))
    e, raw = file_of(snap, root, "w")
    path = os.path.join(root, e.location)
    with open(path, "r+b") as f:
        f.write(struct.pack("<q", 3))
    with pytest.raises(RuntimeError, match="axis 3"):
        B.Snapshot(root).restore({"m": B.StateDict(w=torch.zeros(10, 12))})
    with open(path, "wb") as f:
        f.write(raw[:-4])
    with pytest.raises(RuntimeError, match="bytes"):
        B.Snapshot(root).restore({"m": B.StateDict(w=torch.zeros(10, 12))})


def test_corrupt_header_and_size_give_clear_errors(tmp_path):
    _corrupt_header_and_size(tmp_path)


def test_corrupt_header_and_size_give_clear_errors_through_an_io_plugin(tmp_path, monkeypatch):
    monkeypatch.setattr(SP, "FSStoragePlugin", Audited)
    _corrupt_header_and_size(tmp_path)


def test_codec_rejects_bad_buffers():
    q, s = per_channel_fp8(torch.randn(4, 6), torch.float8_e4m3fn, 1)
    raw = per_channel_fp8_as_bytes(q, s, 1)
    with pytest.raises(RuntimeError, match="size"):
        per_channel_fp8_from_bytes(raw[:-1], torch.float8_e4m3fn, [4, 6])
    with pytest.raises(RuntimeError, match="axis"):
        per_channel_fp8_from_bytes(struct.pack("<q", 2) + raw[8:], torch.float8_e4m3fn, [4, 6])


# ---- the C ABI directly ---------------------------------------------------------------------------------
def _host_save_desc(x, fp8=torch.float8_e4m3fn, axis=0):
    d = _native.save_desc(x, 8, wire_dtype=fp8, axis=axis)
    return d, 8 + x.numel() + 4 * x.shape[axis]


@pytest.mark.parametrize("fp8", FP8)
def test_host_execute_writes_and_reads_the_format(fp8):
    x = torch.randn(12, 20, dtype=torch.float64)
    d, n = _host_save_desc(x, fp8, 1)
    wire = bytearray(n)
    _native.host_execute([d], wire)
    assert bytes(wire) == expected_file(x, fp8, 1)
    for target in FLOATS:
        out = torch.zeros(12, 20, dtype=target)
        r = _native.per_channel(_native.load_desc(out, 8, wire_dtype=fp8), [12, 20], 1, 8)
        _native.host_execute([r], wire)
        assert torch.equal(out, restored_like(x, fp8, 1, target)), target


def test_per_channel_pairs_outside_float_and_float8_are_unsupported():
    x = torch.randn(4, 6)
    wire = bytearray(8 + 24 + 64)
    # fp8 source -> fp8 wire under the per-channel scheme
    src8 = x.to(torch.float8_e4m3fn)
    d = _native.per_channel(_native.save_desc(src8, 8, wire_dtype=torch.float8_e5m2), [4, 6], 0, 8)
    with pytest.raises(_native.NativeError) as ei:
        _native.host_execute([d], wire)
    assert ei.value.code == EUNSUP
    # fp8 wire -> fp8 / int destinations
    for target in (torch.float8_e5m2, torch.float8_e4m3fn, torch.int32):
        r = _native.per_channel(_native.load_desc(torch.zeros(4, 6, dtype=target), 8, wire_dtype=torch.float8_e4m3fn), [4, 6], 0, 8)
        with pytest.raises(_native.NativeError) as ei:
            _native.host_execute([r], wire)
        assert ei.value.code == EUNSUP, target
    # int source -> fp8 wire, qint8 wire -> fp8 destination
    d = _native.per_channel(_native.save_desc(torch.arange(24).reshape(4, 6), 8, wire_dtype=torch.float8_e4m3fn), [4, 6], 0, 8)
    r = _native.per_channel(_native.load_desc(torch.zeros(4, 6, dtype=torch.float8_e4m3fn), 8, wire_dtype=torch.qint8), [4, 6], 0, 8)
    for bad in (d, r):
        with pytest.raises(_native.NativeError) as ei:
            _native.host_execute([bad], wire)
        assert ei.value.code == EUNSUP


@pytest.mark.parametrize(
    "field,value,match",
    [
        ("channels", 0, "positive"),
        ("inner", -1, "positive"),
        ("params_addr", 9, "whole number"),
        ("params_addr", 56, "whole piece"),
        ("axis", 5, "axis"),
    ],
)
def test_malformed_records_are_rejected(field, value, match):
    x = torch.randn(4, 6)
    d, n = _host_save_desc(x)
    setattr(d._qchannel, field, value)
    with pytest.raises(_native.NativeError, match=match):
        _native.host_execute([d], bytearray(n + 64))


def test_short_wire_buffer_is_rejected():
    d, n = _host_save_desc(torch.randn(4, 6))
    with pytest.raises(_native.NativeError, match="exceeds"):
        _native.host_execute([d], bytearray(n - 1))
    _native.host_execute([_host_save_desc(torch.randn(4, 6))[0]], bytearray(n))  # exactly 4 B per channel is enough


def test_plan_describe_accepts_the_new_pairs():
    x = torch.randn(16, 32)
    d, _ = _host_save_desc(x, torch.float8_e5m2, 0)
    info = _native.plan_describe([d])
    assert info["n_members_host"] == 1


# ---- two gloo ranks: per-rank sharded pieces, restored resharded ---------------------------------------
ROWS, COLS = 24, 18


def _full():
    return torch.randn(ROWS, COLS, generator=torch.Generator().manual_seed(3)) * torch.logspace(-7, 0, COLS)


def _worker(rank, world, store_path, root):
    from torch.distributed._shard.sharded_tensor import Shard, ShardedTensor, ShardMetadata

    dist.init_process_group("gloo", init_method=f"file://{store_path}", rank=rank, world_size=world)
    full, step = _full(), ROWS // world
    local = full[rank * step : (rank + 1) * step].contiguous()
    st = ShardedTensor._init_from_local_shards(
        [Shard(tensor=local, metadata=ShardMetadata(shard_offsets=[rank * step, 0], shard_sizes=[step, COLS], placement=f"rank:{rank}/cpu"))], (ROWS, COLS)
    )
    B.Snapshot.take(os.path.join(root, "snap"), {"m": B.StateDict(t=st)}, _custom_tensor_prepare_func=B.quantize_on_save(torch.float8_e4m3fn, axis=1))
    dist.barrier()
    TensorBufferConsumer.deserialize_tensor = staticmethod(_no_codec)
    cols = COLS // world
    band = torch.zeros(ROWS, cols, dtype=torch.bfloat16)
    tgt = ShardedTensor._init_from_local_shards(
        [Shard(tensor=band, metadata=ShardMetadata(shard_offsets=[0, rank * cols], shard_sizes=[ROWS, cols], placement=f"rank:{rank}/cpu"))], (ROWS, COLS)
    )
    B.Snapshot(os.path.join(root, "snap")).restore({"m": B.StateDict(t=tgt)})
    want = torch.cat([restored_like(full[r * step : (r + 1) * step], torch.float8_e4m3fn, 1, torch.bfloat16) for r in range(world)])
    assert torch.equal(band, want[:, rank * cols : (rank + 1) * cols])
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_resharded_restore(tmp_path):
    store = tempfile.NamedTemporaryFile(delete=False)
    try:
        mp.spawn(_worker, args=(2, store.name, str(tmp_path)), nprocs=2, join=True)
    finally:
        if os.path.exists(store.name):
            os.unlink(store.name)
