"""quantize_on_save(axis=...) on CPU tensors: the host engine writes the reference's per-channel format, byte for byte
what torch.quantize_per_channel gives with the default rule, and restores it natively into float targets."""
import os
import struct
import sys
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import torchsnapshot_b200 as B
from torchsnapshot_b200 import _native
from torchsnapshot_b200 import storage_plugin as SP
from torchsnapshot_b200.io_preparers.tensor import TensorBufferConsumer
from torchsnapshot_b200.prepare import per_channel_qparams
from torchsnapshot_b200.serialization import per_channel_qtensor_from_bytes
from torchsnapshot_b200.storage_plugins.fs import FSStoragePlugin
from tests.util import HAVE_REF, REF_PARENT

FLOATS = [torch.float32, torch.bfloat16, torch.float16, torch.float64]


def expected_file(x: torch.Tensor, qdtype: torch.dtype, axis: int) -> bytes:
    """[axis][int_repr][scales][zero_points] with the default rule computed by torch."""
    scales, zps = per_channel_qparams(x.cpu(), qdtype, axis)
    q = torch.quantize_per_channel(x.detach().cpu().float(), scales, zps, axis, qdtype)
    return struct.pack("<q", axis) + q.int_repr().contiguous().numpy().tobytes() + scales.numpy().tobytes() + zps.numpy().tobytes()


def dequantized_like(x: torch.Tensor, qdtype: torch.dtype, axis: int) -> torch.Tensor:
    """dst.copy_(q.dequantize()) for a destination shaped and typed like x."""
    scales, zps = per_channel_qparams(x.cpu(), qdtype, axis)
    q = torch.quantize_per_channel(x.detach().cpu().float(), scales, zps, axis, qdtype)
    dst = torch.empty(x.shape, dtype=x.dtype)
    dst.copy_(q.dequantize())
    return dst


def sources(dtype):
    g = torch.Generator().manual_seed(7)
    rows = torch.logspace(-2, 2, 37, dtype=torch.float64)[:, None]  # channels of very different ranges
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
    raise AssertionError("per-channel restore fell back to the Python codec")


@pytest.mark.parametrize("qdtype", [torch.qint8, torch.quint8])
@pytest.mark.parametrize("dtype", FLOATS)
@pytest.mark.parametrize("axis", [0, 1, -1])
def test_file_bytes_and_native_restore(qdtype, dtype, axis, tmp_path, monkeypatch):
    src = sources(dtype)
    root = str(tmp_path / "s")
    snap = take(root, src, B.quantize_on_save(qdtype, axis=axis))
    for key in ("w", "w_t", "narrow", "cube"):
        x = src[key]
        ax = axis % x.dim()
        e, raw = file_of(snap, root, key)
        assert e.serializer == "per_channel_qtensor" and e.dtype == str(qdtype) and list(e.shape) == list(x.shape)
        assert raw == expected_file(x, qdtype, ax), key
        # the package's codec decodes it
        q = per_channel_qtensor_from_bytes(raw, qdtype, list(x.shape))
        assert q.q_per_channel_axis() == ax and torch.equal(q.int_repr(), torch.frombuffer(bytearray(raw[8 : 8 + x.numel()]), dtype=q.int_repr().dtype).reshape(x.shape))
    e, raw = file_of(snap, root, "bias")
    assert e.serializer == "buffer_protocol" and raw == src["bias"].contiguous().view(torch.uint8).numpy().tobytes()

    # restore runs through the engine, not the Python codec
    monkeypatch.setattr(TensorBufferConsumer, "deserialize_tensor", staticmethod(_no_codec))
    tgt = {k: torch.full_like(v, 123.0) for k, v in src.items()}
    B.Snapshot(root).restore({"m": B.StateDict(**tgt)})
    for key in ("w", "w_t", "narrow", "cube"):
        want = dequantized_like(src[key], qdtype, axis % src[key].dim())
        assert torch.equal(tgt[key], want), key
    assert torch.equal(tgt["bias"], src["bias"])


@pytest.mark.parametrize("target", [torch.float32, torch.bfloat16, torch.float64])
def test_restore_into_other_float_dtypes_and_views(target, tmp_path):
    x = torch.randn(33, 48)
    root = str(tmp_path / "s")
    take(root, {"w": x}, B.quantize_on_save(torch.qint8, axis=1))
    base = torch.zeros(48, 33, dtype=target)
    dst = base.t()  # a strided destination
    B.Snapshot(root).restore({"m": B.StateDict(w=dst)})
    want = torch.zeros(33, 48, dtype=target)
    scales, zps = per_channel_qparams(x, torch.qint8, 1)
    want.copy_(torch.quantize_per_channel(x, scales, zps, 1, torch.qint8).dequantize())
    assert torch.equal(dst, want)


def test_read_object_and_quantised_target_keep_python_path(tmp_path):
    x = torch.randn(20, 30)
    root = str(tmp_path / "s")
    take(root, {"w": x}, B.quantize_on_save(torch.quint8, axis=0))
    q = B.Snapshot(root).read_object("0/m/w")
    scales, zps = per_channel_qparams(x, torch.quint8, 0)
    want = torch.quantize_per_channel(x, scales, zps, 0, torch.quint8)
    assert q.is_quantized and q.qscheme() == torch.per_channel_affine
    assert torch.equal(q.int_repr(), want.int_repr()) and torch.equal(q.q_per_channel_scales(), want.q_per_channel_scales())


def test_chunked_tensor_pieces_have_their_own_parameters(tmp_path, monkeypatch):
    monkeypatch.setenv("TORCHSNAPSHOT_MAX_CHUNK_SIZE_BYTES_OVERRIDE", "4096")
    x = torch.randn(64, 48) * torch.linspace(0.1, 10, 64)[:, None]
    root = str(tmp_path / "s")
    snap = take(root, {"w": x}, B.quantize_on_save(torch.qint8, axis=-1))
    entry = snap.get_manifest()["0/m/w"]
    assert entry.type == "ChunkedTensor" and len(entry.chunks) > 1
    full = torch.zeros_like(x)
    for c in entry.chunks:
        assert c.tensor.serializer == "per_channel_qtensor"
        piece = x[c.offsets[0] : c.offsets[0] + c.sizes[0]]
        raw = open(os.path.join(root, c.tensor.location), "rb").read()
        assert raw == expected_file(piece, torch.qint8, 1)
        full[c.offsets[0] : c.offsets[0] + c.sizes[0]] = dequantized_like(piece, torch.qint8, 1)
    tgt = torch.zeros_like(x)
    B.Snapshot(root).restore({"m": B.StateDict(w=tgt)})
    assert torch.equal(tgt, full)


@pytest.mark.skipif(not HAVE_REF, reason="reference not staged under oracle/_ref")
def test_reference_codec_decodes_the_files(tmp_path):
    sys.path.insert(0, REF_PARENT)
    try:
        from torchsnapshot.serialization import per_channel_qtensor_from_bytes as ref_decode
    except Exception as e:  # the staged reference may not import on this torch
        pytest.skip(f"reference codec unavailable: {e}")
    finally:
        sys.path.remove(REF_PARENT)
    x = torch.randn(24, 40)
    root = str(tmp_path / "s")
    for axis in (0, 1):
        snap = take(root + str(axis), {"w": x}, B.quantize_on_save(torch.qint8, axis=axis))
        _, raw = file_of(snap, root + str(axis), "w")
        q = ref_decode(raw, torch.qint8, [24, 40])
        scales, zps = per_channel_qparams(x, torch.qint8, axis)
        want = torch.quantize_per_channel(x, scales, zps, axis, torch.qint8)
        assert torch.equal(q.int_repr(), want.int_repr()) and q.q_per_channel_axis() == axis


def test_api_errors_and_skips(tmp_path):
    with pytest.raises(ValueError):
        B.quantize_on_save(torch.qint8, qparams=lambda p, t: (1.0, 0), axis=0)
    hook = B.quantize_on_save(torch.qint8, axis=2)
    src = {"two_d": torch.randn(4, 5), "one_d": torch.randn(6), "ints": torch.arange(12).reshape(3, 4), "empty": torch.zeros(0, 3)}
    root = str(tmp_path / "s")
    snap = take(root, src, hook)
    for key in src:  # axis 2 applies to none of them
        assert snap.get_manifest()[f"0/m/{key}"].serializer == "buffer_protocol", key


def test_nonfinite_channel_fails_the_take(tmp_path):
    x = torch.randn(8, 8)
    x[3, 5] = float("nan")
    with pytest.raises(Exception, match="NaN or Inf"):
        take(str(tmp_path / "s"), {"w": x}, B.quantize_on_save(torch.qint8, axis=0))
    y = torch.randn(8, 8)
    y[1, 1] = float("inf")
    with pytest.raises(Exception, match="NaN or Inf"):
        take(str(tmp_path / "t"), {"w": y}, B.quantize_on_save(torch.quint8, axis=1))


def test_async_take_copies_cpu_sources(tmp_path):
    x = torch.randn(64, 32)
    want = expected_file(x, torch.qint8, 0)
    root = str(tmp_path / "s")
    pending = take(root, {"w": x}, B.quantize_on_save(torch.qint8, axis=0), async_=True)
    x.mul_(-3.0).add_(1.0)  # after async_take returned
    snap = pending.wait()
    _, raw = file_of(snap, root, "w")
    assert raw == want


def test_plugin_that_overrides_io_gets_the_same_bytes(tmp_path, monkeypatch):
    monkeypatch.setattr(SP, "FSStoragePlugin", Audited)
    src = sources(torch.float32)
    root = str(tmp_path / "s")
    snap = take(root, src, B.quantize_on_save(torch.qint8, axis=0))
    for key in ("w", "w_t", "narrow", "cube"):
        assert file_of(snap, root, key)[1] == expected_file(src[key], torch.qint8, 0), key
    tgt = {k: torch.zeros_like(v) for k, v in src.items()}
    B.Snapshot(root).restore({"m": B.StateDict(**tgt)})
    for key in ("w", "w_t", "narrow", "cube"):
        assert torch.equal(tgt[key], dequantized_like(src[key], torch.qint8, 0)), key


# ---- the C ABI directly ---------------------------------------------------------------------------------
def _host_save_desc(x, qdtype=torch.qint8, axis=0):
    d = _native.save_desc(x, 8, wire_dtype=qdtype, axis=axis)
    return d, 8 + x.numel() + 16 * x.shape[axis]


def test_host_execute_writes_the_format():
    x = torch.randn(12, 20)
    d, n = _host_save_desc(x, torch.quint8, 1)
    wire = bytearray(n)
    _native.host_execute([d], wire)
    assert bytes(wire) == expected_file(x, torch.quint8, 1)
    out = torch.zeros(12, 20)
    r = _native.per_channel(_native.load_desc(out, 8, wire_dtype=torch.quint8), [12, 20], 1, 8)
    _native.host_execute([r], wire)
    assert torch.equal(out, dequantized_like(x, torch.quint8, 1))


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
def test_malformed_qchannel_records_are_rejected(field, value, match):
    x = torch.randn(4, 6)
    d, n = _host_save_desc(x)
    setattr(d._qchannel, field, value)
    with pytest.raises(_native.NativeError, match=match):
        _native.host_execute([d], bytearray(n + 64))


def test_bad_scheme_and_missing_record_are_rejected():
    x = torch.randn(4, 6)
    d, n = _host_save_desc(x)
    d.reserved = 7
    with pytest.raises(_native.NativeError, match="quantisation scheme"):
        _native.host_execute([d], bytearray(n))
    d, n = _host_save_desc(x)
    d.q_zero_point = 0
    with pytest.raises(_native.NativeError, match="record"):
        _native.host_execute([d], bytearray(n))
    d, n = _host_save_desc(x)
    with pytest.raises(_native.NativeError, match="exceeds"):
        _native.host_execute([d], bytearray(n - 1))
    # per-channel pairs exist only for per-channel descriptors
    plain = _native.load_desc(torch.zeros(4, 6), 8, wire_dtype=torch.qint8)
    with pytest.raises(_native.NativeError):
        _native.host_execute([plain], bytearray(n))


def test_corrupt_header_and_size_give_clear_errors(tmp_path):
    _corrupt_header_and_size(tmp_path)


def test_corrupt_header_and_size_give_clear_errors_through_an_io_plugin(tmp_path, monkeypatch):
    """The stage / consume seam reads the layout from the buffer it is handed and fails the same way."""
    monkeypatch.setattr(SP, "FSStoragePlugin", Audited)
    _corrupt_header_and_size(tmp_path)


def _corrupt_header_and_size(tmp_path):
    x = torch.randn(10, 12)
    root = str(tmp_path / "s")
    snap = take(root, {"w": x}, B.quantize_on_save(torch.qint8, axis=0))
    e, raw = file_of(snap, root, "w")
    path = os.path.join(root, e.location)
    with open(path, "r+b") as f:
        f.write(struct.pack("<q", 3))
    with pytest.raises(RuntimeError, match="axis 3"):
        B.Snapshot(root).restore({"m": B.StateDict(w=torch.zeros(10, 12))})
    with open(path, "wb") as f:
        f.write(raw[:-8])
    with pytest.raises(RuntimeError, match="bytes"):
        B.Snapshot(root).restore({"m": B.StateDict(w=torch.zeros(10, 12))})


# ---- two gloo ranks: per-rank sharded pieces, restored resharded ---------------------------------------
ROWS, COLS = 24, 18


def _full():
    return torch.randn(ROWS, COLS, generator=torch.Generator().manual_seed(3)) * torch.linspace(0.5, 4, COLS)


def _worker(rank, world, store_path, root, audited):
    from torch.distributed._shard.sharded_tensor import Shard, ShardedTensor, ShardMetadata

    if audited:
        SP.FSStoragePlugin = Audited  # a process of its own
    dist.init_process_group("gloo", init_method=f"file://{store_path}", rank=rank, world_size=world)
    full, step = _full(), ROWS // world
    local = full[rank * step : (rank + 1) * step].contiguous()
    st = ShardedTensor._init_from_local_shards(
        [Shard(tensor=local, metadata=ShardMetadata(shard_offsets=[rank * step, 0], shard_sizes=[step, COLS], placement=f"rank:{rank}/cpu"))], (ROWS, COLS)
    )
    B.Snapshot.take(os.path.join(root, "snap"), {"m": B.StateDict(t=st)}, _custom_tensor_prepare_func=B.quantize_on_save(torch.qint8, axis=1))
    dist.barrier()
    # resharded restore: every rank reads a column band that crosses both saved pieces, and the engine dequantises it
    TensorBufferConsumer.deserialize_tensor = staticmethod(_no_codec)
    cols = COLS // world
    band = torch.zeros(ROWS, cols)
    tgt = ShardedTensor._init_from_local_shards(
        [Shard(tensor=band, metadata=ShardMetadata(shard_offsets=[0, rank * cols], shard_sizes=[ROWS, cols], placement=f"rank:{rank}/cpu"))], (ROWS, COLS)
    )
    B.Snapshot(os.path.join(root, "snap")).restore({"m": B.StateDict(t=tgt)})
    want = torch.cat([dequantized_like(full[r * step : (r + 1) * step], torch.qint8, 1) for r in range(world)])
    assert torch.equal(band, want[:, rank * cols : (rank + 1) * cols])
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_resharded_restore(tmp_path):
    _two_rank_resharded_restore(tmp_path, audited=False)


def test_two_rank_resharded_restore_through_an_io_plugin(tmp_path):
    """The stage / consume seam dequantises reshard overlaps on the engine as well."""
    _two_rank_resharded_restore(tmp_path, audited=True)


def _two_rank_resharded_restore(tmp_path, audited):
    store = tempfile.NamedTemporaryFile(delete=False)
    try:
        mp.spawn(_worker, args=(2, store.name, str(tmp_path), audited), nprocs=2, join=True)
    finally:
        if os.path.exists(store.name):
            os.unlink(store.name)
