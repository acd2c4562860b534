"""torch.float8_e4m3fn / torch.float8_e5m2 on the device: the LSU cast path (16 B vector path, ragged tails, tile seams,
scalar strided path, unaligned wire sides) against torch's Tensor.to / copy_ on the same device, NaN bits included, and
raw and converting fp8 snapshots through the API."""
import os
import tempfile

import pytest
import torch
import torch.distributed as dist

import torchsnapshot_b200 as B
from tests.conversion_cases import FLOATS, LAYOUTS, SAVE_LAYOUTS
from tests.float8_cases import FP8, FP8_PAIRS, restore_case, same_values, save_case
from tests.test_float8_cpu import FROM_FP8, NAMED, _PAIR_IDS, _image, _name, _payload
from torchsnapshot_b200 import _native as N
from torchsnapshot_b200 import scheduler as S
from torchsnapshot_b200 import storage_plugin as SP
from torchsnapshot_b200.storage_plugins.fs import FSStoragePlugin

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
_TILE = 128 << 10  # LSU tile: destination bytes
E4, E5 = torch.float8_e4m3fn, torch.float8_e5m2


@pytest.fixture(scope="module")
def engine():
    eng = N.Engine(device=0, io_threads=2, pinned_slot_bytes=4 << 20, pinned_slots=4)
    yield eng
    eng.close()


def _stage(engine, descs, nbytes, keep) -> torch.Tensor:
    sb = engine.stage(descs, nbytes, stream=torch.cuda.current_stream().cuda_stream, keepalive=keep)
    got = torch.frombuffer(bytearray(sb.wait()), dtype=torch.uint8)
    sb.release()
    return got


def _on_lsu_cast_path(desc, nbytes):
    info = N.plan_describe([desc])
    assert info["n_members_lsu"] == 1 and info["n_members_bulk"] == info["n_members_rows"] == info["n_members_host"] == 0, info
    assert info["n_tiles_lsu"] == -(-nbytes // _TILE), info


def _device_cast(engine, x: torch.Tensor, dst: torch.dtype) -> torch.Tensor:
    desc = N.save_desc(x, 0, wire_dtype=dst)
    n = x.numel() * torch.empty(0, dtype=dst).element_size()
    _on_lsu_cast_path(desc, n)
    return _stage(engine, [desc], n, [x]).view(dst)


@pytest.mark.parametrize("layout", SAVE_LAYOUTS, ids=lambda l: l.name)
@pytest.mark.parametrize("src,dst", FP8_PAIRS, ids=_PAIR_IDS)
def test_cast_on_save(engine, src, dst, layout):
    c = save_case(layout, src, dst, DEV)
    n = c.expected.numel() * c.expected.element_size()
    desc = N.save_desc(c.view, c.offset, wire_dtype=dst)
    _on_lsu_cast_path(desc, n)
    if layout.name.startswith("dense"):
        assert n > _TILE  # the vector path crosses a tile seam
    pre = torch.full((c.offset,), 0xA5, dtype=torch.uint8, device=DEV)
    got = _stage(engine, ([N.save_desc(pre, 0)] if c.offset else []) + [desc], c.offset + n, [pre, c.view])
    assert bool((got[: c.offset] == 0xA5).all())
    err = same_values(got[c.offset :].clone().view(dst), c.expected.cpu(), nan_bits=True)
    assert err is None, err


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: l.name)
@pytest.mark.parametrize("src,dst", FP8_PAIRS, ids=_PAIR_IDS)
def test_cast_on_restore(engine, src, dst, layout):
    c = restore_case(layout, src, dst, DEV)
    desc = N.load_desc(c.view, c.desc_offset, wire_dtype=src, wire_strides=c.wire_strides)
    _on_lsu_cast_path(desc, c.view.numel() * c.view.element_size())
    engine.consume(c.wire.cpu().numpy(), [desc])
    torch.cuda.synchronize()
    err = same_values(c.storage.cpu(), c.expected.cpu(), nan_bits=True)
    assert err is None, err


@pytest.mark.parametrize("src,dst", FROM_FP8, ids=[f"{_name(s)}-{_name(d)}" for s, d in FROM_FP8])
def test_every_fp8_pattern(engine, src, dst):
    x = torch.arange(256 * 67 + 5, dtype=torch.int32).remainder(256).to(torch.uint8).view(src).to(DEV)  # 16 B groups and a tail
    err = same_values(_device_cast(engine, x, dst), x.to(dst).cpu(), nan_bits=True)
    assert err is None, err
    err = same_values(_device_cast(engine, x[1:], dst), x[1:].to(dst).cpu(), nan_bits=True)  # unaligned: scalar path
    assert err is None, err


@pytest.mark.parametrize("dst", FP8, ids=_name)
@pytest.mark.parametrize("src", [torch.float16, torch.bfloat16], ids=_name)
def test_every_16_bit_pattern(engine, src, dst):
    x = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(src).to(DEV)
    err = same_values(_device_cast(engine, x, dst), x.to(dst).cpu(), nan_bits=True)
    assert err is None, err


@pytest.mark.parametrize("src", [torch.float32, torch.float64], ids=_name)
def test_named_values(engine, src):
    x = torch.tensor([v for v, _, _ in NAMED] * 3, dtype=src, device=DEV)  # vector path (fp32) and tail
    for dst, col in ((E4, 1), (E5, 2)):
        got = _device_cast(engine, x, dst).view(torch.uint8).tolist()
        assert got == [r[col] for r in NAMED] * 3, _name(dst)
        assert got == x.to(dst).view(torch.uint8).cpu().tolist(), _name(dst)


# ---- through the API --------------------------------------------------------------------------------------------
def _fp8(shape, dtype, seed=0) -> torch.Tensor:
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(tuple(shape), generator=g, device=DEV) * 8).to(dtype)


def _same(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.dtype == b.dtype and torch.equal(a.view(torch.uint8) if a.element_size() == 1 else a, b.view(torch.uint8) if b.element_size() == 1 else b)


@pytest.mark.parametrize("dtype", FP8, ids=_name)
def test_raw_save_on_the_bulk_path_and_transposed_view(dtype, tmp_path):
    big = _fp8((2048, 1536), dtype, 1)
    assert N.plan_describe([N.save_desc(big, 0)])["n_tiles_bulk"] > 0
    base = _fp8((257, 130), dtype, 2)
    state = {"big": big, "t": base.t(), "scalar": _fp8((), dtype, 3), "odd": _fp8((33,), dtype, 4)}
    root = str(tmp_path / "s")
    snap = B.Snapshot.take(root, {"m": B.StateDict(**state)})
    for k, v in state.items():
        assert snap.get_manifest()[f"0/m/{k}"].dtype == str(dtype)
        assert _payload(snap, root, k) == _image(v.cpu()), k
    tgt = {k: torch.zeros_like(v) for k, v in state.items()}
    tgt["t"] = torch.zeros_like(base).t()
    B.Snapshot(root).restore({"m": B.StateDict(**tgt)})
    for k, v in state.items():
        assert _same(tgt[k], v), k


@pytest.fixture(scope="module")
def pg():
    if not dist.is_initialized():
        f = tempfile.NamedTemporaryFile(delete=False)
        dist.init_process_group("gloo", init_method=f"file://{f.name}", rank=0, world_size=1)
    yield
    if dist.is_initialized():
        dist.destroy_process_group()


def test_sharded_and_dtensor_column_shards(pg, tmp_path):
    from torch.distributed._shard.sharded_tensor import Shard, ShardedTensor, ShardMetadata
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.tensor import DTensor, Shard as DShard

    full = _fp8((96, 160), E4, 5)
    st = ShardedTensor._init_from_local_shards(
        [Shard(tensor=full[:, c : c + 80].contiguous(), metadata=ShardMetadata(shard_offsets=[0, c], shard_sizes=[96, 80], placement="rank:0/cuda:0")) for c in (0, 80)],
        (96, 160),
    )
    mesh = init_device_mesh("cuda", (1,))
    dt = DTensor.from_local(full.clone(), mesh, [DShard(1)], run_check=False)
    root = str(tmp_path / "s")
    snap = B.Snapshot.take(root, {"m": B.StateDict(st=st, dt=dt)})
    for key in ("st", "dt"):
        for shard in snap.get_manifest()[f"0/m/{key}"].shards:
            assert shard.tensor.dtype == str(E4)
    # resharded restore into column bands that cut a saved piece, once as fp8 and once converted to bf16
    for dtype in (E4, torch.bfloat16):
        bands = [torch.zeros(96, 40, dtype=dtype, device=DEV), torch.zeros(96, 120, dtype=dtype, device=DEV)]
        tgt = ShardedTensor._init_from_local_shards(
            [Shard(tensor=b, metadata=ShardMetadata(shard_offsets=[0, c], shard_sizes=[96, b.shape[1]], placement="rank:0/cuda:0")) for b, c in zip(bands, (0, 40))],
            (96, 160),
        )
        dt_out = DTensor.from_local(torch.zeros(96, 160, dtype=dtype, device=DEV), mesh, [DShard(1)], run_check=False)
        B.Snapshot(root).restore({"m": B.StateDict(st=tgt, dt=dt_out)})
        want = full.to(dtype)
        assert _same(bands[0], want[:, :40]) and _same(bands[1], want[:, 40:]), dtype
        assert _same(dt_out.to_local(), want), dtype


def test_async_take_then_mutation_leaves_the_file(tmp_path):
    x = torch.randn(4096, 512, device=DEV) * 100
    want = _image(x.to(E4).cpu())
    root = str(tmp_path / "s")
    pending = B.Snapshot.async_take(root, {"m": B.StateDict(w=x)}, _custom_tensor_prepare_func=B.cast_on_save(E4))
    x.mul_(-2.0).add_(3.0)  # queued on the current stream after async_take returned
    snap = pending.wait()
    assert _payload(snap, root, "w") == want


@pytest.fixture()
def fresh_engines():
    saved = os.environ.get("TSNAP_B200_ENGINE_FLAGS")
    N.reset_engines()
    yield
    N.reset_engines()
    if saved is None:
        os.environ.pop("TSNAP_B200_ENGINE_FLAGS", None)
    else:
        os.environ["TSNAP_B200_ENGINE_FLAGS"] = saved


def _cast_take_and_restore(root, state, dtype=E5):
    snap = B.Snapshot.take(root, {"m": B.StateDict(**state)}, _custom_tensor_prepare_func=B.cast_on_save(dtype))
    for k, v in state.items():
        assert _payload(snap, root, k) == _image(v.to(dtype).cpu()), k
    tgt = {k: torch.zeros(v.shape, dtype=dtype, device=DEV) for k, v in state.items()}
    B.Snapshot(root).restore({"m": B.StateDict(**tgt)})
    for k, v in state.items():
        assert _same(tgt[k], v.to(dtype)), k


def test_arena_less_mode(tmp_path, fresh_engines):
    os.environ["TSNAP_B200_ENGINE_FLAGS"] = str(N.ENGINE_NO_ARENA)
    g = torch.Generator(device=DEV).manual_seed(6)
    state = {"w": torch.randn(700, 300, device=DEV, generator=g), "h": torch.randn(1 << 16, device=DEV, generator=g).to(torch.bfloat16)}
    _cast_take_and_restore(str(tmp_path / "s"), state)
    st = max(S.LAST_STATS["save"], key=lambda j: j.get("n_kernel_launches", 0))
    assert st["n_kernel_launches"] >= 1


class _AuditedFS(FSStoragePlugin):
    """Overrides write / read: the engine leaves the I/O to it and goes through the stage / consume seam."""

    async def write(self, write_io):
        return await super().write(write_io)

    async def read(self, read_io):
        return await super().read(read_io)


def test_plugin_seam(tmp_path, monkeypatch):
    monkeypatch.setattr(SP, "FSStoragePlugin", _AuditedFS)
    g = torch.Generator(device=DEV).manual_seed(7)
    state = {"w": torch.randn(300, 257, device=DEV, generator=g).t(), "h": torch.randn(4099, device=DEV, generator=g).to(torch.float16)}
    _cast_take_and_restore(str(tmp_path / "s"), state)


def test_bf16_model_cast_to_e4m3fn_restores_into_bf16(tmp_path, pg):
    from torch.distributed._shard.sharded_tensor import Shard, ShardedTensor, ShardMetadata

    g = torch.Generator(device=DEV).manual_seed(8)
    w = (torch.randn(1024, 768, device=DEV, generator=g) * 30).to(torch.bfloat16)
    md = ShardMetadata(shard_offsets=[0, 0], shard_sizes=[1024, 768], placement="rank:0/cuda:0")
    root = str(tmp_path / "s")
    B.Snapshot.take(root, {"m": B.StateDict(w=ShardedTensor._init_from_local_shards([Shard(tensor=w, metadata=md)], (1024, 768)))},
                    _custom_tensor_prepare_func=B.cast_on_save(E4))
    out = torch.zeros_like(w)
    k0 = B.get_engine(0).stats()["kernels_launched"]
    B.Snapshot(root).restore({"m": B.StateDict(w=ShardedTensor._init_from_local_shards([Shard(tensor=out, metadata=md)], (1024, 768)))})
    assert B.get_engine(0).stats()["kernels_launched"] > k0  # converted by the scatter kernel
    err = same_values(out.cpu(), w.to(E4).to(torch.bfloat16).cpu(), nan_bits=True)
    assert err is None, err
