"""quantize_on_save(float8 dtype, axis=...) on CUDA tensors: the statistics, parameter and scaled float8 pack kernels
write the bytes the torch statement of the rule (prepare.per_channel_fp8) gives on the same device, and the dequantising
scatter restores them natively."""
import os
import tempfile

import pytest
import torch
import torch.distributed as dist

pytestmark = pytest.mark.gpu

import torchsnapshot_b200 as B  # noqa: E402
from torchsnapshot_b200 import _native as N  # noqa: E402
from torchsnapshot_b200 import prepare as P  # noqa: E402
from torchsnapshot_b200 import scheduler as S  # noqa: E402
from torchsnapshot_b200 import storage_plugin as SP  # noqa: E402
from torchsnapshot_b200.io_preparers.tensor import TensorBufferConsumer  # noqa: E402
from torchsnapshot_b200.serialization import per_channel_fp8_as_bytes  # noqa: E402
from torchsnapshot_b200.storage_plugins.fs import FSStoragePlugin  # noqa: E402

DEV = "cuda:0"
FP8 = [torch.float8_e4m3fn, torch.float8_e5m2]
FLOATS = [torch.float64, torch.float32, torch.float16, torch.bfloat16]


def expected_file(x: torch.Tensor, fp8: torch.dtype, axis: int) -> bytes:
    """[axis][float8 bytes][f32 scales]: the rule computed by torch on x's device."""
    q, s = P.per_channel_fp8(x, fp8, axis)
    return per_channel_fp8_as_bytes(q, s, axis)


def restored_like(x: torch.Tensor, fp8: torch.dtype, axis: int, dtype=None) -> torch.Tensor:
    """(q.float() * s).to(dtype) on x's device"""
    q, s = P.per_channel_fp8(x, fp8, axis)
    return P.dequantize_fp8(q, s, axis).to(dtype or x.dtype)


def _no_codec(*a, **k):
    raise AssertionError("per-channel float8 restore fell back to the Python codec")


@pytest.fixture()
def fresh_engines():
    saved = {k: os.environ.get(k) for k in ("TSNAP_B200_ENGINE_FLAGS", "TSNAP_B200_HBM_STAGING_BYTES")}
    N.reset_engines()
    yield
    N.reset_engines()
    for k, v in saved.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


def _state():
    g = torch.Generator(device=DEV).manual_seed(11)
    scale = torch.logspace(-9, 3, 512, device=DEV)[:, None]
    return {
        "w": torch.randn(512, 1000, device=DEV, generator=g) * scale,          # channels of very different ranges
        "w_bf16": torch.randn(300, 257, device=DEV, generator=g).to(torch.bfloat16),
        "w_t": torch.randn(384, 96, device=DEV, generator=g).t(),              # transposed view
        "cols": torch.randn(128, 200, device=DEV, generator=g)[:, 13:170],     # narrowed, unaligned rows
        "cube": torch.randn(16, 24, 40, device=DEV, generator=g),
        "many_tiles": torch.randn(2048, 1024, device=DEV, generator=g),        # 2 MiB of float8: 16 save tiles
        "tall": torch.randn(4100, 64, device=DEV, generator=g),                # axis 0: more channels than a CTA table holds
        "wide": torch.randn(64, 4096, device=DEV, generator=g),                # axis 1: per-thread channel positions
        "bias": torch.randn(1000, device=DEV, generator=g),
    }


def _file(snap, root, key):
    e = snap.get_manifest()[f"0/m/{key}"]
    return e, open(os.path.join(root, e.location), "rb").read()


def _take_and_check(root, state, fp8, axis, **kw):
    snap = B.Snapshot.take(root, {"m": B.StateDict(**state)}, _custom_tensor_prepare_func=B.quantize_on_save(fp8, axis=axis), **kw)
    for key, x in state.items():
        e, raw = _file(snap, root, key)
        if x.dim() < 2:
            assert e.serializer == "buffer_protocol"
            continue
        assert e.serializer == "per_channel_fp8" and e.dtype == str(fp8), key
        assert raw == expected_file(x, fp8, axis % x.dim()), key
    return snap


@pytest.mark.parametrize("fp8", FP8)
@pytest.mark.parametrize("axis", [0, 1, -1])
def test_device_bytes_match_torch_and_restore_natively(fp8, axis, tmp_path, monkeypatch):
    state = _state()
    eng = B.get_engine(0)
    k0 = eng.stats()["kernels_launched"]

    def no_torch_rule(*a, **k):
        raise AssertionError("the take computed per-channel scales with torch")

    monkeypatch.setattr(P, "per_channel_fp8", no_torch_rule)
    for name in ("amax", "amin", "aminmax"):
        monkeypatch.setattr(torch.Tensor, name, no_torch_rule)
    root = str(tmp_path / "s")
    snap = B.Snapshot.take(root, {"m": B.StateDict(**state)}, _custom_tensor_prepare_func=B.quantize_on_save(fp8, axis=axis))
    monkeypatch.undo()
    assert eng.stats()["kernels_launched"] - k0 >= 3
    for key, x in state.items():
        e, raw = _file(snap, root, key)
        if x.dim() < 2:
            assert e.serializer == "buffer_protocol"
            continue
        assert raw == expected_file(x, fp8, axis % x.dim()), key

    monkeypatch.setattr(TensorBufferConsumer, "deserialize_tensor", staticmethod(_no_codec))
    h2d0 = eng.stats()["bytes_h2d"]
    tgt = {k: torch.full_like(v, 7.0) for k, v in state.items()}
    tgt["w_bf16"] = torch.zeros(300, 257, device=DEV)  # another float dtype on either side
    tgt["w"] = torch.zeros(512, 1000, device=DEV, dtype=torch.bfloat16)
    snap.restore({"m": B.StateDict(**tgt)})
    assert eng.stats()["bytes_h2d"] > h2d0
    for key, x in state.items():
        if x.dim() >= 2:
            assert torch.equal(tgt[key], restored_like(x, fp8, axis % x.dim(), tgt[key].dtype)), key


@pytest.mark.parametrize("fp8", FP8)
def test_native_restore_into_every_float_dtype(fp8, tmp_path, monkeypatch):
    g = torch.Generator(device=DEV).manual_seed(2)
    x = torch.randn(257, 1030, device=DEV, generator=g) * torch.logspace(-20, 20, 257, device=DEV)[:, None]
    root = str(tmp_path / "s")
    _take_and_check(root, {"w": x}, fp8, 0)
    monkeypatch.setattr(TensorBufferConsumer, "deserialize_tensor", staticmethod(_no_codec))
    for target in FLOATS:
        dense = torch.zeros(257, 1030, device=DEV, dtype=target)
        strided = torch.zeros(1030, 257, device=DEV, dtype=target).t()
        B.Snapshot(root).restore({"m": B.StateDict(w=dense)})
        B.Snapshot(root).restore({"m": B.StateDict(w=strided)})
        want = restored_like(x, fp8, 0, target)
        assert torch.equal(dense, want) and torch.equal(strided, want), target


def test_adam_like_state_keeps_every_nonzero(tmp_path):
    g = torch.Generator(device=DEV).manual_seed(3)
    rows = torch.logspace(-12, -7, 4096, device=DEV)[:, None]
    cols = torch.logspace(0, 2, 256, device=DEV)[None, :] / 100.0
    exp_avg_sq = torch.rand(4096, 256, device=DEV, generator=g) * rows * cols + 1e-12
    root = str(tmp_path / "s")
    _take_and_check(root, {"v": exp_avg_sq}, torch.float8_e4m3fn, 0)
    out = torch.zeros_like(exp_avg_sq)
    B.Snapshot(root).restore({"m": B.StateDict(v=out)})
    assert int((out == 0).sum()) == 0
    rel = ((out - exp_avg_sq).abs() / exp_avg_sq).median().item()
    assert rel < 0.07


def test_nonfinite_channel_fails_the_take(tmp_path):
    x = torch.randn(64, 64, device=DEV)
    x[10, 3] = float("nan")
    with pytest.raises(Exception, match="NaN or Inf"):
        B.Snapshot.take(str(tmp_path / "s"), {"m": B.StateDict(w=x)}, _custom_tensor_prepare_func=B.quantize_on_save(torch.float8_e4m3fn, axis=0))
    assert not os.path.exists(str(tmp_path / "s" / ".snapshot_metadata"))


def test_bounded_arena_multi_wave(tmp_path, fresh_engines):
    os.environ["TSNAP_B200_HBM_STAGING_BYTES"] = str(8 << 20)
    g = torch.Generator(device=DEV).manual_seed(5)
    state = {f"p{i}": torch.randn(1536, 1024, device=DEV, generator=g) for i in range(8)}  # 1.5 MiB of float8 each
    _take_and_check(str(tmp_path / "s"), state, torch.float8_e5m2, 0)
    st = max(S.LAST_STATS["save"], key=lambda j: j.get("n_waves", 0))
    assert st["n_waves"] >= 3 and st["arena_bytes"] <= (8 << 20)


def test_arena_less_mode_still_stages_per_channel_members(tmp_path, fresh_engines):
    os.environ["TSNAP_B200_ENGINE_FLAGS"] = str(N.ENGINE_NO_ARENA)
    g = torch.Generator(device=DEV).manual_seed(6)
    state = {"w": torch.randn(700, 300, device=DEV, generator=g), "dense": torch.randn(1 << 16, device=DEV, generator=g)}
    _take_and_check(str(tmp_path / "s"), state, torch.float8_e4m3fn, 1)
    st = max(S.LAST_STATS["save"], key=lambda j: j.get("n_kernel_launches", 0))
    assert st["arena_bytes"] > 0 and st["n_kernel_launches"] >= 3


def test_async_take_then_mutation_leaves_the_file(tmp_path):
    x = torch.randn(4096, 512, device=DEV)
    want = expected_file(x, torch.float8_e4m3fn, 0)
    root = str(tmp_path / "s")
    pending = B.Snapshot.async_take(root, {"m": B.StateDict(w=x)}, _custom_tensor_prepare_func=B.quantize_on_save(torch.float8_e4m3fn, axis=0))
    x.mul_(-2.0).add_(3.0)  # queued on the current stream after async_take returned
    snap = pending.wait()
    assert _file(snap, root, "w")[1] == want


class _AuditedFS(FSStoragePlugin):
    """Overrides write / read: the engine leaves the I/O to it and goes through the stage / consume seam."""

    async def write(self, write_io):
        return await super().write(write_io)

    async def read(self, read_io):
        return await super().read(read_io)


def test_plugin_seam_bytes_and_restore(tmp_path, monkeypatch):
    state = {k: v for k, v in _state().items() if k in ("w", "w_t", "cols", "bias")}
    monkeypatch.setattr(SP, "FSStoragePlugin", _AuditedFS)
    root = str(tmp_path / "s")
    _take_and_check(root, state, torch.float8_e5m2, 1)
    tgt = {k: torch.zeros_like(v) for k, v in state.items()}
    B.Snapshot(root).restore({"m": B.StateDict(**tgt)})
    for key, x in state.items():
        want = restored_like(x, torch.float8_e5m2, 1) if x.dim() >= 2 else x
        assert torch.equal(tgt[key], want), key


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

    fp8 = torch.float8_e4m3fn
    full = torch.randn(96, 160, device=DEV) * torch.logspace(-8, 0, 160, device=DEV)
    st = ShardedTensor._init_from_local_shards(
        [Shard(tensor=full[:, c : c + 80].contiguous(), metadata=ShardMetadata(shard_offsets=[0, c], shard_sizes=[96, 80], placement="rank:0/cuda:0")) for c in (0, 80)],
        (96, 160),
    )
    mesh = init_device_mesh("cuda", (1,))
    dt = DTensor.from_local(full.clone(), mesh, [DShard(1)], run_check=False)
    root = str(tmp_path / "s")
    snap = B.Snapshot.take(root, {"m": B.StateDict(st=st, dt=dt)}, _custom_tensor_prepare_func=B.quantize_on_save(fp8, axis=1))
    man = snap.get_manifest()
    for key in ("st", "dt"):
        for shard in man[f"0/m/{key}"].shards:
            assert shard.tensor.serializer == "per_channel_fp8"
            lo = shard.offsets
            piece = full[lo[0] : lo[0] + shard.sizes[0], lo[1] : lo[1] + shard.sizes[1]]
            assert open(os.path.join(root, shard.tensor.location), "rb").read() == expected_file(piece, fp8, 1)
    # resharded restore: column shards [0, 40) and [40, 160) cut the first saved piece in two (sub-boxes of its image)
    bands = [torch.zeros(96, 40, device=DEV), torch.zeros(96, 120, device=DEV)]
    tgt = ShardedTensor._init_from_local_shards(
        [Shard(tensor=b, metadata=ShardMetadata(shard_offsets=[0, c], shard_sizes=[96, b.shape[1]], placement="rank:0/cuda:0")) for b, c in zip(bands, (0, 40))],
        (96, 160),
    )
    dt_out = DTensor.from_local(torch.zeros(96, 160, device=DEV), mesh, [DShard(1)], run_check=False)
    h2d0 = B.get_engine(0).stats()["bytes_h2d"]
    B.Snapshot(root).restore({"m": B.StateDict(st=tgt, dt=dt_out)})
    assert B.get_engine(0).stats()["bytes_h2d"] > h2d0
    cols = torch.cat([restored_like(full[:, c : c + 80], fp8, 1) for c in (0, 80)], dim=1)
    assert torch.equal(torch.cat(bands, dim=1), cols)
    # the DTensor's saved pieces: whatever the planner cut, each restored piece equals the rule applied to it
    got = dt_out.to_local()
    for shard in man["0/m/dt"].shards:
        lo, sz = shard.offsets, shard.sizes
        piece = full[lo[0] : lo[0] + sz[0], lo[1] : lo[1] + sz[1]]
        assert torch.equal(got[lo[0] : lo[0] + sz[0], lo[1] : lo[1] + sz[1]], restored_like(piece, fp8, 1))
