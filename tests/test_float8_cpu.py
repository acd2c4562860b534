"""torch.float8_e4m3fn / torch.float8_e5m2 on the host engine and through the API, against torch on the CPU: raw fp8
snapshots, cast_on_save to fp8, and restores that convert between fp8 and the wide floats.  Bit-exact, except that NaNs
are compared by position: torch's CPU NaN encoding depends on which of its loops ran (e5m2 -> fp32 quiets a NaN in the
vectorised loop and keeps its payload in the scalar one)."""
import os
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import torchsnapshot_b200 as B
from tests.conversion_cases import FLOATS, LAYOUTS, SAVE_LAYOUTS
from tests.float8_cases import FP8, FP8_PAIRS, every_pattern, restore_case, same_values, save_case
from torchsnapshot_b200 import _native as N
from torchsnapshot_b200.native_plan import raw_castable
from torchsnapshot_b200.serialization import ALL_SUPPORTED_DTYPES, BUFFER_PROTOCOL_SUPPORTED_DTYPES

_name = lambda dt: str(dt).replace("torch.", "")
_PAIR_IDS = [f"{_name(s)}-{_name(d)}" for s, d in FP8_PAIRS]
E4, E5 = torch.float8_e4m3fn, torch.float8_e5m2


def host_cast(x: torch.Tensor, dst: torch.dtype) -> torch.Tensor:
    """The host engine's wire image of `x` cast to `dst`."""
    wire = torch.full((x.numel() * torch.empty(0, dtype=dst).element_size(),), 0xA5, dtype=torch.uint8)
    N.host_execute([N.save_desc(x, 0, wire_dtype=dst)], wire)
    return wire.view(dst)


def test_pairs():
    assert len(FP8_PAIRS) == 18


@pytest.mark.parametrize("layout", SAVE_LAYOUTS, ids=lambda l: l.name)
@pytest.mark.parametrize("src,dst", FP8_PAIRS, ids=_PAIR_IDS)
def test_cast_on_save(src, dst, layout):
    c = save_case(layout, src, dst, "cpu")
    ed = torch.empty(0, dtype=dst).element_size()
    wire = torch.full((c.offset + c.expected.numel() * ed,), 0xA5, dtype=torch.uint8)
    N.host_execute([N.save_desc(c.view, c.offset, wire_dtype=dst)], wire)
    assert bool((wire[: c.offset] == 0xA5).all())
    err = same_values(wire[c.offset :].clone().view(dst), c.expected, nan_bits=False)
    assert err is None, err


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: l.name)
@pytest.mark.parametrize("src,dst", FP8_PAIRS, ids=_PAIR_IDS)
def test_cast_on_restore(src, dst, layout):
    c = restore_case(layout, src, dst, "cpu")
    N.host_execute([N.load_desc(c.view, c.desc_offset, wire_dtype=src, wire_strides=c.wire_strides)], c.wire)
    err = same_values(c.storage, c.expected, nan_bits=False)
    assert err is None, err


# ---- exhaustive sources and named values ------------------------------------------------------------------------
FROM_FP8 = [(s, d) for s, d in FP8_PAIRS if s in FP8]


@pytest.mark.parametrize("src,dst", FROM_FP8, ids=[f"{_name(s)}-{_name(d)}" for s, d in FROM_FP8])
def test_every_fp8_pattern(src, dst):
    x = every_pattern(src)
    err = same_values(host_cast(x, dst), x.to(dst), nan_bits=False)
    assert err is None, err


@pytest.mark.parametrize("dst", FP8, ids=_name)
@pytest.mark.parametrize("src", [torch.float16, torch.bfloat16], ids=_name)
def test_every_16_bit_pattern(src, dst):
    x = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(src)
    err = same_values(host_cast(x, dst), x.to(dst), nan_bits=True)  # the result of a narrowing has one NaN per sign
    assert err is None, err


# (value, e4m3fn bits, e5m2 bits): the rounding rules torch applies, spelled out
NAMED = [
    (0.0, 0x00, 0x00), (-0.0, 0x80, 0x80), (448.0, 0x7E, 0x5F), (464.0, 0x7E, 0x5F), (464.0 + 2**-10, 0x7F, 0x5F),
    (479.0, 0x7F, 0x5F), (1e30, 0x7F, 0x7C), (float("inf"), 0x7F, 0x7C), (float("-inf"), 0xFF, 0xFC),
    (float("nan"), 0x7F, 0x7F), (57344.0, 0x7F, 0x7B), (61439.0, 0x7F, 0x7B), (61440.0, 0x7F, 0x7C), (-61440.0, 0xFF, 0xFC),
    (2.0**-9, 0x01, 0x18), (2.0**-10, 0x00, 0x14), (1.5 * 2**-10, 0x01, 0x16), (2.0**-16, 0x00, 0x01), (2.0**-17, 0x00, 0x00),
    (1.5 * 2**-17, 0x00, 0x01), (1.0625, 0x38, 0x3C), (1.1875, 0x3A, 0x3D), (1.125, 0x39, 0x3C), (1.375, 0x3B, 0x3E),
]


@pytest.mark.parametrize("src", [torch.float32, torch.float64], ids=_name)
def test_named_values(src):
    x = torch.tensor([v for v, _, _ in NAMED], dtype=src)
    for dst, col in ((E4, 1), (E5, 2)):
        got = host_cast(x, dst).view(torch.uint8).tolist()
        assert got == [r[col] for r in NAMED], _name(dst)
        assert got == x.to(dst).view(torch.uint8).tolist(), _name(dst)


def test_fp64_rounds_through_fp32():
    # rounding once would give 0x39 (e4m3fn) and 0x3D (e5m2): fp32 lands on the tie first, which rounds to even
    x = torch.tensor([1.0625 + 2**-30, 1.125 + 2**-30], dtype=torch.float64)
    assert host_cast(x[:1], E4).view(torch.uint8).tolist() == [0x38] == x[:1].to(E4).view(torch.uint8).tolist()
    assert host_cast(x[1:], E5).view(torch.uint8).tolist() == [0x3C] == x[1:].to(E5).view(torch.uint8).tolist()


def test_planner_rules():
    assert N.plan_describe([N.save_desc(torch.zeros(64, dtype=E4), 0)])["n_members_host"] == 1
    for f8 in FP8:
        with pytest.raises(N.NativeError, match="-6"):
            N.plan_describe([N.save_desc(torch.zeros(64, dtype=f8), 0, wire_dtype=torch.qint8, qparams=(0.5, 0))])
        for other in FLOATS + FP8:
            assert raw_castable(f8, other) and raw_castable(other, f8)
        assert not raw_castable(f8, torch.int8) and not raw_castable(torch.int32, f8)


def test_public_dtype_lists_are_the_references():
    assert not set(FP8) & set(ALL_SUPPORTED_DTYPES) and not set(FP8) & set(BUFFER_PROTOCOL_SUPPORTED_DTYPES)
    assert len(ALL_SUPPORTED_DTYPES) == 15 and len(BUFFER_PROTOCOL_SUPPORTED_DTYPES) == 10


# ---- through the API --------------------------------------------------------------------------------------------
def _fp8(shape, dtype, seed=0) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(tuple(shape), generator=g) * 8).to(dtype)


def _payload(snap, root, key) -> bytes:
    e = snap.get_manifest()[f"0/m/{key}"]
    raw = open(os.path.join(root, e.location), "rb").read()
    return raw if e.byte_range is None else raw[e.byte_range[0] : e.byte_range[1]]


def _image(t: torch.Tensor) -> bytes:
    return t.contiguous().view(torch.uint8).numpy().tobytes()


@pytest.mark.parametrize("dtype", FP8, ids=_name)
def test_raw_snapshot_round_trip(dtype, tmp_path):
    base = _fp8((40, 33), dtype)
    state = {"dense": base, "view": base.t()[3:30], "scalar": _fp8((), dtype, 1), "empty": torch.empty(0, 5, dtype=dtype),
             "big": _fp8((300, 257), dtype, 2)}
    root = str(tmp_path / "s")
    snap = B.Snapshot.take(root, {"m": B.StateDict(**state)})
    man = snap.get_manifest()
    for k, v in state.items():
        e = man[f"0/m/{k}"]
        assert e.dtype == str(dtype) and e.serializer == "buffer_protocol" and list(e.shape) == list(v.shape), k
        assert _payload(snap, root, k) == _image(v), k
        got = B.Snapshot(root).read_object(f"0/m/{k}")
        assert got.dtype == dtype and got.device.type == "cpu" and torch.equal(got.view(torch.uint8), v.view(torch.uint8)), k
    tgt = {k: torch.zeros_like(v) for k, v in state.items()}
    tgt["view"] = torch.zeros_like(base).t()[3:30]
    B.Snapshot(root).restore({"m": B.StateDict(**tgt)})
    for k, v in state.items():
        assert torch.equal(tgt[k].view(torch.uint8), v.view(torch.uint8)), k


def test_chunked_and_slabbed(tmp_path, monkeypatch):
    monkeypatch.setenv("TORCHSNAPSHOT_MAX_CHUNK_SIZE_BYTES_OVERRIDE", "4096")
    state = {"chunked": _fp8((100, 97), E4, 3), "a": _fp8((7,), E5, 4), "b": _fp8((13, 3), E4, 5), "c": torch.randn(5),
             "flag": torch.tensor([True, False, True])}
    root = str(tmp_path / "s")
    snap = B.Snapshot.take(root, {"m": B.StateDict(**state)})
    man = snap.get_manifest()
    assert len(man["0/m/chunked"].chunks) > 1
    assert man["0/m/a"].location == man["0/m/b"].location == man["0/m/c"].location  # one slab, odd-sized members
    for k in ("a", "b", "c"):
        assert _payload(snap, root, k) == _image(state[k]), k
    tgt = {k: torch.zeros_like(v) for k, v in state.items()}
    B.Snapshot(root).restore({"m": B.StateDict(**tgt)})
    for k, v in state.items():
        assert torch.equal(tgt[k].view(torch.uint8), v.view(torch.uint8)), k
    assert torch.equal(B.Snapshot(root).read_object("0/m/chunked").view(torch.uint8), state["chunked"].view(torch.uint8))


def _sharded(t: torch.Tensor):
    from torch.distributed._shard.sharded_tensor import Shard, ShardedTensor, ShardMetadata

    md = ShardMetadata(shard_offsets=[0] * t.dim(), shard_sizes=list(t.shape), placement="rank:0/cpu")
    return ShardedTensor._init_from_local_shards([Shard(tensor=t, metadata=md)], tuple(t.shape))


@pytest.fixture(scope="module")
def pg():
    if not dist.is_initialized():
        f = tempfile.NamedTemporaryFile(delete=False)
        dist.init_process_group("gloo", init_method=f"file://{f.name}", rank=0, world_size=1)
    yield
    if dist.is_initialized():
        dist.destroy_process_group()


def _module(x: torch.Tensor) -> torch.nn.Module:
    mod = torch.nn.Module()
    mod.p = torch.nn.Parameter(x, requires_grad=False)
    return mod


@pytest.mark.parametrize("saved,target", [(E4, torch.bfloat16), (E5, torch.float32), (torch.bfloat16, E4), (torch.float32, E5), (E4, E5)],
                         ids=lambda v: _name(v))
def test_restore_converts(saved, target, tmp_path, pg):
    """Into a sharded target (the engine converts) and into a module's parameter (load_state_dict copies)."""
    x = (torch.randn(24, 40, generator=torch.Generator().manual_seed(6)) * 100).to(saved)
    root = str(tmp_path / "s")
    B.Snapshot.take(root, {"m": B.StateDict(w=_sharded(x.clone())), "mod": _module(x.clone())})
    tw = torch.zeros(24, 40, dtype=target)
    mod = _module(torch.zeros(24, 40, dtype=target))
    B.Snapshot(root).restore({"m": B.StateDict(w=_sharded(tw)), "mod": mod})
    want = x.to(target)
    for got in (tw, mod.p.data):
        assert got.dtype == target
        err = same_values(got, want, nan_bits=False)
        assert err is None, err


def test_cast_on_save_to_fp8(tmp_path):
    state = {"model.w": torch.randn(50, 30) * 100, "model.b": torch.randn(30, dtype=torch.float64), "opt.m": torch.randn(50, 30),
             "model.h": torch.randn(9, 7).to(torch.bfloat16), "model.f8": _fp8((6,), E5, 8), "model.i": torch.arange(5)}
    root = str(tmp_path / "s")
    snap = B.Snapshot.take(root, {"m": B.StateDict(**state)}, _custom_tensor_prepare_func=B.cast_on_save(E4, only="m/model.*"))
    man = snap.get_manifest()
    for k, v in state.items():
        e = man[f"0/m/{k}"]
        cast = k.startswith("model.") and v.dtype in FLOATS
        assert e.dtype == str(E4 if cast else v.dtype), k
        assert _payload(snap, root, k) == _image(v.to(E4) if cast else v), k
    for f8 in FP8:
        assert B.cast_on_save(f8) is not None
    with pytest.raises(ValueError):
        B.cast_on_save(torch.float8_e4m3fnuz)


def test_quantize_on_save_leaves_fp8_alone(tmp_path):
    state = {"w": torch.randn(20, 30), "f": _fp8((20, 30), E4, 9)}
    for hook in (B.quantize_on_save(torch.qint8), B.quantize_on_save(torch.quint8, axis=0)):
        root = str(tmp_path / f"s{id(hook)}")
        snap = B.Snapshot.take(root, {"m": B.StateDict(**state)}, _custom_tensor_prepare_func=hook)
        e = snap.get_manifest()["0/m/f"]
        assert e.serializer == "buffer_protocol" and e.dtype == str(E4)
        assert _payload(snap, root, "f") == _image(state["f"])


@pytest.mark.parametrize("dtype", [torch.float8_e4m3fnuz, torch.float8_e5m2fnuz], ids=_name)
def test_other_float8_formats_stay_unsupported(dtype, tmp_path):
    with pytest.raises(ValueError, match="Unsupported dtype"):
        B.Snapshot.take(str(tmp_path / "s"), {"m": B.StateDict(x=torch.zeros(4).to(dtype))})


# ---- two gloo ranks: fp8 pieces restored resharded --------------------------------------------------------------
ROWS, COLS = 24, 18


def _full():
    return (torch.randn(ROWS, COLS, generator=torch.Generator().manual_seed(3)) * 50).to(E4)


def _worker(rank, world, store_path, root):
    from torch.distributed._shard.sharded_tensor import Shard, ShardedTensor, ShardMetadata

    dist.init_process_group("gloo", init_method=f"file://{store_path}", rank=rank, world_size=world)
    full, step = _full(), ROWS // world
    local = full[rank * step : (rank + 1) * step].contiguous()
    st = ShardedTensor._init_from_local_shards(
        [Shard(tensor=local, metadata=ShardMetadata(shard_offsets=[rank * step, 0], shard_sizes=[step, COLS], placement=f"rank:{rank}/cpu"))], (ROWS, COLS)
    )
    B.Snapshot.take(os.path.join(root, "snap"), {"m": B.StateDict(t=st)})
    dist.barrier()
    # every rank reads a column band that crosses both saved pieces: once as fp8, once converted to bf16
    cols = COLS // world
    for dtype in (E4, torch.bfloat16):
        band = torch.zeros(ROWS, cols, dtype=dtype)
        tgt = ShardedTensor._init_from_local_shards(
            [Shard(tensor=band, metadata=ShardMetadata(shard_offsets=[0, rank * cols], shard_sizes=[ROWS, cols], placement=f"rank:{rank}/cpu"))], (ROWS, COLS)
        )
        B.Snapshot(os.path.join(root, "snap")).restore({"m": B.StateDict(t=tgt)})
        want = full[:, rank * cols : (rank + 1) * cols].to(dtype)
        assert torch.equal(band.view(torch.uint8) if dtype == E4 else band, want.view(torch.uint8) if dtype == E4 else want)
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_resharded_restore(tmp_path):
    store = tempfile.NamedTemporaryFile(delete=False)
    try:
        mp.spawn(_worker, args=(2, store.name, str(tmp_path)), nprocs=2, join=True)
    finally:
        if os.path.exists(store.name):
            os.unlink(store.name)
