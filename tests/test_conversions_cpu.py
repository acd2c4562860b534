"""The host engine's converting and quantising copies against torch on the CPU, at the values and layouts where
conversions go wrong (tests/conversion_cases.py).  Bit-exact, except that NaNs are compared by position: torch's CPU
NaN encoding depends on which of its loops ran."""
import os
import struct
import tempfile

import pytest
import torch
import torch.distributed as dist

import torchsnapshot_b200 as B
from tests.conversion_cases import (FLOATS, PAIRS, LAYOUTS, SAVE_LAYOUTS, case_values, restore_case, same_values,
                                    save_case, tie_channels, tie_values)
from torchsnapshot_b200 import _native as N
from torchsnapshot_b200.prepare import per_channel_qparams

_name = lambda dt: str(dt).replace("torch.", "")


@pytest.mark.parametrize("layout", SAVE_LAYOUTS, ids=lambda l: l.name)
@pytest.mark.parametrize("src,dst", PAIRS, ids=[f"{_name(s)}-{_name(d)}" for s, d in PAIRS])
def test_cast_on_save(src, dst, layout):
    c = save_case(layout, src, dst, "cpu")
    ed = torch.empty(0, dtype=dst).element_size()
    wire = torch.full((c.offset + c.expected.numel() * ed,), 0xA5, dtype=torch.uint8)
    N.host_execute([N.save_desc(c.view, c.offset, wire_dtype=dst)], wire)
    assert bool((wire[: c.offset] == 0xA5).all())
    err = same_values(wire[c.offset :].clone().view(dst), c.expected, nan_bits=False)
    assert err is None, err


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: l.name)
@pytest.mark.parametrize("src,dst", PAIRS, ids=[f"{_name(s)}-{_name(d)}" for s, d in PAIRS])
def test_cast_on_restore(src, dst, layout):
    c = restore_case(layout, src, dst, "cpu")
    N.host_execute([N.load_desc(c.view, c.desc_offset, wire_dtype=src, wire_strides=c.wire_strides)], c.wire)
    err = same_values(c.storage, c.expected, nan_bits=False)
    assert err is None, err


# scales that are not powers of two; quint8 zero points at both ends and the middle of the range
QPARAMS = [(torch.qint8, 0.0123, 0), (torch.qint8, 1 / 3, 0), (torch.quint8, 0.37, 0), (torch.quint8, 0.0123, 128), (torch.quint8, 2.5e-3, 255)]


def _per_tensor_expected(view, scale, zp, qdtype) -> bytes:
    q = torch.quantize_per_tensor(view.float(), scale, zp, qdtype)
    return q.int_repr().contiguous().cpu().numpy().tobytes() + struct.pack("<dq", scale, zp)


@pytest.mark.parametrize("src", FLOATS, ids=_name)
@pytest.mark.parametrize("qdtype,scale,zp", QPARAMS)
def test_quantize_per_tensor_at_ties(qdtype, scale, zp, src):
    x = tie_values(scale, zp, qdtype).to(src)
    n = x.numel() // 3 * 3
    for view, off in ((x, 0), (x[:n].view(3, -1).t(), 0), (x[:n].view(3, -1)[:, 5:], 3)):
        wire = torch.full((off + view.numel() + 16,), 0xA5, dtype=torch.uint8)
        N.host_execute([N.save_desc(view, off, wire_dtype=qdtype, qparams=(scale, zp))], wire)
        assert bytes(wire[:off].numpy()) == b"\xa5" * off
        assert bytes(wire[off:].numpy()) == _per_tensor_expected(view, scale, zp, qdtype), (tuple(view.shape), off)


def _per_channel_file(x, qdtype, axis) -> bytes:
    scales, zps = per_channel_qparams(x, qdtype, axis)
    q = torch.quantize_per_channel(x.float(), scales.to(x.device), zps.to(x.device), axis, qdtype)
    return struct.pack("<q", axis) + q.int_repr().contiguous().cpu().numpy().tobytes() + scales.cpu().numpy().tobytes() + zps.cpu().numpy().tobytes()


@pytest.mark.parametrize("qdtype", [torch.qint8, torch.quint8], ids=_name)
@pytest.mark.parametrize("src", FLOATS, ids=_name)
def test_quantize_per_channel_at_ties(qdtype, src):
    t = tie_channels(37, 300, qdtype)
    for x, axis in ((t, 0), (t.t().contiguous(), 1), (t.t(), 1), (t.t().reshape(30, 10, 37), 2)):
        x = x.to(src)
        wire = torch.zeros(8 + x.numel() + 16 * x.shape[axis], dtype=torch.uint8)
        N.host_execute([N.save_desc(x, 8, wire_dtype=qdtype, axis=axis)], wire)
        assert bytes(wire.numpy()) == _per_channel_file(x, qdtype, axis), (tuple(x.shape), axis)


# ---- through the API --------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pg():
    if not dist.is_initialized():
        f = tempfile.NamedTemporaryFile(delete=False)
        dist.init_process_group("gloo", init_method=f"file://{f.name}", rank=0, world_size=1)
    yield
    if dist.is_initialized():
        dist.destroy_process_group()


def _sharded(t: torch.Tensor):
    from torch.distributed._shard.sharded_tensor import Shard, ShardedTensor, ShardMetadata

    dev = "cpu" if t.device.type == "cpu" else f"cuda:{t.device.index or 0}"
    md = ShardMetadata(shard_offsets=[0] * t.dim(), shard_sizes=list(t.shape), placement=f"rank:0/{dev}")
    return ShardedTensor._init_from_local_shards([Shard(tensor=t, metadata=md)], tuple(t.shape))


def slab_with_bool_restore(tmp_path, device, target, nan_bits):
    """{flag: bool[3], w: fp32 [8, 8], v: fp64 [8, 8]} in one slab, so w and v sit at offsets that are not multiples of
    their element size; restored into sharded targets of `target` with Tensor.copy_ semantics."""
    w = case_values(torch.float32, target, 64).reshape(8, 8).to(device)
    v = case_values(torch.float64, target, 64).reshape(8, 8).to(device)
    flag = torch.tensor([True, False, True], device=device)
    root = str(tmp_path / "s")
    snap = B.Snapshot.take(root, {"m": B.StateDict(flag=flag, w=_sharded(w.clone()), v=_sharded(v.clone()))})
    man = snap.get_manifest()
    pieces = [man[f"0/m/{k}"].shards[0].tensor for k in ("w", "v")]
    assert pieces[0].location == pieces[1].location == man["0/m/flag"].location
    assert any(p.byte_range[0] % 4 for p in pieces), [p.byte_range for p in pieces]
    tw, tv = torch.zeros(8, 8, dtype=target, device=device), torch.zeros(8, 8, dtype=target, device=device)
    snap.restore({"m": B.StateDict(flag=torch.zeros(3, dtype=torch.bool, device=device), w=_sharded(tw), v=_sharded(tv))})
    for got, src in ((tw, w), (tv, v)):
        err = same_values(got, torch.zeros_like(got).copy_(src), nan_bits)
        assert err is None, (src.dtype, err)


@pytest.mark.parametrize("target", FLOATS, ids=_name)
def test_slab_member_behind_a_bool_restores_into_another_dtype(target, tmp_path, pg):
    slab_with_bool_restore(tmp_path, "cpu", target, nan_bits=False)


def test_cast_on_save_fp64_to_fp16_rounds_through_fp32(tmp_path):
    x = case_values(torch.float64, torch.float16, 300)
    root = str(tmp_path / "s")
    snap = B.Snapshot.take(root, {"m": B.StateDict(x=x)}, _custom_tensor_prepare_func=B.cast_on_save(torch.float16))
    e = snap.get_manifest()["0/m/x"]
    raw = open(os.path.join(root, e.location), "rb").read()
    if e.byte_range is not None:
        raw = raw[e.byte_range[0] : e.byte_range[1]]
    err = same_values(torch.frombuffer(bytearray(raw), dtype=torch.float16), x.to(torch.float16), nan_bits=False)
    assert err is None, err
