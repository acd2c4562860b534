"""The device's converting and quantising kernels against torch on the same device, at the values and layouts where
conversions go wrong (tests/conversion_cases.py): the cast path of the LSU kernel (vector fast path, its ragged tail,
tile seams, the scalar strided path, unaligned wire sides), the per-tensor quantiser, the per-channel statistics,
parameter and quantising-pack kernels, and the dequantising scatter.  Bit-exact, NaN bits included."""
import pytest
import torch

from tests.conversion_cases import (FLOATS, PAIRS, LAYOUTS, SAVE_LAYOUTS, restore_case, same_values, save_case,
                                    tie_channels, tie_values)
from tests.test_conversions_cpu import QPARAMS, _per_channel_file, _per_tensor_expected, pg, slab_with_bool_restore  # noqa: F401
from torchsnapshot_b200 import _native as N
from torchsnapshot_b200.prepare import per_channel_qparams

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
_name = lambda dt: str(dt).replace("torch.", "")
_TILE = 128 << 10  # LSU tile: destination bytes


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
    """The member is planned as one LSU member of ceil(nbytes / tile) tiles (the cast path: nothing on the copy engine)."""
    info = N.plan_describe([desc])
    assert info["n_members_lsu"] == 1 and info["n_members_bulk"] == info["n_members_rows"] == info["n_members_host"] == 0, info
    assert info["n_tiles_lsu"] == -(-nbytes // _TILE), info


def _with_filler(off):
    """A 1-byte member in front of an odd wire offset, as a bool or odd-sized buffer puts it in a slab."""
    pre = torch.full((off,), 0xA5, dtype=torch.uint8, device=DEV)
    return [N.save_desc(pre, 0)] if off else [], [pre]


@pytest.mark.parametrize("layout", SAVE_LAYOUTS, ids=lambda l: l.name)
@pytest.mark.parametrize("src,dst", PAIRS, ids=[f"{_name(s)}-{_name(d)}" for s, d in PAIRS])
def test_cast_on_save(engine, src, dst, layout):
    c = save_case(layout, src, dst, DEV)
    n = c.expected.numel() * c.expected.element_size()
    desc = N.save_desc(c.view, c.offset, wire_dtype=dst)
    _on_lsu_cast_path(desc, n)
    if layout.name.startswith("dense"):
        assert n >= 3 * _TILE
    pre, keep = _with_filler(c.offset)
    got = _stage(engine, pre + [desc], c.offset + n, keep + [c.view])
    assert bool((got[: c.offset] == 0xA5).all())
    err = same_values(got[c.offset :].clone().view(dst), c.expected.cpu(), nan_bits=True)
    assert err is None, err


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: l.name)
@pytest.mark.parametrize("src,dst", PAIRS, ids=[f"{_name(s)}-{_name(d)}" for s, d in PAIRS])
def test_cast_on_restore(engine, src, dst, layout):
    c = restore_case(layout, src, dst, DEV)
    desc = N.load_desc(c.view, c.desc_offset, wire_dtype=src, wire_strides=c.wire_strides)
    _on_lsu_cast_path(desc, c.view.numel() * c.view.element_size())
    engine.consume(c.wire.cpu().numpy(), [desc])
    torch.cuda.synchronize()
    err = same_values(c.storage.cpu(), c.expected.cpu(), nan_bits=True)
    assert err is None, err


@pytest.mark.parametrize("src", FLOATS, ids=_name)
@pytest.mark.parametrize("qdtype,scale,zp", QPARAMS)
def test_quantize_per_tensor_at_ties(engine, qdtype, scale, zp, src):
    x = tie_values(scale, zp, qdtype).to(src).to(DEV)
    assert x.numel() % 16
    n = x.numel() // 3 * 3
    # dense, transposed, narrowed at an odd wire offset (the trailer is then written byte by byte)
    for view, off in ((x, 0), (x[:n].view(3, -1).t(), 0), (x[:n].view(3, -1)[:, 5:], 3)):
        pre, keep = _with_filler(off)
        got = _stage(engine, pre + [N.save_desc(view, off, wire_dtype=qdtype, qparams=(scale, zp))], off + view.numel() + 16, keep + [view])
        assert bytes(got[:off].numpy()) == b"\xa5" * off
        assert bytes(got[off:].numpy()) == _per_tensor_expected(view, scale, zp, qdtype), (tuple(view.shape), off)


def _channel_tensor(shape, axis, qdtype, dtype, dense=True):
    """A tensor of `shape` whose channels along `axis` are tie_channels."""
    C = shape[axis]
    rest = [s for i, s in enumerate(shape) if i != axis % len(shape)]
    t = tie_channels(C, max(1, torch.Size(rest).numel()), qdtype).reshape(C, *rest).movedim(0, axis).to(dtype).to(DEV)
    return t.contiguous() if dense else t


# (shape, axis, source dtype, qdtype, dense source).  2048 channels is the most the statistics kernel keeps in shared
# memory; 2049 takes its global-atomic path.  Periodic: channels x inner divides 4096, the statistics kernel's
# per-thread accumulation.
QCHANNEL = {
    "one_channel": ((1, 5000), 0, torch.float32, torch.qint8, True),
    "c2048": ((2048, 40), 0, torch.float32, torch.qint8, True),
    "c2048_quint8": ((2048, 40), 0, torch.float32, torch.quint8, True),
    "c2049": ((2049, 33), 0, torch.float32, torch.quint8, True),
    "c2049_bf16": ((2049, 33), 0, torch.bfloat16, torch.qint8, True),
    "periodic_axis1": ((96, 256), 1, torch.float32, torch.quint8, True),
    "periodic_axis-1_fp16": ((6, 20, 128), -1, torch.float16, torch.qint8, True),
    "nonperiodic_axis1": ((64, 300), 1, torch.float32, torch.qint8, True),
    "nonperiodic_axis-1_fp64": ((8, 12, 100), -1, torch.float64, torch.quint8, True),
    "axis1_bf16": ((300, 77), 1, torch.bfloat16, torch.quint8, True),
    "axis0_strided_fp64": ((64, 500), 0, torch.float64, torch.qint8, False),
    "axis1_strided_fp16": ((130, 90), 1, torch.float16, torch.quint8, False),
}


@pytest.mark.parametrize("case", list(QCHANNEL))
def test_quantize_per_channel_at_ties(engine, case):
    shape, axis, dtype, qdtype, dense = QCHANNEL[case]
    x = _channel_tensor(shape, axis, qdtype, dtype, dense)
    ax = axis % x.dim()
    k0 = engine.stats()["kernels_launched"]
    got = _stage(engine, [N.save_desc(x, 8, wire_dtype=qdtype, axis=ax)], 8 + x.numel() + 16 * shape[ax], [x])
    assert engine.stats()["kernels_launched"] - k0 >= 3  # statistics, parameters, quantising pack
    want = _per_channel_file(x, qdtype, ax)
    if bytes(got.numpy()) != want:
        w = torch.frombuffer(bytearray(want), dtype=torch.uint8)
        bad = (got != w).nonzero().reshape(-1)[:8].tolist()
        pytest.fail(f"{int((got != w).sum())} bytes differ, first at {bad}: got {got[bad].tolist()} want {w[bad].tolist()}")


def _dequant_source(shape, axis, qdtype):
    x = _channel_tensor(shape, axis, qdtype, torch.float32)
    scales, zps = per_channel_qparams(x, qdtype, axis)
    q = torch.quantize_per_channel(x, scales.to(DEV), zps.to(DEV), axis, qdtype)
    return q, _per_channel_file(x, qdtype, axis)


# numel = 1, 2, 3 (mod 4): the dense path's ragged tail; (129, 1031) spans several tiles
DEQUANT_SHAPES = [((37, 41), 0, torch.qint8), ((33, 50), 1, torch.quint8), ((3, 1001), 1, torch.qint8), ((129, 1031), 0, torch.quint8)]


@pytest.mark.parametrize("target", FLOATS, ids=_name)
@pytest.mark.parametrize("shape,axis,qdtype", DEQUANT_SHAPES, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else str(v))
def test_dequantize_per_channel(engine, target, shape, axis, qdtype):
    q, wire = _dequant_source(shape, axis, qdtype)
    dst = torch.full(shape, 7.0, dtype=target, device=DEV)
    k0 = engine.stats()["kernels_launched"]
    engine.consume(wire, [N.per_channel(N.load_desc(dst, 8, wire_dtype=qdtype), list(shape), axis, 8)])
    torch.cuda.synchronize()
    assert engine.stats()["kernels_launched"] > k0
    err = same_values(dst.cpu(), torch.empty_like(dst).copy_(q.dequantize()).cpu(), nan_bits=True)
    assert err is None, err


@pytest.mark.parametrize("target", FLOATS, ids=_name)
def test_dequantize_per_channel_into_reshard_subbox(engine, target):
    piece, box = (40, 67), (slice(7, 31), slice(5, 50))
    q, wire = _dequant_source(piece, 1, torch.quint8)
    local = torch.full((30, 60), 7.0, dtype=target, device=DEV)
    view = local[3:27, 10:55]
    first = 7 * 67 + 5
    desc = N.per_channel(N.load_desc(view, 8 + first, wire_dtype=torch.quint8, wire_strides=[67, 1]), list(piece), 1, 8)
    engine.consume(wire, [desc])
    torch.cuda.synchronize()
    want = torch.full_like(local, 7.0)
    want[3:27, 10:55].copy_(q.dequantize()[box])
    err = same_values(local.cpu(), want.cpu(), nan_bits=True)
    assert err is None, err


@pytest.mark.parametrize("target", FLOATS, ids=_name)
def test_slab_member_behind_a_bool_restores_into_another_dtype(target, tmp_path, pg):  # noqa: F811
    slab_with_bool_restore(tmp_path, DEV, target, nan_bits=True)
