"""The stager seam on the host engine: a stage is a save job whose one file is the pinned buffer.  Whatever the layout,
the staged image is byte for byte what host_execute writes for the same descriptors."""
import pytest
import torch

from tests.util import det_tensor
from torchsnapshot_b200 import _native as N


@pytest.fixture(scope="module")
def engine():
    eng = N.Engine(device=-1, io_threads=2)
    yield eng
    eng.close()


def _slab():
    """Members back to back, so that every byte of the image is written: dense, strided, casting, per-tensor and
    per-channel quantised (the last with its 8-byte header in front of the body)."""
    g = torch.Generator().manual_seed(3)
    dense = det_tensor((37, 11), torch.float32, 1)
    strided = det_tensor((40, 24), torch.int16, 2).t()[3:20]
    cast = torch.randn(9, 13, generator=g)
    qt = torch.randn(17, 5, generator=g)
    qc = torch.randn(6, 10, generator=g)
    descs, off = [], 0
    descs.append(N.save_desc(dense, off))
    off += dense.numel() * 4
    descs.append(N.save_desc(strided, off))
    off += strided.numel() * 2
    descs.append(N.save_desc(cast, off, wire_dtype=torch.bfloat16))
    off += cast.numel() * 2
    descs.append(N.save_desc(qt, off, wire_dtype=torch.qint8, qparams=(0.05, 3)))
    off += qt.numel() + 16
    descs.append(N.save_desc(qc, off + 8, wire_dtype=torch.quint8, axis=1))
    off += 8 + qc.numel() + 16 * qc.shape[1]
    return descs, off, [dense, strided, cast, qt, qc]


def _direct():
    """One dense member that covers the buffer: copied with a single memcpy."""
    t = det_tensor((64, 33), torch.int32, 5)
    return [N.save_desc(t, 0)], t.numel() * 4, [t]


def _empty():
    t = torch.empty(0, 3)
    return [N.save_desc(t, 0)], 0, [t]


def _expected(descs, nbytes) -> bytes:
    wire = bytearray(nbytes)
    N.host_execute(descs, wire)
    return bytes(wire)


@pytest.mark.parametrize("layout", [_slab, _direct, _empty], ids=["slab", "direct", "empty"])
def test_stage_matches_host_execute(engine, layout):
    descs, nbytes, keep = layout()
    before = engine.stats()
    sb = engine.stage(descs, nbytes, keepalive=keep)
    got = bytes(sb.wait())
    sb.release()
    assert len(got) == nbytes
    assert got == _expected(descs, nbytes)
    after = engine.stats()
    assert after["bytes_written"] == before["bytes_written"]  # the sink is memory, not a file


def test_release_right_after_submit_and_after_wait(engine):
    descs, nbytes, keep = _slab()
    expected = _expected(descs, nbytes)
    sb = engine.stage(descs, nbytes, keepalive=keep)
    sb.release()  # waits for the job before the buffer goes back to the pin cache
    sb = engine.stage(descs, nbytes, keepalive=keep)
    assert bytes(sb.wait()) == expected
    sb.release()
