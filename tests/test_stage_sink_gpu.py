"""A stage that mixes HOST and DEVICE members: the host members are copied into the pinned buffer, and only the device
members' wire extents come back from the GPU, each whole (per-tensor trailer, per-channel header and parameters)."""
import pytest
import torch

from tests.util import det_tensor
from torchsnapshot_b200 import _native as N

pytestmark = pytest.mark.gpu


def test_mixed_stage_copies_back_whole_device_extents(tmp_path):
    # a 4-slot, 1 MiB ring: nothing of a stage may depend on the ring
    eng = N.Engine(device=0, io_threads=2, pinned_slot_bytes=1 << 20, pinned_slots=4)
    try:
        g = torch.Generator().manual_seed(0)
        dense = det_tensor((300, 7), torch.float32, 1).cuda()
        strided = det_tensor((64, 48), torch.bfloat16, 2).cuda().t()[5:40]
        qt = torch.randn(33, 19, generator=g).cuda()
        qc = torch.randn(12, 25, generator=g).cuda()
        h_dense = det_tensor((50, 3), torch.int64, 3)
        h_strided = det_tensor((20, 30), torch.float16, 4)[::2, 1:]
        # host and device members interleaved, back to back: every byte of the image belongs to one member
        dev, host, off = [], [], 0
        dev.append(N.save_desc(dense, off))
        off += dense.numel() * 4
        host.append(N.save_desc(h_dense, off))
        off += h_dense.numel() * 8
        dev.append(N.save_desc(strided, off))
        off += strided.numel() * 2
        dev.append(N.save_desc(qt, off, wire_dtype=torch.qint8, qparams=(0.02, -3)))
        off += qt.numel() + 16
        host.append(N.save_desc(h_strided, off))
        off += h_strided.numel() * 2
        dev.append(N.save_desc(qc, off + 8, wire_dtype=torch.quint8, axis=1))
        off += 8 + qc.numel() + 16 * qc.shape[1]
        nbytes = off
        extents = nbytes - h_dense.numel() * 8 - h_strided.numel() * 2
        keep = [dense, strided, qt, qc, h_dense, h_strided]
        stream = torch.cuda.current_stream().cuda_stream

        # expected: the device members staged alone (a device-only stage, copied back whole), then the host members
        # written into that image; the device quantisers are not reproduced on the host
        before = eng.stats()
        alone = eng.stage(dev, nbytes, stream=stream, keepalive=keep)
        expected = bytearray(alone.wait())
        mid = eng.stats()
        N.host_execute(host, expected)

        mixed = eng.stage(dev[:1] + host[:1] + dev[1:3] + host[1:] + dev[3:], nbytes, stream=stream, keepalive=keep)
        got = bytes(mixed.wait())
        after = eng.stats()
        alone.release()  # held until now: the mixed stage must not reuse its buffer
        mixed.release()
        assert len(got) == nbytes
        assert got == bytes(expected)
        assert mid["bytes_d2h"] - before["bytes_d2h"] == nbytes
        assert after["bytes_d2h"] - mid["bytes_d2h"] == extents
        assert after["bytes_written"] == before["bytes_written"]

        # a stage never allocates the pinned ring: what the engine holds is the pin cache, two buffers
        cap = (max(nbytes, 4096) + 4095) // 4096 * 4096
        assert eng.stats()["pinned_bytes"] == 2 * cap

        # a real file still refuses the mix
        job = eng.save_job()
        fi = job.add_file(str(tmp_path / "mixed"), dense.numel() * 4 + h_dense.numel() * 8)
        job.add_member(fi, dev[0], dense)
        job.add_member(fi, host[0], h_dense)
        with pytest.raises(N.NativeError, match="mixes HOST and DEVICE"):
            job.submit(stream)
        job.destroy()
    finally:
        eng.close()
