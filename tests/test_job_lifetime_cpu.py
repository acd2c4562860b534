"""Lifetime of engine jobs on a host engine: every job finishes exactly once, whichever order the caller waits and
destroys in, on success and on failure, and leaves no file descriptor open behind it."""
import os

import pytest
import torch

from tests.util import det_tensor, wire_bytes
from torchsnapshot_b200 import _native as N

SLOT = 1 << 20


@pytest.fixture
def eng():
    e = N.Engine(device=-1, pinned_slot_bytes=SLOT, pinned_slots=2)
    yield e
    e.close()


def open_fds() -> int:
    return len(os.listdir("/proc/self/fd"))


def host_files(k: int):
    """(name, [(wire offset, source view)], nbytes) of one job: empty files, slabs and dense files above a slot."""
    out = []
    for i in range(k):
        out.append((f"e{i}", [], 0))
        a = det_tensor((300, 7), torch.float32, 10 + i)
        b = det_tensor((1001,), torch.uint8, 20 + i)
        c = det_tensor((40, 30), torch.int16, 30 + i).t()
        members, off = [], 0
        for v in (a, b, c):
            members.append((off, v))
            off += v.numel() * v.element_size()
        out.append((f"s{i}", members, off))
        d = det_tensor((5 * SLOT // 2 + 8 * i,), torch.uint8, 40 + i)  # several parts on load
        out.append((f"d{i}", [(0, d)], d.numel()))
    return out


def save_job(eng, root, files):
    job = eng.save_job()
    for name, members, nbytes in files:
        fi = job.add_file(os.path.join(root, name), nbytes)
        for off, v in members:
            job.add_member(fi, N.save_desc(v, off), v)
    return job


def check_saved(root, files):
    for name, members, nbytes in files:
        data = open(os.path.join(root, name), "rb").read()
        assert len(data) == nbytes, name
        for off, v in members:
            want = wire_bytes(v)
            assert data[off : off + len(want)] == want, name


@pytest.mark.parametrize("order", ["wait_then_destroy", "destroy_only", "wait_twice_then_destroy"])
def test_save_and_load_round_trip_close_every_file(eng, tmp_path, order):
    files = host_files(6)
    base = open_fds()
    job = save_job(eng, str(tmp_path), files)
    job.submit()
    if order != "destroy_only":
        job.wait()
    if order == "wait_twice_then_destroy":
        job.wait()
    job.destroy()
    assert open_fds() == base
    check_saved(str(tmp_path), files)

    outs = []
    job = eng.load_job()
    for name, members, nbytes in files:
        fi = job.add_file(str(tmp_path / name), nbytes)
        for off, v in members:
            dst = torch.zeros(v.shape, dtype=v.dtype)
            if not v.is_contiguous():
                dst = torch.zeros(v.shape[::-1], dtype=v.dtype).t()
            outs.append((v, dst))
            job.add_member(fi, N.load_desc(dst, off), dst)
    job.submit()
    if order != "destroy_only":
        job.wait()
        assert job.done()
    job.destroy()
    assert open_fds() == base
    for v, dst in outs:
        assert wire_bytes(dst) == wire_bytes(v)


def test_save_with_an_uncreatable_path_fails_and_finishes_the_others(tmp_path):
    # a failed job stops writing: one worker takes the files in order, so every file before the bad one is complete
    eng = N.Engine(device=-1, io_threads=1, pinned_slot_bytes=SLOT, pinned_slots=2)
    try:
        (tmp_path / "blocker").write_bytes(b"not a directory")
        bad = str(tmp_path / "blocker" / "x")
        files = host_files(3)
        base = open_fds()
        job = save_job(eng, str(tmp_path), files)
        t = det_tensor((3 * SLOT,), torch.uint8, 99)
        fi = job.add_file(bad, t.numel())
        job.add_member(fi, N.save_desc(t, 0), t)
        job.submit()
        with pytest.raises(N.NativeError, match=bad):
            job.wait()
        job.destroy()
        assert open_fds() == base
        check_saved(str(tmp_path), files)
    finally:
        eng.close()


@pytest.mark.parametrize("dense", [True, False], ids=["dense", "slab"])
def test_load_past_the_end_of_a_file_fails_and_closes_it(eng, tmp_path, dense):
    src = det_tensor((3 * SLOT,), torch.uint8, 5)
    path = tmp_path / "short"
    path.write_bytes(wire_bytes(src))
    base = open_fds()
    job = eng.load_job()
    fi = job.add_file(str(path), src.numel(), offset=100)  # the range runs 100 bytes past the end
    dst = torch.zeros_like(src)
    if dense:
        job.add_member(fi, N.load_desc(dst, 0), dst)
    else:
        job.add_member(fi, N.load_desc(dst[:SLOT], 0), dst)
        job.add_member(fi, N.load_desc(dst[SLOT:], SLOT), dst)
    job.submit()
    with pytest.raises(N.NativeError, match="pread"):
        job.wait()
    job.destroy()
    assert open_fds() == base


def test_destroy_right_after_submit_waits_for_every_part(eng, tmp_path):
    files = host_files(40)
    base = open_fds()
    job = save_job(eng, str(tmp_path), files)
    job.submit()
    job.destroy()  # returns once the job has finished: every file is complete and closed
    assert open_fds() == base
    check_saved(str(tmp_path), files)
