"""Execution of write/read plans.

The reference drives every request through an asyncio state machine (stage -> write, budget gated,
4 staging threads, <=16 I/Os; T:scheduler.py:222-339, 386-446).  Here requests are split in two:

  * raw tensor traffic against a local filesystem — the hot path — becomes ONE engine job per device:
    all members are described to the C ABI, packed by a single kernel launch pair, drained through
    the pinned ring and written by native workers (save), or read, uploaded and scattered (restore);
  * everything else (pickled leaves, third-party storage plugins) keeps the reference's pipeline
    semantics: staging is admitted while the host-memory budget allows, at most
    ``get_max_per_rank_io_concurrency()`` storage operations are in flight.

``execute_write_reqs`` returns when every source tensor has been read (the async_take gate,
T:scheduler.py:299); ``PendingIOWork.complete`` drains the I/O."""
from __future__ import annotations

import asyncio
import logging
import os
import socket
import time
from collections import defaultdict
from concurrent.futures import ThreadPoolExecutor
from typing import Dict, List, Optional, Set, Tuple

import psutil
import torch

from . import _native
from .io_types import ReadIO, ReadReq, StoragePlugin, WriteIO, WriteReq
from .knobs import get_max_per_rank_io_concurrency, get_memory_budget_override
from .native_plan import HostCloneBudget, describe_consumer, describe_stager, native_root as _native_root
from .pg_wrapper import PGWrapper

logger = logging.getLogger(__name__)

_MAX_PER_RANK_MEMORY_BUDGET_BYTES = 32 * 1024**3
_AVAILABLE_MEMORY_MULTIPLIER = 0.6
_MAX_PER_RANK_CPU_CONCURRENCY = 4


_LOCAL_WORLD: Dict[int, Tuple[object, int]] = {}  # id(pg) -> (pg kept alive so the id stays unique, ranks on this host)


def get_local_world_size(pg: PGWrapper) -> int:
    """Ranks of `pg` on this host (T:scheduler.py:35-44).  Host placement does not change during a job, so the
    hostname all-gather is paid once per process group instead of once per snapshot."""
    key = id(pg.pg)
    ent = _LOCAL_WORLD.get(key)
    if ent is None or ent[0] is not pg.pg:
        me = socket.gethostname()
        names = [None] * pg.get_world_size()
        pg.all_gather_object(names, me)
        ent = (pg.pg, sum(1 for n in names if n == me))
        _LOCAL_WORLD[key] = ent
    return ent[1]


def get_process_memory_budget_bytes(pg: PGWrapper) -> int:
    override = get_memory_budget_override()
    if override is not None:
        return override
    avail = int(psutil.virtual_memory().available * _AVAILABLE_MEMORY_MULTIPLIER)
    return min(avail // get_local_world_size(pg), _MAX_PER_RANK_MEMORY_BUDGET_BYTES)


# ---- routing -------------------------------------------------------------------------------------
def _engine_key(tensors: List[torch.Tensor]) -> int:
    for t in tensors:
        if t.is_cuda:
            return t.device.index if t.device.index is not None else torch.cuda.current_device()
    return -1


def _one_device(tensors: List[torch.Tensor]) -> bool:
    """A request goes to ONE engine (one GPU).  A slab whose members live on several GPUs of this process (the batcher
    keys GPU slabs by is_cuda only, like T:batcher.py:300-303) is left to its own stage_buffer, which stages member by
    member through each tensor's engine."""
    devs = {t.device.index if t.device.index is not None else torch.cuda.current_device() for t in tensors if t.is_cuda}
    return len(devs) <= 1


class _NativeJobs:
    """One engine job per device that appears in the plan."""

    def __init__(self, save: bool) -> None:
        self.save = save
        self.jobs: Dict[int, "_native.Job"] = {}
        self.payload_bytes = 0

    def job_for(self, key: int) -> "_native.Job":
        j = self.jobs.get(key)
        if j is None:
            eng = _native.get_engine(key)
            j = eng.save_job() if self.save else eng.load_job()
            self.jobs[key] = j
        return j

    def submit(self, memory_budget_bytes: int = 0) -> None:
        for key, j in self.jobs.items():
            stream = torch.cuda.current_stream(key).cuda_stream if key >= 0 else None
            # the per-rank host-memory budget (T:scheduler.py:47-67) bounds the pinned slots a job holds at once
            j.set_host_budget(memory_budget_bytes // max(1, len(self.jobs)))
            j.submit(stream)

    def wait_device(self) -> None:
        # failures (e.g. an unwritable path) are reported by wait(), i.e. by PendingSnapshot.wait() for
        # async_take — the same place the reference surfaces storage errors (tests/test_async_take.py:58-66)
        for j in self.jobs.values():
            try:
                j.wait_device()
            except _native.NativeError:
                pass

    def wait(self) -> None:
        err = None
        for j in self.jobs.values():
            try:
                j.wait()
            except Exception as e:  # keep draining the others before raising
                err = err or e
        if err is not None:
            raise err

    def stats(self) -> List[dict]:
        return [j.stats() for j in self.jobs.values()]

    def traces(self) -> List[List[dict]]:
        """Per-chunk timelines (only when the engine was created with ENGINE_TRACE)."""
        return [j.trace() for j in self.jobs.values() if j.engine.flags & _native.ENGINE_TRACE]

    def destroy(self) -> None:
        for j in self.jobs.values():
            j.destroy()
        self.jobs.clear()


LAST_STATS: Dict[str, object] = {}  # filled by the last executed plan; read by bench.py


class PendingIOWork:
    def __init__(self, native: Optional[_NativeJobs], io_tasks: Set["asyncio.Task"], begin_ts: float, rank: int, nbytes: int,
                 deferred_error: Optional[BaseException] = None) -> None:
        self.native = native
        self.io_tasks = io_tasks
        self.begin_ts = begin_ts
        self.rank = rank
        self.nbytes = nbytes
        self.deferred_error = deferred_error  # a storage error of the blocking part: reported where async errors are

    async def complete(self) -> None:
        loop = asyncio.get_running_loop()
        try:
            if self.io_tasks:
                await asyncio.gather(*self.io_tasks)
            if self.native is not None:
                await loop.run_in_executor(None, self.native.wait)
                LAST_STATS["save"] = self.native.stats()
                LAST_STATS["save_trace"] = self.native.traces()
        finally:
            if self.native is not None:
                self.native.destroy()
        if self.deferred_error is not None:
            raise self.deferred_error
        dt = max(time.monotonic() - self.begin_ts, 1e-9)
        logger.info(f"Rank {self.rank} completed writing in {dt:.2f} seconds (throughput {self.nbytes / 2**20 / dt:.2f}MB/s)")

    def sync_complete(self, event_loop: asyncio.AbstractEventLoop) -> None:
        event_loop.run_until_complete(self.complete())


async def execute_write_reqs(
    write_reqs: List[WriteReq], storage: StoragePlugin, memory_budget_bytes: int, rank: int
) -> PendingIOWork:
    begin = time.monotonic()
    phases: Dict[str, float] = {}
    t_mark = [time.perf_counter()]

    def lap(name: str) -> None:
        now = time.perf_counter()
        phases[name] = (now - t_mark[0]) * 1e3
        t_mark[0] = now

    loop = asyncio.get_running_loop()
    root = _native_root(storage, "write")
    native: Optional[_NativeJobs] = None
    blocking: Optional[_NativeJobs] = None  # async_take: CPU tensors beyond the clone budget, written before returning
    clones = HostCloneBudget(memory_budget_bytes)
    generic: List[WriteReq] = []
    total = 0
    for wr in write_reqs:
        described = describe_stager(wr.buffer_stager, clones) if root is not None else None
        in_place = clones.take_blocking()
        if described is not None and not _one_device(described[1]):
            described = None
        if described is not None:
            descs, keep, nbytes = described
            if in_place:
                if blocking is None:
                    blocking = _NativeJobs(save=True)
                group = blocking
            else:
                if native is None:
                    native = _NativeJobs(save=True)
                group = native
            job = group.job_for(_engine_key(keep))
            fi = job.add_file(os.path.join(root, wr.path), nbytes)
            for d in descs:
                job.add_member(fi, d)
            job._keepalive.extend(keep)
            total += nbytes
        else:
            generic.append(wr)
    lap("describe+build_job")
    if native is not None:
        native.submit(memory_budget_bytes)
    lap("submit")
    deferred_error: Optional[BaseException] = None
    if blocking is not None:
        # read from the caller's memory: these files are complete before control returns to the caller
        try:
            blocking.submit(memory_budget_bytes)
            await loop.run_in_executor(None, blocking.wait)
        except Exception as e:  # surfaced by PendingSnapshot.wait(), like every other storage error of async_take
            deferred_error = e
        finally:
            blocking.destroy()
        lap("blocking_host_writes")
    LAST_STATS["host_clone_bytes"] = clones.cloned_bytes
    LAST_STATS["host_blocking_bytes"] = clones.blocking_bytes

    # generic pipeline: budget-gated staging, bounded concurrent writes
    io_tasks: Set[asyncio.Task] = set()
    if generic:
        executor = ThreadPoolExecutor(max_workers=_MAX_PER_RANK_CPU_CONCURRENCY)
        budget = memory_budget_bytes
        io_slots = asyncio.Semaphore(get_max_per_rank_io_concurrency())
        credit = asyncio.Condition()
        inflight = 0

        async def write_out(wr: WriteReq, buf) -> int:
            nonlocal budget, inflight
            n = len(buf)
            try:
                async with io_slots:
                    await storage.write(WriteIO(path=wr.path, buf=buf))
            finally:
                del buf
                async with credit:
                    budget += n
                    inflight -= 1
                    credit.notify_all()
            return n

        pending = sorted(generic, key=lambda w: w.buffer_stager.get_staging_cost_bytes())
        staging: Set[asyncio.Task] = set()

        async def stage_one(wr: WriteReq, cost: int) -> None:
            nonlocal budget
            buf = await wr.buffer_stager.stage_buffer(executor)
            async with credit:
                budget += cost - len(buf)  # the estimate is replaced by the real footprint
            io_tasks.add(asyncio.ensure_future(write_out(wr, buf)))

        for wr in pending:
            cost = wr.buffer_stager.get_staging_cost_bytes()
            async with credit:
                # an over-budget request is only admitted when nothing else is in flight (T:scheduler.py:266-272)
                await credit.wait_for(lambda: cost < budget or inflight == 0)
                budget -= cost
                inflight += 1
            staging.add(asyncio.ensure_future(stage_one(wr, cost)))
            total += cost
        if staging:
            await asyncio.gather(*staging)
        executor.shutdown(wait=False)

    lap("generic_staging")
    if native is not None:
        await loop.run_in_executor(None, native.wait_device)
    lap("wait_device")
    LAST_STATS["write_phases_ms"] = phases
    logger.info(f"Rank {rank} completed staging in {time.monotonic() - begin:.2f} seconds")
    return PendingIOWork(native, io_tasks, begin, rank, total, deferred_error)


def sync_execute_write_reqs(
    write_reqs: List[WriteReq], storage: StoragePlugin, memory_budget_bytes: int, rank: int, event_loop: asyncio.AbstractEventLoop
) -> PendingIOWork:
    return event_loop.run_until_complete(execute_write_reqs(write_reqs, storage, memory_budget_bytes, rank))


# ---- read-once restore of replicated state over NVLink --------------------------------------------------------------
_READ_ONCE_MIN_BYTES = 4 << 20
_READ_ONCE_BUF_BYTES = 256 << 20


def _plan_shared_reads(pg: PGWrapper, mine: Dict[Tuple[str, int, int], int]) -> Dict[Tuple[str, int, int], int]:
    """{(path, lo, hi): reader rank} for the byte ranges EVERY rank of `pg` is about to read into GPU tensors — DDP /
    replicated state, which the reference reads from storage once per rank (T:manifest_ops.py:69-85).  One object
    all-gather; the greedy least-loaded assignment is evaluated identically on every rank."""
    world = pg.get_world_size()
    gathered: List[Optional[List[Tuple[str, int, int]]]] = [None] * world
    pg.all_gather_object(gathered, sorted(mine))
    common = set(gathered[0] or [])
    for g in gathered[1:]:
        common &= set(g or [])
    if sum(hi - lo for _, lo, hi in common) < _READ_ONCE_MIN_BYTES:
        return {}
    load = [0] * world
    owner: Dict[Tuple[str, int, int], int] = {}
    for key in sorted(common, key=lambda k: (-(k[2] - k[1]), k)):
        r = min(range(world), key=lambda i: (load[i], i))
        owner[key] = r
        load[r] += key[2] - key[1]
    return owner


def _read_once_eligible(pg: Optional[PGWrapper]) -> bool:
    import torch.distributed as dist

    if pg is None or pg.pg is None or pg.get_world_size() < 2 or os.environ.get("TSNAP_B200_READ_ONCE", "1") == "0":
        return False
    try:
        if dist.get_backend(pg.pg) != "nccl":
            return False
    except Exception:
        return False
    # peers exchange the file images GPU to GPU: only worth it (and only NVLink) inside one host
    return get_local_world_size(pg) == pg.get_world_size()


def _shift_descs(descs, delta: int):
    return [_native.rebase(d, delta) for d in descs]


def _execute_shared_reads(pg: PGWrapper, root: str, shared: List[Tuple[Tuple[str, int, int], list, list]], owner: Dict[Tuple[str, int, int], int]) -> int:
    """Every shared byte range is read from storage by its owner only (file -> pinned ring -> H2D straight into a
    staging tensor), broadcast GPU-to-GPU, and scattered into the live tensors by every rank's scatter kernels.
    Returns the bytes this rank read from storage."""
    import torch.distributed as dist

    rank, world = pg.get_rank(), pg.get_world_size()
    dev = torch.cuda.current_device()
    eng = _native.get_engine(dev)
    by_key = {k: (descs, keep) for k, descs, keep in shared}
    # identical on every rank: per owner, ranges packed into buffers of <= _READ_ONCE_BUF_BYTES (256 B-aligned members)
    plan: List[Tuple[int, int, List[Tuple[Tuple[str, int, int], int]]]] = []  # (owner, nbytes, [(key, offset)])
    for r in range(world):
        cur: List[Tuple[Tuple[str, int, int], int]] = []
        off = 0
        for key in sorted(k for k, o in owner.items() if o == r):
            n = key[2] - key[1]
            if cur and off + n > _READ_ONCE_BUF_BYTES:
                plan.append((r, off, cur))
                cur, off = [], 0
            cur.append((key, off))
            off += (n + 255) // 256 * 256
        if cur:
            plan.append((r, off, cur))
    # my own buffers are filled first, all in one engine job (reads of all ranks proceed concurrently)
    mine = {i: torch.empty(nb, dtype=torch.uint8, device=f"cuda:{dev}") for i, (r, nb, _) in enumerate(plan) if r == rank}
    job = None
    read_bytes = 0
    if mine:
        job = eng.load_job()
        for i, buf in mine.items():
            for key, off in plan[i][2]:
                path, lo, hi = key
                fi = job.add_file(os.path.join(root, path), hi - lo, offset=lo)
                job.add_member(fi, _native.load_desc(buf[off : off + (hi - lo)], 0), buf)
                read_bytes += hi - lo
        job.submit(torch.cuda.current_stream(dev).cuda_stream)
    err: Optional[BaseException] = None
    try:
        waited = False
        for i, (r, nb, members) in enumerate(plan):
            if r == rank:
                if not waited:
                    try:
                        job.wait()
                    except Exception as e:  # keep taking part in the exchange: the peers are already waiting in it
                        err = e
                    waited = True
                buf = mine[i]
            else:
                buf = torch.empty(nb, dtype=torch.uint8, device=f"cuda:{dev}")
            dist.broadcast(buf, src=dist.get_global_rank(pg.pg, r), group=pg.pg)
            descs = []
            for key, off in members:
                descs += _shift_descs(by_key[key][0], off)
            # ordered after the broadcast on the current stream; synchronous, so `buf` may be dropped afterwards
            if err is None:
                try:
                    eng.scatter_device(buf, descs, stream=torch.cuda.current_stream(dev).cuda_stream)
                except Exception as e:
                    err = e
            mine.pop(i, None)
        # a read error on one rank must fail the restore on every rank (each rank would have hit it reading for itself)
        flag = torch.tensor([1 if err is not None else 0], dtype=torch.int32, device=f"cuda:{dev}")
        dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=pg.pg)
        if err is not None:
            raise err
        if int(flag.item()):
            raise RuntimeError("read-once restore: a peer rank failed to read or scatter a replicated byte range (see its log)")
    finally:
        if job is not None:
            job.destroy()
    return read_bytes


async def execute_read_reqs(
    read_reqs: List[ReadReq], storage: StoragePlugin, memory_budget_bytes: int, rank: int, shared_pg: Optional[PGWrapper] = None
) -> None:
    """`shared_pg`: set by Snapshot.restore (a collective call on that group): byte ranges that every rank reads into
    GPU tensors are then read from storage once and exchanged over NVLink (see _execute_shared_reads)."""
    begin = time.monotonic()
    loop = asyncio.get_running_loop()
    root = _native_root(storage, "read")
    native: Optional[_NativeJobs] = None
    generic: List[ReadReq] = []
    total = 0
    # every rank of the group takes part in the negotiation, also one with nothing to share (storage the engine does
    # not drive, CPU-only targets): the all-gather is a collective
    read_once = _read_once_eligible(shared_pg)
    candidates: List[Tuple[Tuple[str, int, int], list, list]] = []
    described_reqs = []
    for rr in read_reqs:
        described = describe_consumer(rr.buffer_consumer, root) if root is not None else None
        if described is not None and not _one_device(described[1]):
            described = None
        if described is not None:
            descs, keep, wire_nbytes = described
            if rr.byte_range is not None:
                lo, hi = rr.byte_range
            else:
                lo, hi = 0, wire_nbytes
            if not descs:
                continue
            described_reqs.append((rr, descs, keep, lo, hi))
        else:
            generic.append(rr)
    owner: Dict[Tuple[str, int, int], int] = {}
    if read_once:
        mine = {}
        for rr, descs, keep, lo, hi in described_reqs:
            if hi > lo and all(d.dst_space == _native.SPACE_DEVICE for d in descs) and (rr.path, lo, hi) not in mine:
                mine[(rr.path, lo, hi)] = hi - lo
        owner = _plan_shared_reads(shared_pg, mine)
    seen_shared = set()
    for rr, descs, keep, lo, hi in described_reqs:
        key = (rr.path, lo, hi)
        if key in owner and all(d.dst_space == _native.SPACE_DEVICE for d in descs):
            if key in seen_shared:  # two consumers of the same range: both scatter from the one image
                for c in candidates:
                    if c[0] == key:
                        c[1].extend(descs)
                        c[2].extend(keep)
            else:
                seen_shared.add(key)
                candidates.append((key, list(descs), list(keep)))
            total += hi - lo
            continue
        if native is None:
            native = _NativeJobs(save=False)
        job = native.job_for(_engine_key(keep))
        fi = job.add_file(os.path.join(root, rr.path), hi - lo, offset=lo)
        for d in descs:
            job.add_member(fi, d)
        job._keepalive.extend(keep)
        total += hi - lo
    try:
        if native is not None:
            native.submit(memory_budget_bytes)
        if candidates:
            LAST_STATS["read_once"] = {"ranges": len(candidates), "bytes": sum(k[2] - k[1] for k, _, _ in candidates),
                                       "bytes_read_by_this_rank": _execute_shared_reads(shared_pg, root, candidates, owner)}
        else:
            LAST_STATS["read_once"] = None
        if generic:
            executor = ThreadPoolExecutor(max_workers=_MAX_PER_RANK_CPU_CONCURRENCY)
            io_slots = asyncio.Semaphore(get_max_per_rank_io_concurrency())
            budget = memory_budget_bytes
            credit = asyncio.Condition()
            inflight = 0

            async def one(rr: ReadReq, cost: int) -> None:
                nonlocal budget, inflight
                try:
                    async with io_slots:
                        rio = ReadIO(path=rr.path, byte_range=rr.byte_range)
                        await storage.read(rio)
                    buf = rio.buf.getbuffer()
                    await rr.buffer_consumer.consume_buffer(buf, executor)
                finally:
                    async with credit:
                        budget += cost
                        inflight -= 1
                        credit.notify_all()

            tasks = []
            for rr in generic:
                cost = rr.buffer_consumer.get_consuming_cost_bytes()
                async with credit:
                    await credit.wait_for(lambda: cost < budget or inflight == 0)
                    budget -= cost
                    inflight += 1
                tasks.append(asyncio.ensure_future(one(rr, cost)))
                total += cost
            await asyncio.gather(*tasks)
            executor.shutdown(wait=False)
        if native is not None:
            await loop.run_in_executor(None, native.wait)
            LAST_STATS["load"] = native.stats()
            LAST_STATS["load_trace"] = native.traces()
    finally:
        if native is not None:
            native.destroy()
    dt = max(time.monotonic() - begin, 1e-9)
    logger.info(f"Rank {rank} finished loading. Throughput: {total / 2**20 / dt:.2f}MB/s")


def sync_execute_read_reqs(
    read_reqs: List[ReadReq], storage: StoragePlugin, memory_budget_bytes: int, rank: int, event_loop: asyncio.AbstractEventLoop,
    shared_pg: Optional[PGWrapper] = None,
) -> None:
    event_loop.run_until_complete(execute_read_reqs(read_reqs, storage, memory_budget_bytes, rank, shared_pg))
