"""ctypes binding of ``libtsnap_b200.so`` (the C ABI declared in ``include/tsnap_b200.h``).

The library is the product: there is no Python/PyTorch fallback for the device path.  If the shared
object is missing this module raises at import time, and if the engine cannot get a usable sm_90
device it raises at engine creation — loudly, never silently degrading to torch ops.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from typing import Iterable, List, Optional, Sequence, Tuple

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libtsnap_b200.so")

MAX_DIMS = 8

# enum tsnap_dtype
U8, I8, I16, I32, I64, F16, BF16, F32, F64, BOOL, QINT8, QUINT8, F8E4M3FN, F8E5M2 = range(14)
# enum tsnap_space
SPACE_DEVICE, SPACE_HOST, SPACE_WIRE = 0, 1, 2

ENGINE_FSYNC = 2
ENGINE_ODIRECT = 4
ENGINE_TRACE = 8
ENGINE_NO_ARENA = 16

PROBE_D2H, PROBE_H2D, PROBE_WRITE, PROBE_READ = 0, 1, 2, 3
TRACE_KINDS = ("plan", "kernel", "d2h", "pwrite", "slot_wait", "pread", "h2d", "open")

# the ten buffer-protocol dtypes of the reference (T:serialization.py:162-173) and the two float8 formats
TORCH_TO_TSNAP = {
    torch.uint8: U8,
    torch.int8: I8,
    torch.int16: I16,
    torch.int32: I32,
    torch.int64: I64,
    torch.float16: F16,
    torch.bfloat16: BF16,
    torch.float32: F32,
    torch.float64: F64,
    torch.bool: BOOL,
    torch.float8_e4m3fn: F8E4M3FN,
    torch.float8_e5m2: F8E5M2,
}


class NativeError(RuntimeError):
    def __init__(self, code: int, msg: str) -> None:
        super().__init__(f"tsnap_b200 error {code}: {msg}")
        self.code = code


class CopyDesc(C.Structure):
    _fields_ = [
        ("src_addr", C.c_uint64),
        ("dst_addr", C.c_uint64),
        ("sizes", C.c_int64 * MAX_DIMS),
        ("src_strides", C.c_int64 * MAX_DIMS),
        ("dst_strides", C.c_int64 * MAX_DIMS),
        ("ndim", C.c_int32),
        ("src_dtype", C.c_int32),
        ("dst_dtype", C.c_int32),
        ("src_space", C.c_int32),
        ("dst_space", C.c_int32),
        ("reserved", C.c_int32),
        ("q_scale", C.c_double),
        ("q_zero_point", C.c_int64),
    ]


# tsnap_copy_desc.reserved: quantisation scheme
QSCHEME_PER_TENSOR, QSCHEME_PER_CHANNEL = 0, 1


class QChannel(C.Structure):
    """tsnap_qchannel: where the per-channel format's parts of one piece sit in the wire image."""

    _fields_ = [
        ("channels", C.c_int64),
        ("inner", C.c_int64),
        ("body_addr", C.c_uint64),
        ("params_addr", C.c_uint64),
        ("axis", C.c_int64),
    ]


def per_channel(d: CopyDesc, shape: Sequence[int], axis: int, body: int) -> CopyDesc:
    """Marks ``d`` as a per-channel copy of the piece of ``shape`` whose int body starts at wire offset ``body`` (the
    axis header sits 8 bytes before it, the parameters right behind it).  The record is kept on the descriptor: the
    library reads it while the descriptor is handed over (add_member, stage, consume, ...)."""
    numel = 1
    for n in shape:
        numel *= int(n)
    inner = 1
    for n in shape[axis + 1 :]:
        inner *= int(n)
    rec = QChannel(channels=int(shape[axis]), inner=inner, body_addr=body, params_addr=body + numel, axis=axis)
    d.reserved = QSCHEME_PER_CHANNEL
    d.q_zero_point = C.addressof(rec)
    d._qchannel = rec
    return d


def rebase(d: CopyDesc, delta: int) -> CopyDesc:
    """A copy of load descriptor ``d`` whose wire image starts ``delta`` bytes later (a per-channel record moves too)."""
    c = CopyDesc.from_buffer_copy(d)
    c.src_addr = d.src_addr + delta
    if d.reserved == QSCHEME_PER_CHANNEL:
        r = QChannel.from_buffer_copy(d._qchannel)
        r.body_addr += delta
        r.params_addr += delta
        c.q_zero_point = C.addressof(r)
        c._qchannel = r
    return c


class EngineConfig(C.Structure):
    _fields_ = [
        ("device", C.c_int32),
        ("io_threads", C.c_int32),
        ("pinned_slot_bytes", C.c_uint64),
        ("pinned_slots", C.c_int32),
        ("flags", C.c_int32),
        ("hbm_staging_bytes", C.c_uint64),
    ]


class EngineStats(C.Structure):
    _fields_ = [
        ("pinned_bytes", C.c_uint64),
        ("hbm_arena_bytes", C.c_uint64),
        ("kernels_launched", C.c_uint64),
        ("bytes_d2h", C.c_uint64),
        ("bytes_h2d", C.c_uint64),
        ("bytes_written", C.c_uint64),
        ("bytes_read", C.c_uint64),
        ("sm_count", C.c_int32),
        ("device", C.c_int32),
    ]


class JobStats(C.Structure):
    _fields_ = [
        ("payload_bytes", C.c_uint64),
        ("n_files", C.c_uint64),
        ("n_members", C.c_uint64),
        ("n_tiles_bulk", C.c_uint64),
        ("n_tiles_lsu", C.c_uint64),
        ("n_kernel_launches", C.c_uint64),
        ("plan_ms", C.c_double),
        ("kernel_ms", C.c_double),
        ("kernel_bulk_ms", C.c_double),
        ("kernel_lsu_ms", C.c_double),
        ("device_done_ms", C.c_double),
        ("total_ms", C.c_double),
        ("table_h2d_bytes", C.c_uint64),
        ("slot_wait_ms", C.c_double),
        ("io_busy_ms", C.c_double),
        ("io_queue_ms", C.c_double),
        ("copy_ms", C.c_double),
        ("arena_bytes", C.c_uint64),
        ("n_waves", C.c_uint64),
        ("direct_bytes", C.c_uint64),
        ("n_memcpy", C.c_uint64),
        ("bytes_bulk", C.c_uint64),
        ("bytes_lsu", C.c_uint64),
        ("bytes_rows", C.c_uint64),
        ("n_tiles_rows", C.c_uint64),
        ("kernel_rows_ms", C.c_double),
        ("max_slots_in_flight", C.c_uint64),
        ("link_starved_ms", C.c_double),
    ]

    def as_dict(self) -> dict:
        return {k: getattr(self, k) for k, _ in self._fields_}


class ArenaHint(C.Structure):
    _fields_ = [
        ("total_bytes", C.c_uint64),
        ("largest_file_bytes", C.c_uint64),
        ("strided_total_bytes", C.c_uint64),
        ("strided_largest_bytes", C.c_uint64),
    ]


class TraceRec(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("lane", C.c_int32),
        ("file", C.c_int32),
        ("reserved", C.c_int32),
        ("t0_ms", C.c_double),
        ("t1_ms", C.c_double),
        ("bytes", C.c_uint64),
    ]


class PlanInfo(C.Structure):
    _fields_ = [
        ("n_members_bulk", C.c_uint64),
        ("n_members_lsu", C.c_uint64),
        ("n_members_host", C.c_uint64),
        ("n_tiles_bulk", C.c_uint64),
        ("n_tiles_lsu", C.c_uint64),
        ("bytes_bulk", C.c_uint64),
        ("bytes_lsu", C.c_uint64),
        ("bytes_host", C.c_uint64),
        ("n_members_rows", C.c_uint64),
        ("n_tiles_rows", C.c_uint64),
        ("bytes_rows", C.c_uint64),
    ]


# every symbol include/tsnap_b200.h declares; tests assert the .so exports all of them
EXPORTED_SYMBOLS = [
    "tsnap_abi_version",
    "tsnap_last_error",
    "tsnap_dtype_size",
    "tsnap_engine_create",
    "tsnap_engine_destroy",
    "tsnap_engine_trim",
    "tsnap_engine_get_stats",
    "tsnap_save_job_create",
    "tsnap_save_job_add_file",
    "tsnap_save_job_add_member",
    "tsnap_save_job_submit",
    "tsnap_job_wait_device",
    "tsnap_job_wait",
    "tsnap_job_done",
    "tsnap_job_destroy",
    "tsnap_job_get_stats",
    "tsnap_load_job_create",
    "tsnap_load_job_add_file",
    "tsnap_load_job_add_member",
    "tsnap_load_job_submit",
    "tsnap_stage_submit",
    "tsnap_buffer_wait_device",
    "tsnap_buffer_wait",
    "tsnap_buffer_release",
    "tsnap_buffer_get_stats",
    "tsnap_consume",
    "tsnap_plan_describe",
    "tsnap_host_execute",
    "tsnap_job_arena_hint",
    "tsnap_job_set_arena",
    "tsnap_job_get_trace",
    "tsnap_engine_probe",
    "tsnap_scatter_device",
    "tsnap_job_set_host_budget",
]


def _load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C torchsnapshot_b200/csrc`. torchsnapshot_b200 has no fallback data path."
        )
    lib = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    lib.tsnap_abi_version.restype = C.c_int
    lib.tsnap_last_error.restype = C.c_char_p
    lib.tsnap_dtype_size.restype = C.c_size_t
    lib.tsnap_dtype_size.argtypes = [C.c_int]
    lib.tsnap_engine_create.argtypes = [C.POINTER(EngineConfig), C.POINTER(vp)]
    lib.tsnap_engine_destroy.argtypes = [vp]
    lib.tsnap_engine_trim.argtypes = [vp]
    lib.tsnap_engine_get_stats.argtypes = [vp, C.POINTER(EngineStats)]
    lib.tsnap_save_job_create.argtypes = [vp, C.POINTER(vp)]
    lib.tsnap_load_job_create.argtypes = [vp, C.POINTER(vp)]
    lib.tsnap_save_job_add_file.argtypes = [vp, C.c_char_p, C.c_uint64, C.POINTER(C.c_int32)]
    lib.tsnap_load_job_add_file.argtypes = [vp, C.c_char_p, C.c_uint64, C.c_uint64, C.POINTER(C.c_int32)]
    lib.tsnap_save_job_add_member.argtypes = [vp, C.c_int32, C.POINTER(CopyDesc)]
    lib.tsnap_load_job_add_member.argtypes = [vp, C.c_int32, C.POINTER(CopyDesc)]
    lib.tsnap_save_job_submit.argtypes = [vp, vp]
    lib.tsnap_load_job_submit.argtypes = [vp, vp]
    lib.tsnap_job_wait_device.argtypes = [vp]
    lib.tsnap_job_wait.argtypes = [vp]
    lib.tsnap_job_done.argtypes = [vp]
    lib.tsnap_job_destroy.argtypes = [vp]
    lib.tsnap_job_get_stats.argtypes = [vp, C.POINTER(JobStats)]
    lib.tsnap_stage_submit.argtypes = [vp, C.POINTER(CopyDesc), C.c_int32, C.c_uint64, vp, C.POINTER(vp)]
    lib.tsnap_buffer_wait_device.argtypes = [vp]
    lib.tsnap_buffer_wait.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_uint64)]
    lib.tsnap_buffer_release.argtypes = [vp]
    lib.tsnap_buffer_get_stats.argtypes = [vp, C.POINTER(JobStats)]
    lib.tsnap_consume.argtypes = [vp, vp, C.c_uint64, C.POINTER(CopyDesc), C.c_int32, vp]
    lib.tsnap_plan_describe.argtypes = [C.POINTER(CopyDesc), C.c_int32, C.c_uint64, C.POINTER(PlanInfo)]
    lib.tsnap_host_execute.argtypes = [C.POINTER(CopyDesc), C.c_int32, vp, C.c_uint64, C.c_int32]
    lib.tsnap_job_arena_hint.argtypes = [vp, C.POINTER(ArenaHint)]
    lib.tsnap_job_set_arena.argtypes = [vp, vp, C.c_uint64]
    lib.tsnap_job_get_trace.argtypes = [vp, C.POINTER(TraceRec), C.c_uint64, C.POINTER(C.c_uint64)]
    lib.tsnap_engine_probe.argtypes = [vp, C.c_int, C.c_char_p, C.c_uint64, C.POINTER(C.c_double)]
    lib.tsnap_scatter_device.argtypes = [vp, vp, C.c_uint64, C.POINTER(CopyDesc), C.c_int32, vp]
    lib.tsnap_job_set_host_budget.argtypes = [vp, C.c_uint64]
    for name in EXPORTED_SYMBOLS:
        fn = getattr(lib, name)
        if name not in ("tsnap_last_error", "tsnap_dtype_size"):
            fn.restype = C.c_int
    if lib.tsnap_abi_version() != 2:
        raise ImportError("libtsnap_b200.so ABI version mismatch; rebuild it")
    return lib


lib = _load()


def check(rc: int) -> None:
    if rc != 0:
        raise NativeError(rc, (lib.tsnap_last_error() or b"").decode("utf-8", "replace"))


def tsnap_dtype(dtype: torch.dtype) -> int:
    try:
        return TORCH_TO_TSNAP[dtype]
    except KeyError:
        raise NativeError(-6, f"dtype {dtype} has no raw wire format (not a buffer-protocol dtype)") from None


def _space_of(t: torch.Tensor) -> int:
    if t.is_cuda:
        return SPACE_DEVICE
    if t.device.type == "cpu":
        return SPACE_HOST
    raise NativeError(-6, f"tensors on {t.device} are not supported")


def _merge_dims(sizes: Sequence[int], *stride_sets: Sequence[int]):
    """Folds size-1 dims away and merges neighbours that are dense across their boundary on EVERY side (what the native
    planner does as well); used to fit views of more than MAX_DIMS dims into a descriptor."""
    out_sizes: List[int] = []
    out_strides: List[List[int]] = [[] for _ in stride_sets]
    for i, n in enumerate(sizes):
        if n == 1:
            continue
        st = [ss[i] for ss in stride_sets]
        if out_sizes and all(o[-1] == s_i * n for o, s_i in zip(out_strides, st)):
            out_sizes[-1] *= n
            for o, s_i in zip(out_strides, st):
                o[-1] = s_i
        else:
            out_sizes.append(n)
            for o, s_i in zip(out_strides, st):
                o.append(s_i)
    return out_sizes, out_strides


def _c_strides(shape: Sequence[int]) -> List[int]:
    acc, out = 1, [0] * len(shape)
    for i in range(len(shape) - 1, -1, -1):
        out[i] = acc
        acc *= shape[i]
    return out


def needs_contiguous_copy(t: torch.Tensor) -> bool:
    """True for the (exotic) views that still need more than MAX_DIMS strided dims after folding: the caller makes
    them contiguous first — what the reference does for every non-contiguous source (T:batcher.py:156) — and keeps
    that copy alive for the duration of the job."""
    if t.dim() <= MAX_DIMS:
        return False
    sizes, _ = _merge_dims(list(t.shape), list(t.stride()), _c_strides(list(t.shape)))
    return len(sizes) > MAX_DIMS


_QUANT = {torch.qint8: QINT8, torch.quint8: QUINT8}


def save_desc(
    t: torch.Tensor, wire_offset: int, wire_dtype: Optional[torch.dtype] = None, qparams: Optional[Tuple[float, int]] = None,
    axis: Optional[int] = None,
) -> CopyDesc:
    """tensor view -> wire image at ``wire_offset`` (C-contiguous layout of ``t.shape``).  ``wire_dtype`` fuses a float
    cast; with ``wire_dtype`` torch.qint8/quint8 and ``qparams=(scale, zero_point)`` the pack kernel quantises and
    appends the 16-byte per-tensor trailer (T:serialization.py:278-310).  With ``axis`` instead of ``qparams`` the engine
    quantises per channel along ``axis`` (non-negative): ``wire_offset`` is then where the int body starts, behind the
    8-byte axis header, and the channel parameters follow the body.  ``axis`` with a float8 ``wire_dtype`` is the
    per-channel scaled float8 format, laid out the same way with one f32 scale per channel."""
    d = CopyDesc()
    sizes, strides = list(t.shape), list(t.stride())
    if len(sizes) > MAX_DIMS:
        # the wire side is C-contiguous: it merges wherever the source does
        sizes, (strides, _) = _merge_dims(sizes, strides, _c_strides(sizes))
        if len(sizes) > MAX_DIMS:
            raise NativeError(-6, f"view does not reduce to {MAX_DIMS} strided dims (see needs_contiguous_copy)")
    d.ndim = len(sizes)
    for i, (n, s) in enumerate(zip(sizes, strides)):
        d.sizes[i] = n
        d.src_strides[i] = s
    d.src_addr = t.data_ptr()
    d.dst_addr = wire_offset
    d.src_dtype = tsnap_dtype(t.dtype)
    if wire_dtype in _QUANT:
        d.dst_dtype = _QUANT[wire_dtype]
        if axis is not None:
            per_channel(d, list(t.shape), axis, wire_offset)
        elif qparams is not None:
            d.q_scale, d.q_zero_point = float(qparams[0]), int(qparams[1])
        else:
            raise NativeError(-1, "quantising descriptors need qparams=(scale, zero_point) or an axis")
    else:
        d.dst_dtype = tsnap_dtype(wire_dtype or t.dtype)
        if axis is not None:  # a float8 wire dtype: per-channel scaled float8
            per_channel(d, list(t.shape), axis, wire_offset)
    d.src_space = _space_of(t)
    d.dst_space = SPACE_WIRE
    return d


def load_desc(
    t: torch.Tensor,
    wire_offset: int,
    wire_dtype: Optional[torch.dtype] = None,
    wire_strides: Optional[Sequence[int]] = None,
) -> CopyDesc:
    """wire bytes at ``wire_offset`` -> tensor view.  ``wire_strides`` (elements) describe the saved
    piece when ``t`` receives a sub-box of it (reshard-on-load); default: the piece has ``t``'s shape."""
    d = CopyDesc()
    sizes, dstrides = list(t.shape), list(t.stride())
    wstrides = list(wire_strides) if wire_strides is not None else _c_strides(sizes)
    if len(sizes) > MAX_DIMS:
        sizes, (wstrides, dstrides) = _merge_dims(sizes, wstrides, dstrides)
        if len(sizes) > MAX_DIMS:
            raise NativeError(-6, f"destination view does not reduce to {MAX_DIMS} strided dims")
    d.ndim = len(sizes)
    for i, (n, ws, ds) in enumerate(zip(sizes, wstrides, dstrides)):
        d.sizes[i] = n
        d.src_strides[i] = ws
        d.dst_strides[i] = ds
    d.src_addr = wire_offset
    d.dst_addr = t.data_ptr()
    d.src_dtype = _QUANT[wire_dtype] if wire_dtype in _QUANT else tsnap_dtype(wire_dtype or t.dtype)
    d.dst_dtype = tsnap_dtype(t.dtype)
    d.src_space = SPACE_WIRE
    d.dst_space = _space_of(t)
    return d


def _desc_array(descs: Sequence[CopyDesc]):
    arr = (CopyDesc * max(1, len(descs)))()
    for i, d in enumerate(descs):
        arr[i] = d
    return arr


class Job:
    """A save or load job.  Keeps the tensors it references alive until it is destroyed."""

    def __init__(self, engine: "Engine", handle: C.c_void_p, save: bool) -> None:
        self.engine = engine
        self._h = handle
        self._save = save
        self._keepalive: List[object] = []
        self._arena: Optional[torch.Tensor] = None
        self._destroyed = False

    def add_file(self, path: str, nbytes: int, offset: int = 0) -> int:
        idx = C.c_int32(-1)
        if self._save:
            check(lib.tsnap_save_job_add_file(self._h, os.fsencode(path), nbytes, C.byref(idx)))
        else:
            check(lib.tsnap_load_job_add_file(self._h, os.fsencode(path), offset, nbytes, C.byref(idx)))
        return idx.value

    def add_member(self, file_index: int, desc: CopyDesc, keepalive: object = None) -> None:
        fn = lib.tsnap_save_job_add_member if self._save else lib.tsnap_load_job_add_member
        check(fn(self._h, file_index, C.byref(desc)))
        if keepalive is not None:
            self._keepalive.append(keepalive)

    def arena_hint(self) -> dict:
        h = ArenaHint()
        check(lib.tsnap_job_arena_hint(self._h, C.byref(h)))
        return {k: getattr(h, k) for k, _ in h._fields_}

    def set_arena(self, tensor: Optional[torch.Tensor]) -> None:
        """Lend the job its HBM staging (a uint8 CUDA tensor, kept alive until the job is destroyed); None selects the
        arena-less mode: dense members are drained straight from the live tensors."""
        if tensor is None:
            check(lib.tsnap_job_set_arena(self._h, None, 0))
            return
        check(lib.tsnap_job_set_arena(self._h, C.c_void_p(tensor.data_ptr()), tensor.numel() * tensor.element_size()))
        self._arena = tensor

    def set_host_budget(self, nbytes: int) -> None:
        """Host-memory budget of this job (T:scheduler.py:47-67): bounds the pinned ring slots it holds at once."""
        check(lib.tsnap_job_set_host_budget(self._h, max(0, int(nbytes))))

    def _provision_arena(self) -> None:
        """HBM staging comes from PyTorch's caching allocator, so it is visible to — and reusable by — the training job
        the moment the snapshot has drained (the reference's GPU slab is a torch.cuda.ByteTensor too, T:batcher.py:147).
        Policy: the whole payload when that leaves max(1/8 of HBM, 4 GiB) free; else as much as that reserve allows if it
        still holds two of the largest files (multi-wave staging); else no arena — dense members then go over the link
        straight from the live tensors and only strided/converting members are staged (the reference falls back to a
        CPU slab when its GPU slab OOMs, T:batcher.py:148-152)."""
        dev = self.engine.device
        if dev < 0 or self.engine.owns_arena:
            return
        hint = self.arena_hint()
        total, largest = hint["total_bytes"], hint["largest_file_bytes"]
        if total == 0:
            return
        no_dense_staging = bool(self.engine.flags & ENGINE_NO_ARENA)
        if no_dense_staging and hint["strided_total_bytes"] == 0:
            self.set_arena(None)
            return
        cap = self.engine.hbm_staging_bytes
        with torch.cuda.device(dev):
            free_b, total_b = torch.cuda.mem_get_info(dev)
            cached = torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
            reserve = max(total_b // 8, 4 << 30)
            allowed = max(0, free_b + cached - reserve)
            if cap:
                allowed = min(allowed, cap)
            cands = []
            if no_dense_staging:
                pass  # only what the strided / converting members need (below)
            elif total <= allowed:
                cands.append(total)
            elif allowed >= 2 * largest:
                cands.append(allowed)
            nd_total, nd_largest = hint["strided_total_bytes"], hint["strided_largest_bytes"]
            if nd_total:
                if nd_total <= allowed and nd_total not in cands:
                    cands.append(nd_total)
                cands.append(min(nd_total, 2 * nd_largest))
            for i, want in enumerate(cands):
                want = (want + (2 << 20) - 1) // (2 << 20) * (2 << 20)
                for attempt in range(2):
                    try:
                        self.set_arena(torch.empty(want, dtype=torch.uint8, device=f"cuda:{dev}"))
                        return
                    except torch.OutOfMemoryError:
                        if attempt == 0:
                            torch.cuda.empty_cache()  # give cached-but-fragmented blocks back and retry once
            self.set_arena(None)

    def submit(self, stream: Optional[int] = None) -> None:
        self._provision_arena()
        fn = lib.tsnap_save_job_submit if self._save else lib.tsnap_load_job_submit
        check(fn(self._h, C.c_void_p(stream or 0)))

    def trace(self) -> List[dict]:
        n = C.c_uint64(0)
        check(lib.tsnap_job_get_trace(self._h, None, 0, C.byref(n)))
        if n.value == 0:
            return []
        arr = (TraceRec * n.value)()
        check(lib.tsnap_job_get_trace(self._h, arr, n.value, C.byref(n)))
        return [dict(kind=TRACE_KINDS[r.kind], lane=r.lane, file=r.file, t0_ms=r.t0_ms, t1_ms=r.t1_ms, bytes=r.bytes) for r in arr]

    def wait_device(self) -> None:
        check(lib.tsnap_job_wait_device(self._h))

    def wait(self) -> None:
        check(lib.tsnap_job_wait(self._h))

    def done(self) -> bool:
        return bool(lib.tsnap_job_done(self._h))

    def stats(self) -> dict:
        st = JobStats()
        check(lib.tsnap_job_get_stats(self._h, C.byref(st)))
        return st.as_dict()

    def destroy(self) -> None:
        if not self._destroyed:
            self._destroyed = True
            lib.tsnap_job_destroy(self._h)  # waits for the job: nothing reads the arena any more
            self._keepalive.clear()
            self._arena = None

    def __del__(self) -> None:  # pragma: no cover - best effort
        try:
            self.destroy()
        except Exception:
            pass


class StagedBuffer:
    """Pinned host buffer produced by the stager seam; exposes the buffer protocol via memoryview."""

    def __init__(self, engine: "Engine", handle: C.c_void_p, nbytes: int, keepalive: List[object]) -> None:
        self.engine = engine
        self._h = handle
        self.nbytes = nbytes
        self._keepalive = keepalive
        self._released = False

    def wait_device(self) -> None:
        check(lib.tsnap_buffer_wait_device(self._h))

    def wait(self) -> memoryview:
        ptr = C.c_void_p()
        n = C.c_uint64()
        check(lib.tsnap_buffer_wait(self._h, C.byref(ptr), C.byref(n)))
        if n.value == 0:
            return memoryview(b"")
        arr = (C.c_char * n.value).from_address(ptr.value)
        # the memoryview keeps `arr` alive, `arr._owner` keeps this object (and the pinned block) alive
        arr._owner = self
        return memoryview(arr).cast("B")

    def stats(self) -> dict:
        st = JobStats()
        check(lib.tsnap_buffer_get_stats(self._h, C.byref(st)))
        return st.as_dict()

    def release(self) -> None:
        if not self._released:
            self._released = True
            lib.tsnap_buffer_release(self._h)
            self._keepalive = []

    def __del__(self) -> None:  # pragma: no cover - best effort
        try:
            self.release()
        except Exception:
            pass


class Engine:
    def __init__(
        self,
        device: int = -1,
        io_threads: int = 0,
        pinned_slot_bytes: int = 0,
        pinned_slots: int = 0,
        flags: int = 0,
        hbm_staging_bytes: int = 0,
    ) -> None:
        cfg = EngineConfig(device, io_threads, pinned_slot_bytes, pinned_slots, flags, hbm_staging_bytes)
        h = C.c_void_p()
        check(lib.tsnap_engine_create(C.byref(cfg), C.byref(h)))
        self._h = h
        self.device = device
        self.flags = flags
        self.hbm_staging_bytes = hbm_staging_bytes
        self.io_threads = io_threads or 16
        self.pinned_slots = pinned_slots or 32
        self.pinned_slot_bytes = pinned_slot_bytes or (32 << 20)
        # TSNAP_B200_ENGINE_ARENA=1: staging is the engine's own cudaMalloc'ed arena (what a C caller gets) instead
        # of memory lent from PyTorch's allocator
        self.owns_arena = os.environ.get("TSNAP_B200_ENGINE_ARENA", "0") == "1"
        self._closed = False

    def save_job(self) -> Job:
        h = C.c_void_p()
        check(lib.tsnap_save_job_create(self._h, C.byref(h)))
        return Job(self, h, True)

    def load_job(self) -> Job:
        h = C.c_void_p()
        check(lib.tsnap_load_job_create(self._h, C.byref(h)))
        return Job(self, h, False)

    def stage(self, descs: Sequence[CopyDesc], nbytes: int, stream: Optional[int] = None, keepalive=None) -> StagedBuffer:
        arr = _desc_array(descs)
        h = C.c_void_p()
        check(lib.tsnap_stage_submit(self._h, arr, len(descs), nbytes, C.c_void_p(stream or 0), C.byref(h)))
        return StagedBuffer(self, h, nbytes, list(keepalive or []))

    def probe(self, kind: int, nbytes: int, directory: Optional[str] = None) -> float:
        """GB/s of the engine's own link (PROBE_D2H/H2D) or sink/source (PROBE_WRITE/READ under `directory`)."""
        out = C.c_double(0.0)
        check(lib.tsnap_engine_probe(self._h, kind, os.fsencode(directory) if directory else None, nbytes, C.byref(out)))
        return out.value

    def consume(self, buf, descs: Sequence[CopyDesc], stream: Optional[int] = None) -> None:
        mv = memoryview(buf).cast("B")
        n = mv.nbytes
        if n == 0:
            return
        if mv.readonly:
            # ctypes cannot borrow a read-only buffer without a copy unless we go through its address
            import numpy as np

            addr = np.frombuffer(mv, dtype=np.uint8).__array_interface__["data"][0]
        else:
            addr = C.addressof(C.c_char.from_buffer(mv))
        arr = _desc_array(descs)
        if stream is None and self.device >= 0:
            stream = torch.cuda.current_stream(self.device).cuda_stream
        check(lib.tsnap_consume(self._h, C.c_void_p(addr), n, arr, len(descs), C.c_void_p(stream or 0)))

    def scatter_device(self, wire: torch.Tensor, descs: Sequence[CopyDesc], stream: Optional[int] = None) -> None:
        """Scatter a wire image that already sits in this GPU's memory (`wire`: uint8 CUDA tensor) into destination views."""
        if not descs:
            return
        if stream is None:
            stream = torch.cuda.current_stream(self.device).cuda_stream
        arr = _desc_array(descs)
        check(lib.tsnap_scatter_device(self._h, C.c_void_p(wire.data_ptr()), wire.numel() * wire.element_size(), arr, len(descs), C.c_void_p(stream or 0)))

    def stats(self) -> dict:
        st = EngineStats()
        check(lib.tsnap_engine_get_stats(self._h, C.byref(st)))
        return {k: getattr(st, k) for k, _ in st._fields_}

    def trim(self) -> None:
        check(lib.tsnap_engine_trim(self._h))

    def close(self) -> None:
        if not self._closed:
            self._closed = True
            lib.tsnap_engine_destroy(self._h)

    def __del__(self) -> None:  # pragma: no cover - best effort
        try:
            self.close()
        except Exception:
            pass


def host_execute(descs: Sequence[CopyDesc], wire: "torch.Tensor | bytearray | memoryview", threads: int = 1) -> None:
    """HOST<->WIRE copies against a host wire buffer (shares the planner with the device path)."""
    if isinstance(wire, torch.Tensor):
        addr, n = wire.data_ptr(), wire.numel() * wire.element_size()
    else:
        mv = memoryview(wire).cast("B")
        n = mv.nbytes
        addr = C.addressof(C.c_char.from_buffer(mv)) if n else 0
    arr = _desc_array(descs)
    check(lib.tsnap_host_execute(arr, len(descs), C.c_void_p(addr), n, threads))


def plan_describe(descs: Sequence[CopyDesc], wire_base_align: int = 0) -> dict:
    info = PlanInfo()
    arr = _desc_array(descs)
    check(lib.tsnap_plan_describe(arr, len(descs), wire_base_align, C.byref(info)))
    return {k: getattr(info, k) for k, _ in info._fields_}


# ---- process-wide engines -----------------------------------------------------------------------
_engines: dict = {}
_engines_lock = threading.Lock()


def get_engine(device: int = -1, **kwargs) -> Engine:
    """One engine per device per process (the pinned ring costs ~0.5 s/GiB to create, so it is kept)."""
    with _engines_lock:
        key = device
        eng = _engines.get(key)
        if eng is None:
            env = os.environ
            # the kernel's buffered-write path stops scaling at some tens of concurrent writers per host, so ranks
            # sharing a host draw every chunk I/O from one host-wide pool of 16 tokens (engine.cu: HostTokens); each rank
            # keeps 16 workers so that a rank draining alone can use the whole pool.  TSNAP_B200_HOST_IO_TOKENS=0 restores
            # the static split.  Placement: pinned ring interleaved over the NUMA nodes + workers bound to a node and
            # serving that node's slots = every page-cache copy is node-local.  The engine reads both from the environment.
            env.setdefault("TSNAP_B200_RING_NUMA", "interleave")
            env.setdefault("TSNAP_B200_IO_PIN", "node")
            local_world = max(1, int(env.get("LOCAL_WORLD_SIZE", "1")))
            tokens = int(env.get("TSNAP_B200_HOST_IO_TOKENS", "16" if local_world > 1 else "0"))
            default_io = 16 if (tokens > 0 or local_world == 1) else max(2, 16 // local_world)
            opts = dict(
                io_threads=int(env.get("TSNAP_B200_IO_THREADS", str(default_io))),
                pinned_slot_bytes=int(env.get("TSNAP_B200_PINNED_SLOT_BYTES", "0")),
                pinned_slots=int(env.get("TSNAP_B200_PINNED_SLOTS", "64" if local_world == 1 else "32")),
                flags=int(env.get("TSNAP_B200_ENGINE_FLAGS", "0")),
                hbm_staging_bytes=int(env.get("TSNAP_B200_HBM_STAGING_BYTES", "0")),
            )
            opts.update(kwargs)
            eng = Engine(device=device, **opts)
            _engines[key] = eng
        return eng


def reset_engines() -> None:
    with _engines_lock:
        for eng in _engines.values():
            eng.close()
        _engines.clear()
