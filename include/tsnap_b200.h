/*
 * tsnap_b200 — C ABI of the H100-native checkpoint data plane.
 *
 * This is the drop-in boundary for ONE path of pytorch/torchsnapshot: the device->host drain and
 * serialization of tensor state on save, and its mirror on restore.  Every entry point names the
 * reference interface it replaces (paths relative to the reference tree, "T:" = torchsnapshot/).
 * The reference is 100% Python, so a maintainer binds these with ctypes (see INTEGRATION.md); the
 * signatures use only plain pointers, sizes and integer handles — no torch types.
 *
 * Conventions
 *   - every function returns 0 on success and a negative TSNAP_E* code on failure;
 *     tsnap_last_error() returns a thread-local, human-readable message for the last failure.
 *   - all functions are callable from any thread and never take the Python GIL.
 *   - "wire buffer" = the byte image the reference would have produced for one storage object
 *     (one WriteReq / one file): raw C-contiguous native-endian element bytes of each member, back to
 *     back at their byte_range, no header, no padding (T:serialization.py:177-204, T:batcher.py:307).
 */
#ifndef TSNAP_B200_H_
#define TSNAP_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TSNAP_ABI_VERSION 2
#define TSNAP_MAX_DIMS 8

/* error codes */
#define TSNAP_OK 0
#define TSNAP_EINVAL (-1)   /* bad argument / malformed descriptor          */
#define TSNAP_ECUDA (-2)    /* a CUDA runtime call failed (no GPU, OOM, ..)   */
#define TSNAP_EIO (-3)      /* open/pwrite/pread failed                      */
#define TSNAP_ENOMEM (-4)   /* host allocation failed                        */
#define TSNAP_ESTATE (-5)   /* call made in the wrong job state              */
#define TSNAP_EUNSUP (-6)   /* dtype pair / layout not supported             */

/* element types: the ten buffer-protocol dtypes of T:serialization.py:162-173 (raw path), the two quantised wire
 * types and the two plain float8 formats.  The enum value only selects element size and, when src_dtype != dst_dtype,
 * the conversion. */
enum tsnap_dtype {
    TSNAP_U8 = 0,   /* torch.uint8 / torch.bool (1-byte payload, copied verbatim) */
    TSNAP_I8 = 1,
    TSNAP_I16 = 2,
    TSNAP_I32 = 3,
    TSNAP_I64 = 4,
    TSNAP_F16 = 5,
    TSNAP_BF16 = 6,
    TSNAP_F32 = 7,
    TSNAP_F64 = 8,
    TSNAP_BOOL = 9,
    /* 1-byte affine-quantized wire elements (torch.qint8 / torch.quint8 int_repr).  Only as the WIRE side of a save
     * from a floating-point source: q = clamp(round(x / q_scale) + q_zero_point) computed in the pack kernel, followed
     * by the 16-byte trailer of the reference's per-tensor format [q_scale: double][q_zero_point: int64]
     * (T:serialization.py:278-310) — the north star's "quantize in the pack kernel". */
    TSNAP_QINT8 = 10,
    TSNAP_QUINT8 = 11,
    /* torch.float8_e4m3fn / torch.float8_e5m2 (OCP FP8, 1-byte raw images).  Converted to and from F16 / BF16 / F32 /
     * F64 and each other with torch's rounding (through fp32, round to nearest even, subnormals kept; e4m3fn turns
     * values past 464 and +-inf into NaN with the sign kept, e5m2 overflows to +-inf).  Not a quantisation source. */
    TSNAP_F8E4M3FN = 12,
    TSNAP_F8E5M2 = 13,
    TSNAP_DTYPE_COUNT = 14
};

/* where a side of a copy lives */
enum tsnap_space {
    TSNAP_SPACE_DEVICE = 0, /* addr is a device pointer on the engine's GPU                 */
    TSNAP_SPACE_HOST = 1,   /* addr is a host pointer (CPU tensor)                          */
    TSNAP_SPACE_WIRE = 2    /* addr is a byte offset inside the wire buffer of the file    */
};

/*
 * One strided view <-> strided view copy of identical logical shape.  It is the common currency
 * of both directions:
 *   save    : src = live tensor view (DEVICE or HOST), dst = WIRE, dst_strides ignored (the wire
 *             image is the C-contiguous layout of `sizes` starting at dst_addr).
 *             Replaces the body of TensorBufferStager.stage_buffer (T:io_preparers/tensor.py:240-271)
 *             and the per-member .contiguous()+copy_ of GPUBatchedBufferStager.stage_buffer
 *             (T:batcher.py:144-159) / BatchedBufferStager.stage_buffer (T:batcher.py:66-93).
 *   restore : src = WIRE with src_strides describing the saved piece's C-contiguous layout
 *             (possibly a sub-box of it: reshard-on-load), dst = live tensor view.
 *             Replaces TensorBufferConsumer.consume_buffer (T:io_preparers/tensor.py:331-340) and
 *             the narrow()+tensor_copy loop of ShardedTensorBufferConsumer.consume_buffer
 *             (T:io_preparers/sharded_tensor.py:310-323, get_views :285-298).
 * Strides are in ELEMENTS of the respective dtype, as torch reports them; may be 0 or negative is
 * NOT supported (torch never produces negative strides).
 */
typedef struct tsnap_copy_desc {
    uint64_t src_addr;
    uint64_t dst_addr;
    int64_t sizes[TSNAP_MAX_DIMS];
    int64_t src_strides[TSNAP_MAX_DIMS];
    int64_t dst_strides[TSNAP_MAX_DIMS];
    int32_t ndim;
    int32_t src_dtype;  /* enum tsnap_dtype */
    int32_t dst_dtype;  /* enum tsnap_dtype; != src_dtype fuses a cast (north star "cast in the pack kernel") */
    int32_t src_space;  /* enum tsnap_space */
    int32_t dst_space;  /* enum tsnap_space */
    int32_t reserved;   /* quantisation scheme, TSNAP_QSCHEME_*; 0 for every other copy */
    double q_scale;        /* dst_dtype TSNAP_QINT8 / TSNAP_QUINT8 only */
    int64_t q_zero_point;  /* TSNAP_QSCHEME_PER_CHANNEL: address of a host tsnap_qchannel, read during the call */
} tsnap_copy_desc;

/* Quantisation schemes (tsnap_copy_desc.reserved).
 *   PER_TENSOR (0): q_scale / q_zero_point as above.
 *   PER_CHANNEL (1): the reference's per-channel format (T:serialization.py:366-477)
 *       [axis: int64][int_repr bytes, C order][scales: float64 x C][zero_points: int64 x C]
 *     save   : src = float view (DEVICE or HOST), dst_dtype QINT8 / QUINT8, dst WIRE at body_addr.  The engine computes
 *              each channel's (scale, zero_point) from the source — qint8: amax / 127 (1.0 when 0), zero point 0;
 *              quint8: (max(hi, 0) - min(lo, 0)) / 255 (1.0 when 0), zero point round_half_even(-min(lo, 0) / scale) —
 *              and writes the axis header, the int body and both parameter arrays.  A NaN or Inf fails the call / job.
 *     restore: src_dtype QINT8 / QUINT8 in WIRE (the piece or a sub-box of it), dst = float view of any float dtype:
 *              float((q - zero_point) * scale) converted to the destination dtype.
 *   PER_CHANNEL with a float8 wire dtype (F8E4M3FN / F8E5M2): this library's scaled float8 format
 *       [axis: int64][float8 bytes, C order][scales: float32 x C]
 *     save   : src = F16 / BF16 / F32 / F64 view, dst_dtype F8E4M3FN / F8E5M2 in WIRE at body_addr.  With x the element
 *              as fp32 (fp64 rounds once) and FMAX 448 (e4m3fn) or 57344 (e5m2): s = amax(|x|) / FMAX in IEEE fp32
 *              division, 1 when that is 0; q = float8(clamp(x / s, -FMAX, FMAX)), again an IEEE division, then torch's
 *              rounding.  Writes the axis header, the float8 body and the scales.  A NaN or Inf fails the call / job.
 *     restore: float8 WIRE (piece or sub-box) -> float view of F16 / BF16 / F32 / F64: fp32(q) * s in fp32, then
 *              converted once to the destination dtype.
 *     Every other pair under PER_CHANNEL (float8 <-> float8, float8 <-> int, ...) is TSNAP_EUNSUP.
 *   The channel of wire element e is ((e - body_addr) / inner) % channels. */
#define TSNAP_QSCHEME_PER_TENSOR 0
#define TSNAP_QSCHEME_PER_CHANNEL 1
typedef struct tsnap_qchannel {
    int64_t channels;     /* C = piece shape[axis]                                            */
    int64_t inner;        /* prod(piece shape after axis)                                     */
    uint64_t body_addr;   /* WIRE offset of the piece's first int / float8 element (the header is 8 B before it) */
    uint64_t params_addr; /* WIRE offset of scales[C] (f64, zero_points[C] follow; f32 for float8) = body_addr + numel */
    int64_t axis;         /* written into the header on save                                  */
} tsnap_qchannel;

typedef struct tsnap_engine tsnap_engine;
typedef struct tsnap_job tsnap_job;

typedef struct tsnap_engine_config {
    int32_t device;            /* CUDA device ordinal; -1 = host-only engine (CPU tensors only)     */
    int32_t io_threads;        /* native pwrite/pread workers (reference: <=16 concurrent I/Os,
                                  T:knobs.py:38); 0 = default 16                                     */
    uint64_t pinned_slot_bytes; /* size of one pinned ring slot; 0 = default 32 MiB                  */
    int32_t pinned_slots;      /* ring depth; 0 = default 32 (=> 1 GiB pinned, allocated once)       */
    int32_t flags;             /* TSNAP_ENGINE_*; bit 1 is unused */
    uint64_t hbm_staging_bytes; /* cap of the HBM staging arena; 0 = default (grow to payload, keep
                                  >= 1/8 of HBM free)                                                */
} tsnap_engine_config;

#define TSNAP_ENGINE_FSYNC 2u     /* fsync each file before the job reports completion ("durable") */
#define TSNAP_ENGINE_ODIRECT 4u   /* open payload files O_DIRECT: the pinned ring is DMA'd to/from the block device
                                     without a page-cache copy (4 KiB-aligned chunk I/O, ragged tails are written
                                     padded and cut with ftruncate).  Falls back to buffered I/O per file when the
                                     filesystem refuses O_DIRECT (tmpfs).  Replaces aiofiles.open+write / read of
                                     FSStoragePlugin (T:storage_plugins/fs.py:28-51). */
#define TSNAP_ENGINE_TRACE 8u     /* record a per-chunk timeline (tsnap_job_get_trace) */
#define TSNAP_ENGINE_NO_ARENA 16u /* never stage in HBM: dense members are drained straight from the live tensors
                                     (what the engine also does by itself when HBM is too full for an arena — the
                                     reference's OOM fallback to a CPU slab, T:batcher.py:144-152) */

/* ---- library ---------------------------------------------------------------------------------- */
int tsnap_abi_version(void);
const char* tsnap_last_error(void);
size_t tsnap_dtype_size(int dtype);

/* ---- engine: owns streams, the pinned ring, the HBM staging arena and the I/O workers.
 * Replaces the per-call ThreadPoolExecutor(4) + asyncio state machine of execute_write_reqs /
 * execute_read_reqs (T:scheduler.py:222-339, 386-446) for the requests it is given. */
int tsnap_engine_create(const tsnap_engine_config* cfg, tsnap_engine** out);
int tsnap_engine_destroy(tsnap_engine* eng);
/* release cached pinned/HBM memory kept between jobs */
int tsnap_engine_trim(tsnap_engine* eng);

typedef struct tsnap_engine_stats {
    uint64_t pinned_bytes;       /* pinned host bytes currently owned                 */
    uint64_t hbm_arena_bytes;    /* HBM staging arena bytes currently owned           */
    uint64_t kernels_launched;   /* cumulative count of tsnap kernel launches         */
    uint64_t bytes_d2h;          /* cumulative                                        */
    uint64_t bytes_h2d;          /* cumulative                                        */
    uint64_t bytes_written;      /* cumulative bytes handed to pwrite                 */
    uint64_t bytes_read;         /* cumulative bytes obtained from pread              */
    int32_t sm_count;
    int32_t device;
} tsnap_engine_stats;
int tsnap_engine_get_stats(tsnap_engine* eng, tsnap_engine_stats* out);

/* ---- save job: {files, members} -> pack kernel -> pinned ring -> pwrite ------------------------
 * One job == the WriteReqs of one Snapshot.take / async_take on this rank that carry raw tensor
 * bytes (buffer_protocol serializer).  add_file == one WriteReq.path (T:io_types.py:34-37);
 * add_member == one (byte_range, TensorBufferStager) pair of a slab (T:batcher.py:190-202) or the
 * single member of an un-batched tensor/chunk/shard piece.                                        */
int tsnap_save_job_create(tsnap_engine* eng, tsnap_job** out);
/* path: absolute file path (parent directories are created).  nbytes: exact size of the wire image. */
int tsnap_save_job_add_file(tsnap_job* job, const char* path, uint64_t nbytes, int32_t* file_index);
/* desc->dst_space must be TSNAP_SPACE_WIRE; desc->dst_addr = byte offset of the member in the file. */
int tsnap_save_job_add_member(tsnap_job* job, int32_t file_index, const tsnap_copy_desc* desc);
/* Plans, launches the pack kernels on the engine's pack stream (ordered after everything already
 * enqueued on `producer_stream`, a cudaStream_t passed as void*; NULL = legacy default stream) and
 * starts the drain.  Returns immediately. */
int tsnap_save_job_submit(tsnap_job* job, void* producer_stream);
/* Blocks until every read of the source tensors has completed — the async_take return gate
 * (T:snapshot.py:230-317 returns when all write requests are staged, T:scheduler.py:299). */
int tsnap_job_wait_device(tsnap_job* job);
/* Blocks until every file of the job is written (PendingIOWork.complete, T:scheduler.py:196-216). */
int tsnap_job_wait(tsnap_job* job);
/* 1 when finished (successfully or not), 0 otherwise */
int tsnap_job_done(tsnap_job* job);
int tsnap_job_destroy(tsnap_job* job);

typedef struct tsnap_job_stats {
    uint64_t payload_bytes;     /* sum of wire bytes of all files                          */
    uint64_t n_files, n_members, n_tiles_bulk, n_tiles_lsu;
    uint64_t n_kernel_launches;
    double plan_ms;             /* host time spent normalising descriptors + building tables */
    double kernel_ms;           /* CUDA-event time of the pack/unpack kernels (sum)          */
    double kernel_bulk_ms, kernel_lsu_ms;
    double device_done_ms;      /* submit -> all device reads complete (blocking window)     */
    double total_ms;            /* submit -> job complete                                    */
    uint64_t table_h2d_bytes;   /* descriptor/tile tables copied host->device                */
    double slot_wait_ms;        /* time the drain thread was blocked waiting for a free pinned slot   */
    double io_busy_ms;          /* sum over I/O workers of time inside pwrite/pread                   */
    double io_queue_ms;         /* sum over chunks of (write start - D2H complete): I/O queueing delay */
    double copy_ms;             /* CUDA-event span of the payload D2H copies on the copy stream
                                   (first copy start -> last copy end); 0 for load jobs      */
    uint64_t arena_bytes;       /* HBM staging used by the job (0 = arena-less)              */
    uint64_t n_waves;           /* arena waves                                               */
    uint64_t direct_bytes;      /* payload drained straight from the live tensors (no pack)  */
    uint64_t n_memcpy;          /* cudaMemcpyAsync calls issued for payload                  */
    uint64_t bytes_bulk;        /* logical bytes moved by the bulk (TMA) kernel              */
    uint64_t bytes_lsu;         /* logical bytes moved by the LSU kernel                     */
    uint64_t bytes_rows;        /* logical bytes moved run by run by the rows (TMA) kernel   */
    uint64_t n_tiles_rows;
    double kernel_rows_ms;
    uint64_t max_slots_in_flight; /* peak number of ring slots the job held at once (host-memory footprint / slot size) */
    double link_starved_ms;     /* part of slot_wait_ms during which NO payload copy was queued or running on the copy
                                   stream: the link really idled for want of a pinned slot (slot_wait_ms alone also
                                   counts waits behind a full queue of copies, which cost nothing)            */
} tsnap_job_stats;
int tsnap_job_get_stats(tsnap_job* job, tsnap_job_stats* out);

/* ---- HBM staging arena supplied by the caller ---------------------------------------------------
 * By default the engine owns a cudaMalloc'ed arena.  A host runtime with its own device allocator
 * (PyTorch's caching allocator) lends one per job instead, so the staging bytes stay visible to — and
 * reusable by — that allocator: the GPU slab of GPUBatchedBufferStager is a torch.cuda.ByteTensor too
 * (T:batcher.py:147).  tsnap_job_arena_hint reports what the job could use; tsnap_job_set_arena must
 * be called before submit, the memory must stay valid until the job is done.  bytes == 0 selects the
 * arena-less mode for this job (see TSNAP_ENGINE_NO_ARENA). */
typedef struct tsnap_arena_hint {
    uint64_t total_bytes;          /* every device file at a 256 B-aligned offset: one-wave size   */
    uint64_t largest_file_bytes;   /* two-wave operation needs 2 x this                            */
    uint64_t strided_total_bytes;  /* files with a strided / converting member: these cannot be    */
    uint64_t strided_largest_bytes;/*   drained without staging                                    */
} tsnap_arena_hint;
int tsnap_job_arena_hint(tsnap_job* job, tsnap_arena_hint* out);
int tsnap_job_set_arena(tsnap_job* job, void* device_ptr, uint64_t nbytes);

/* Host-memory budget of a job (T:scheduler.py:47-67, 257-272: the reference admits staging while the per-rank budget
 * allows).  The engine's host footprint is its pinned ring; a job never holds more than max(2, bytes / slot size) ring
 * slots at a time (filled by the link and not yet written, or read and not yet uploaded).  0 = no limit beyond the ring. */
int tsnap_job_set_host_budget(tsnap_job* job, uint64_t bytes);

/* ---- timeline of a finished job (engines created with TSNAP_ENGINE_TRACE) ------------------------
 * One record per pipeline event; times are milliseconds since submit on the host's monotonic clock.
 * This is the overlap evidence (pack || D2H || pwrite) without an external timeline profiler. */
enum tsnap_trace_kind {
    TSNAP_TR_PLAN = 0,      /* host planning + table build                                  */
    TSNAP_TR_KERNEL = 1,    /* pack / scatter kernels of one wave (duration from CUDA events) */
    TSNAP_TR_D2H = 2,       /* one chunk: copy-engine busy interval (completion-ordered)      */
    TSNAP_TR_PWRITE = 3,    /* one chunk: inside pwrite                                      */
    TSNAP_TR_SLOT_WAIT = 4, /* drain thread blocked on a free pinned slot                     */
    TSNAP_TR_PREAD = 5,     /* one chunk: inside pread                                       */
    TSNAP_TR_H2D = 6,       /* one chunk: upload, completion-ordered                          */
    TSNAP_TR_OPEN = 7       /* file create/open                                              */
};
typedef struct tsnap_trace_rec {
    int32_t kind;   /* enum tsnap_trace_kind */
    int32_t lane;   /* worker thread ordinal (I/O records), wave (kernel records), else 0 */
    int32_t file;   /* file index or -1 */
    int32_t reserved;
    double t0_ms, t1_ms;
    uint64_t bytes;
} tsnap_trace_rec;
/* copies up to `cap` records into `out`; *n receives the total number available */
int tsnap_job_get_trace(tsnap_job* job, tsnap_trace_rec* out, uint64_t cap, uint64_t* n);

/* ---- roofline probes: the engine's own link and sink, measured with its own ring and workers -----
 * D2H/H2D: `bytes` moved in ring-slot-sized cudaMemcpyAsync chunks between a scratch HBM buffer and
 * the pinned ring.  WRITE: `bytes` written from the ring to fresh files under `dir` by the I/O workers
 * (same chunking/interleaving as a save job, no D2H); READ writes such files (untimed) and times reading
 * them back into the ring.  Only the I/O is timed; the probe removes its files.  out_gbs: bytes/1e9/seconds. */
enum tsnap_probe_kind { TSNAP_PROBE_D2H = 0, TSNAP_PROBE_H2D = 1, TSNAP_PROBE_WRITE = 2, TSNAP_PROBE_READ = 3 };
int tsnap_engine_probe(tsnap_engine* eng, int kind, const char* dir, uint64_t bytes, double* out_gbs);

/* ---- load job: pread -> pinned ring -> H2D -> unpack/scatter kernel ---------------------------
 * add_file == one (batched) ReadReq: path + byte range (T:io_types.py:52-56, merged per file like
 * batch_read_requests T:batcher.py:387-478); add_member == one destination region, with
 * desc->src_space == TSNAP_SPACE_WIRE and desc->src_addr relative to `offset`.                  */
int tsnap_load_job_create(tsnap_engine* eng, tsnap_job** out);
int tsnap_load_job_add_file(tsnap_job* job, const char* path, uint64_t offset, uint64_t nbytes, int32_t* file_index);
int tsnap_load_job_add_member(tsnap_job* job, int32_t file_index, const tsnap_copy_desc* desc);
/* The scatter kernels run on the engine's stream, ORDERED AFTER everything already enqueued on
 * `consumer_stream` (a cudaStream_t passed as void*; NULL = legacy default stream) at submit time — work
 * that still writes the destination tensors (init kernels, an in-flight optimizer step) cannot land after
 * the restored bytes, like the reference's dst.copy_() on the current stream (T:io_preparers/tensor.py:358-360).
 * tsnap_job_wait returns after the scatter kernels have finished, so later work on any stream sees them. */
int tsnap_load_job_submit(tsnap_job* job, void* consumer_stream);

/* ---- stager/consumer seam for arbitrary StoragePlugins -----------------------------------------
 * stage: pack members into ONE pinned host buffer and hand it out (BufferStager.stage_buffer ->
 * memoryview, T:io_types.py:24-31).  The buffer stays valid until tsnap_buffer_release. */
typedef struct tsnap_buffer tsnap_buffer;
int tsnap_stage_submit(tsnap_engine* eng, const tsnap_copy_desc* members, int32_t n_members,
                       uint64_t nbytes, void* producer_stream, tsnap_buffer** out);
int tsnap_buffer_wait_device(tsnap_buffer* buf);
int tsnap_buffer_wait(tsnap_buffer* buf, void** host_ptr, uint64_t* nbytes);
int tsnap_buffer_release(tsnap_buffer* buf);
/* timing/stat record of the staging job behind `buf` (valid after tsnap_buffer_wait) */
int tsnap_buffer_get_stats(tsnap_buffer* buf, tsnap_job_stats* out);
/* consume: scatter a host byte buffer (what StoragePlugin.read produced) into destination views
 * (BufferConsumer.consume_buffer, T:io_types.py:40-49).  Synchronous. */
int tsnap_consume(tsnap_engine* eng, const void* host_buf, uint64_t nbytes,
                  const tsnap_copy_desc* members, int32_t n_members, void* consumer_stream);

/* scatter a wire image that is ALREADY in device memory (e.g. received from a peer GPU over NVLink: one rank reads a
 * replicated file from storage, ncclBroadcast delivers it, every rank scatters it — "read once" restore of DDP state,
 * which the reference re-reads from storage on every rank, T:manifest_ops.py:69-85).  Same members as tsnap_consume,
 * desc->src_addr relative to `device_wire`.  Ordered after `consumer_stream`; synchronous. */
int tsnap_scatter_device(tsnap_engine* eng, const void* device_wire, uint64_t nbytes,
                         const tsnap_copy_desc* members, int32_t n_members, void* consumer_stream);

/* ---- planning introspection (host only; used by the CPU test-suite) -----------------------------
 * Normalises `members` exactly as a job would and reports the tile decomposition. */
typedef struct tsnap_plan_info {
    uint64_t n_members_bulk, n_members_lsu, n_members_host;
    uint64_t n_tiles_bulk, n_tiles_lsu;
    uint64_t bytes_bulk, bytes_lsu, bytes_host;
    uint64_t n_members_rows, n_tiles_rows, bytes_rows;
} tsnap_plan_info;
int tsnap_plan_describe(const tsnap_copy_desc* members, int32_t n_members, uint64_t wire_base_align,
                        tsnap_plan_info* out);
/* Executes the copies on the host with `threads` workers, wire side = wire_buf (host memory).  This is
 * how HOST-space members (CPU tensors) are packed/unpacked; it shares the planner with the device path. */
int tsnap_host_execute(const tsnap_copy_desc* members, int32_t n_members, void* wire_buf,
                       uint64_t wire_nbytes, int32_t threads);

#ifdef __cplusplus
}
#endif
#endif /* TSNAP_B200_H_ */
