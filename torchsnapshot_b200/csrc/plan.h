// Planner: turns tsnap_copy_desc (strided view <-> strided view, torch-style element strides) into
// normalised members and a tile cover.  Shared by the device kernels (kernels.cu) and the host
// executor (plan.cpp), so the CPU test-suite exercises the same decomposition the GPU runs.
//
// What is being restated here: the reference makes every source "contiguous" first
// (T:batcher.py:156 `tensor.contiguous()`, T:serialization.py:196 `tensor.contiguous()`) and then does
// a flat byte copy into [byte_range) of the slab (T:batcher.py:157-158); on restore it narrows both
// sides and calls Tensor.copy_ (T:io_preparers/sharded_tensor.py:285-323).  We never materialise the
// contiguous temporary: the strided gather/scatter IS the copy.
#pragma once
#include <cmath>
#include <cstdint>
#include <string>
#include <vector>

#include "convert.h"

namespace tsnap {

constexpr int kMaxOuter = 8;
constexpr uint32_t kTileBulk = 192 * 1024;  // bytes of one bulk (TMA) tile: a multiple of every ring stage size
constexpr uint32_t kTileLsu = 128 * 1024;  // logical dst bytes of one LSU tile (per-tile setup costs ~2 dependent global round trips)
constexpr uint64_t kBulkMin = 1024;        // contiguous runs shorter than this stay on the LSU path

enum Mode : uint32_t {
    kModeBulk = 0,     // contiguous both sides, src/dst/bytes all multiples of 16 -> cp.async.bulk G->S->G
    kModeContig = 1,   // contiguous both sides, arbitrary alignment -> 16B stores + (shifted) loads
    kModeStrided = 2,  // outer dims x inner contiguous run, `unit`-byte granules
    kModeCast = 3,     // element-wise dtype conversion, strided both sides
    kModeTranspose = 5,  // no run is contiguous on both sides, but each side has a unit-stride dimension (a.t(), permute):
                         // shared-memory tiled transpose over those two dims, coalesced on both sides
    kModeTransposeTma = 6,  // kModeTranspose whose bases and strides are 16 B multiples and whose elements are 2, 4 or 8
                            // bytes: tensor-map TMA tile loads -> 16 B-block transposition in registers -> TMA tile stores
                            // (transpose_tma.cu); chosen per wave by the engine, which owns the tensor maps
    kModeRowsTma = 7,       // kModeRows whose runs are at most kRowsTmaMaxRun long: one tensor-map TMA request moves a box of
                            // many runs (rows x run) instead of one copy-engine request per run; chosen per wave by the engine
    kModeRows = 4,     // kModeStrided whose runs, strides and bases are all multiples of 16 B and whose runs are long
                       // enough for the copy engine: one cp.async.bulk per run (or one per stage on a dense side)
    kModeQChannel = 8,  // kModeCast of a TSNAP_QSCHEME_PER_CHANNEL descriptor: float -> QINT8/QUINT8 (save) or back
                        // (restore) with per-channel parameters; q_zero_point indexes the wave's QChannel table
    kModeQChannelFp8 = 9,  // kModeQChannel with a float8 wire dtype: per-channel scaled float8 (one f32 scale per channel)
};
TSNAP_HD bool qchannel_mode(uint32_t mode) { return mode == kModeQChannel || mode == kModeQChannelFp8; }
constexpr uint32_t kRowsSrcDense = 1;  // Member.shift bits in kModeRows: consecutive runs are adjacent on that side
constexpr uint32_t kRowsDstDense = 2;
constexpr uint64_t kRowsMinRun = 256;  // shorter runs stay on the LSU path (one copy-engine request per run does not pay)

// Per-channel parameters of one kModeQChannel member: absolute addresses in the space the wire image lives in.
// The channel of the wire element at address a is ((a - body) / inner) % channels.
struct alignas(16) QChannel {
    uint64_t body;      // first int element of the piece
    uint64_t params;    // scales[channels] (f64), then zero_points[channels] (i64); float8: scales[channels] (f32)
    uint64_t channels;
    uint64_t inner;
    int64_t axis;
    uint64_t keys;      // save: 16 B per channel in the launch table, zeroed in stream order before the wave: 8 B per
                        // channel of running (min, max) keys of the statistics pass, which the parameter pass replaces by
                        // (1 / scale: f32, zero_point: i32) for the quantising pack, then the scales (f64); float8
                        // replaces the keys by (scale: f32, unused).  (The wire image's parameter area cannot hold them:
                        // it follows a body of any length, so it is not even 4 B aligned in general.)
    uint32_t save;      // 1: float -> int / float8 (statistics, parameters, header), 0: back to float
    uint32_t param_bytes;  // parameter bytes per channel in the wire image: 16 (int8), 4 (float8)
};
constexpr uint32_t kQChannelsPerTile = 8192;  // channels per tile of the header/parameter kernels

// Device-visible member record.  Addresses are absolute for the space they live in.
struct alignas(16) Member {
    uint64_t src;
    uint64_t dst;
    uint64_t bytes;  // logical dst bytes
    uint64_t inner;  // kModeStrided: contiguous run in bytes; kModeCast: contiguous run in ELEMENTS
    uint32_t mode;
    uint32_t unit;    // kModeStrided: granule bytes (1,2,4,8,16)
    uint32_t nouter;
    uint32_t shift;   // kModeContig: dst & 15 (tile boundaries are dst-16B aligned); kModeRows: kRows*Dense flags;
                      // kModeTranspose: index of the src-contiguous dim | index of the dst-contiguous dim << 8
    uint32_t src_dtype;
    uint32_t dst_dtype;
    uint32_t src_esz;
    uint32_t dst_esz;
    int64_t osize[kMaxOuter];
    int64_t sstride[kMaxOuter];  // bytes
    int64_t dstride[kMaxOuter];  // bytes
    double q_scale;              // kModeCast to TSNAP_QINT8/QUINT8: affine quantisation parameters; when `shift` bit 0
    int64_t q_zero_point;        // is set the tile holding the last element appends the 16-byte trailer at dst + bytes
                                 // kModeTransposeTma: index of the member's TmaPair in the wave's tensor-map table;
                                 // kModeQChannel: index of its QChannel in the wave's table
};

// Two CUtensorMap objects (128 B each, 64 B-aligned) of one kModeTransposeTma member, both of rank 5:
// src dims {A, B, o0, o1, o2}, dst dims {B, A, o0, o1, o2} (o* = the remaining dims, highest index first, padded with 1)
struct alignas(64) TmaPair {
    unsigned char src[128];
    unsigned char dst[128];
};
constexpr uint32_t kTmaTileBytes = 32 * 1024;  // payload of one kModeTransposeTma tile
constexpr int kTmaMaxOther = 3;                // dims besides A and B a rank-5 tensor map can carry
// elements per tile along A / B: 32 KiB, both sides >= 8 x 16 B vectors (conflict-free shared-memory block transposition)
// and <= 256 elements (TMA box limit).  Variant (Member.shift bits 16-17): 0 square-ish, 1 twice as long along A,
// 2 twice as long along B — the engine picks the one that pads the member's two extents least.
constexpr uint32_t kTmaVariantShift = 16, kTmaVariants = 3;
TSNAP_HD uint32_t transpose_tma_side_a(uint32_t esz, uint32_t variant) {
    const uint32_t a = esz == 2 ? 128 : 64;
    return variant == 1 ? a * 2 : variant == 2 ? a / 2 : a;
}
TSNAP_HD uint32_t transpose_tma_side_b(uint32_t esz, uint32_t variant) {
    const uint32_t b = esz == 8 ? 64 : 128;
    return variant == 1 ? b / 2 : variant == 2 ? b * 2 : b;
}
TSNAP_HD uint32_t transpose_tma_variant_of(uint32_t shift) { return (shift >> kTmaVariantShift) & 3; }
// kModeRowsTma: tensor maps over 8-byte elements, dims {run / 8, last outer dim, the other outer dims from the last down};
// one tile = one box of `rows` consecutive runs along the last outer dim, at most kTmaTileBytes
constexpr uint64_t kRowsTmaMaxRun = 1024;  // longer runs amortise one copy-engine request per run (the rows kernel)
constexpr int kRowsTmaMaxOuter = 4;
TSNAP_HD uint32_t rows_tma_box_rows(uint64_t run) {
    const uint64_t r = kTmaTileBytes / run;
    return uint32_t(r > 256 ? 256 : r);
}

struct Tile {
    uint32_t member;  // index into the member table of the same kernel
    uint32_t index;   // tile ordinal within the member
};

TSNAP_HD bool engine_mode(uint32_t mode) { return mode == kModeBulk || mode == kModeRows; }  // copy-engine kernels

// kModeTranspose: elements per tile along A (the source-contiguous dim) and B (the destination-contiguous dim):
// 16 KiB of payload per tile (4 x 16 B vectors per thread), small enough for 6 resident CTAs per SM
TSNAP_HD uint32_t transpose_side_a(uint32_t esz) { return esz >= 4 ? 64 : 128; }
TSNAP_HD uint32_t transpose_side_b(uint32_t esz) { return esz == 8 ? 32 : esz == 1 ? 128 : 64; }

// number of tiles a member needs
TSNAP_HD uint64_t tile_count(const Member& m) {
    if (m.bytes == 0) return 0;
    if (m.mode == kModeTranspose || m.mode == kModeTransposeTma) {
        const bool tma = m.mode == kModeTransposeTma;
        const uint32_t a = m.shift & 255, b = (m.shift >> 8) & 255;
        const uint32_t var = transpose_tma_variant_of(m.shift);
        const uint32_t sa = tma ? transpose_tma_side_a(m.unit, var) : transpose_side_a(m.unit), sb = tma ? transpose_tma_side_b(m.unit, var) : transpose_side_b(m.unit);
        uint64_t n = 1;
        for (uint32_t i = 0; i < m.nouter; ++i)
            n *= i == a ? (uint64_t(m.osize[i]) + sa - 1) / sa : i == b ? (uint64_t(m.osize[i]) + sb - 1) / sb : uint64_t(m.osize[i]);
        return n;
    }
    if (m.mode == kModeRowsTma) {
        const uint32_t rows = rows_tma_box_rows(m.inner);
        uint64_t n = (uint64_t(m.osize[m.nouter - 1]) + rows - 1) / rows;
        for (uint32_t i = 0; i + 1 < m.nouter; ++i) n *= uint64_t(m.osize[i]);
        return n;
    }
    if (engine_mode(m.mode)) return (m.bytes + kTileBulk - 1) / kTileBulk;
    if (m.mode == kModeContig) return (m.bytes + m.shift + kTileLsu - 1) / kTileLsu;
    return (m.bytes + kTileLsu - 1) / kTileLsu;
}

// Logical byte range [lo, hi) of tile `index` of member m, the range the kernels copy.  One helper per tile family: a
// kernel knows its family and calls that one, tile_range picks it by mode.  (Transpose and kModeRowsTma tiles are
// blocks of elements or runs instead.)
TSNAP_HD void tile_range_bulk(const Member& m, uint32_t index, uint64_t* lo, uint64_t* hi) {  // kModeBulk, kModeRows
    const uint64_t bytes = m.bytes;
    *lo = uint64_t(index) * kTileBulk;
    *hi = *lo + kTileBulk < bytes ? *lo + kTileBulk : bytes;
}
// kModeContig: tile boundaries sit on 16 B boundaries of the destination, so the first tile is m.shift bytes short
TSNAP_HD void tile_range_contig(const Member& m, uint32_t index, uint64_t* lo, uint64_t* hi) {
    const uint64_t a = uint64_t(index) * kTileLsu;
    *lo = a > m.shift ? a - m.shift : 0;
    *hi = a + kTileLsu - m.shift;
    if (*hi > m.bytes) *hi = m.bytes;
}
// the other LSU modes, and the per-channel statistics and quantising or dequantising passes
TSNAP_HD void tile_range_lsu(const Member& m, uint32_t index, uint64_t* lo, uint64_t* hi) {
    *lo = uint64_t(index) * kTileLsu;
    *hi = *lo + kTileLsu;
    if (*hi > m.bytes) *hi = m.bytes;
}
TSNAP_HD void tile_range(const Member& m, uint32_t index, uint64_t* lo, uint64_t* hi) {
    if (engine_mode(m.mode)) tile_range_bulk(m, index, lo, hi);
    else if (m.mode == kModeContig) tile_range_contig(m, index, lo, hi);
    else tile_range_lsu(m, index, lo, hi);
}

// row index -> byte offsets of the row on both sides; 32-bit division while the row index fits
TSNAP_HD void outer_offsets(const Member& m, uint64_t row, int64_t* so, int64_t* dofs) {
    int64_t s = 0, d = 0;
    if ((row >> 32) == 0) {
        uint32_t r = (uint32_t)row;
        for (int i = (int)m.nouter - 1; i >= 0; --i) {
            const uint64_t sz64 = (uint64_t)m.osize[i];
            uint32_t idx;
            if (sz64 >> 32) {
                idx = r;
                r = 0;
            } else {
                const uint32_t sz = (uint32_t)sz64;
                idx = r % sz;
                r = r / sz;
            }
            s += (int64_t)idx * m.sstride[i];
            d += (int64_t)idx * m.dstride[i];
        }
    } else {
        for (int i = (int)m.nouter - 1; i >= 0; --i) {
            const uint64_t sz = (uint64_t)m.osize[i];
            const uint64_t idx = row % sz;
            row /= sz;
            s += (int64_t)idx * m.sstride[i];
            d += (int64_t)idx * m.dstride[i];
        }
    }
    *so = s;
    *dofs = d;
}

struct NormalizedCopy {
    // 0, 1 or 2 members (bulk body + contiguous tail)
    Member m[2];
    int n = 0;
    int src_space = 0, dst_space = 0;
    QChannel qc{};  // m[0].mode == kModeQChannel: its parameters (m[0].q_zero_point is set by whoever tables them)
};

// Normalises one descriptor.  `src_base`/`dst_base` are added to WIRE-space addresses (the absolute
// address of the wire buffer on the side that executes the copy).  Returns 0 or TSNAP_E*; on error
// `err` holds the reason.  allow_bulk=false keeps everything on LSU modes.
int normalize_copy(const tsnap_copy_desc& d, uint64_t wire_base, bool allow_bulk, NormalizedCopy* out,
                   std::string* err);

size_t dtype_size(int dt);
bool cast_supported(int src_dt, int dst_dt);

// Host execution of one member over logical byte range [lo,hi) (memcpy of runs / scalar casts).
void host_copy_range(const Member& m, uint64_t lo, uint64_t hi);

// Host execution of a whole kModeQChannel member: on save the statistics, parameters, header and quantised body; on
// restore the dequantisation.  Returns TSNAP_EINVAL (with `err`) when a saved channel holds a NaN or Inf.
int host_qchannel(const Member& m, const QChannel& q, std::string* err);
// Every member of a normalised copy on the host
int host_copy_all(const NormalizedCopy& nc, std::string* err);

// Ordered-int key of a float (signed comparison of keys == float comparison for non-NaN values), and back.  The
// statistics pass keeps the running min / max of a channel as two keys; both start at key(0.0f) = 0, so every range
// includes 0 — exactly what both default rules need.
TSNAP_HD int32_t qkey(float f) {
    const int32_t i = (int32_t)f32_bits(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
TSNAP_HD float qkey_value(int32_t k) { return f32_from_bits(uint32_t(k >= 0 ? k : k ^ 0x7fffffff)); }
constexpr int32_t kQKeyMax = 0x7f7fffff;                  // key of FLT_MAX: larger keys are +Inf / NaN
constexpr int32_t kQKeyMin = int32_t(0xff7fffffu ^ 0x7fffffffu);  // key of -FLT_MAX: smaller keys are -Inf / NaN
// (scale, zero_point) of one channel from its (min, max) keys, in double as the default rule states; false on NaN / Inf
TSNAP_HD bool qparams_of(int32_t kmin, int32_t kmax, bool is_signed, double* scale, int64_t* zp) {
    if (kmax > kQKeyMax || kmin < kQKeyMin) return false;
    const double lo = (double)qkey_value(kmin), hi = (double)qkey_value(kmax);
    if (is_signed) {
        const double amax = hi > -lo ? hi : -lo;
        *scale = amax / 127.0;
        if (*scale == 0.0) *scale = 1.0;
        *zp = 0;
    } else {
        *scale = (hi - lo) / 255.0;
        if (*scale == 0.0) *scale = 1.0;
        *zp = (int64_t)rint(-lo / *scale);  // round half to even (default rounding mode)
    }
    return true;
}
// Scale of one per-channel scaled float8 channel from its (min, max) keys: s = amax / FMAX as an IEEE fp32 division,
// 1 when that is 0 (an all-zero channel, or an amax so small that s underflows); false on NaN / Inf
TSNAP_HD bool fp8_scale_of(int32_t kmin, int32_t kmax, uint32_t dt, float* s) {
    if (kmax > kQKeyMax || kmin < kQKeyMin) return false;
    const float lo = qkey_value(kmin), hi = qkey_value(kmax);
    const float amax = hi > -lo ? hi : -lo;
#ifdef __CUDA_ARCH__
    *s = __fdiv_rn(amax, fp8_max(dt));
#else
    *s = amax / fp8_max(dt);
#endif
    if (*s == 0.0f) *s = 1.0f;
    return true;
}

}  // namespace tsnap
